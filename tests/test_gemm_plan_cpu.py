"""Host-side invariants of the in-kernel K-split of the store-epilogue GEMMs (llmlb_b200/csrc/gemm_tc.cu), without a GPU.
The kernel's parts MEET at a counter and each finishes a share of the tile, so a launch is only correct when
  * every CTA of the grid is resident at once: tiles x parts <= 132 (one tile per CTA, one CTA per SM),
  * every part owns at least one K block (an empty part would publish an untouched accumulator),
  * the parts cover K exactly with ceil(K blocks / parts) blocks each,
  * the parked tiles fit the workspace and the counters.
This walks the shard shapes of Llama-3-8B / 70B at tp = 1..8 and a random sweep."""
import ctypes as C
import math
import random

from llmlb_b200 import ffi

SMS, BM, BK, WS_BYTES, COUNTERS = 132, 128, 64, 132 * 128 * 256 * 4, 256


def plan(L, T, N, K):
    out = (C.c_uint32 * 4)()
    L.llmlb_debug_store_split.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    assert L.llmlb_debug_store_split(T, N, K, out) == 0
    return tuple(out)


def check(L, T, N, K):
    bn, tiles, s, ctas = plan(L, T, N, K)
    kb = math.ceil(K / BK)
    assert bn in (16, 32, 64, 128, 256) and bn >= min(T, 256) and tiles == math.ceil(N / BM) * math.ceil(T / bn)
    assert 1 <= s <= 16 and ctas == tiles * s
    if s > 1:
        per = math.ceil(kb / s)
        assert ctas <= SMS, (T, N, K, tiles, s)                       # co-resident
        assert tiles <= COUNTERS
        assert (s - 1) * per < kb <= s * per, (T, N, K, kb, s, per)   # every part non-empty, K covered
        assert per >= 4 or kb < 8                                     # at least 4 K blocks per part
        assert tiles * s * bn * BM * 4 <= WS_BYTES                    # parked fp32 tiles fit
    else:
        # no split only when a split could not help or is not allowed
        assert tiles * 2 > SMS or kb // 4 < 2 or tiles > COUNTERS
    return s


def test_shard_shapes_of_the_benchmark_models():
    L = ffi.lib()
    seen_split = 0
    for hidden, n_heads, n_kv, ffn in ((4096, 32, 8, 14336), (8192, 64, 8, 28672)):
        for tp in (1, 2, 4, 8):
            qkv = (n_heads + 2 * n_kv) // tp * 128
            gu = 2 * ffn // tp
            for T in (5, 7, 16, 17, 33, 64, 65, 128, 129, 256, 300, 512, 2048):
                for n_out, k in ((qkv, hidden), (gu, hidden)):
                    seen_split += check(L, T, n_out, k) > 1
    assert seen_split > 40      # the sweep does exercise the split (tp shards, narrow steps)
    # the cases quoted in DESIGN.md
    assert plan(L, 64, 6144, 4096)[2] == 2          # QKV at 64 streams: 48 tiles -> 96 CTAs
    assert plan(L, 128, 768, 4096)[2:] == (16, 96)  # QKV at tp = 8, 128 streams
    assert plan(L, 64, 28672, 4096)[2] == 1         # gate/up at 64 streams: 224 tiles, no split


def test_random_shapes():
    L = ffi.lib()
    rnd = random.Random(11)
    for _ in range(4000):
        T = rnd.choice([1, 5, 8, 16, 31, 64, 100, 128, 200, 256, 511, 512, 1000, 2048])
        N = rnd.choice([128, 130, 256, 768, 1002, 1536, 3072, 3584, 4096, 6144, 7168, 14336, 28672, 128256])
        K = rnd.choice([64, 128, 520, 512, 1024, 1792, 2048, 3584, 4096, 7168, 8192, 14336])
        check(L, T, N, K)
