"""The launches of the GPU kernel tests (tests/test_kernels_sm90_gpu.py, tests/test_gemv_sm90_gpu.py,
tests/test_step_kernels_sm90_gpu.py, tests/test_decode_attention_sm90_gpu.py), made over the fake CUDA runtime with
FAKE_CUDART_LAUNCH_LOG set: every GEMM case through the entry point it uses there, the wave-tail pair, every decode split,
every decode attention case, the decode layer chain's first two layers, both prefill attention kernels, every GEMV case through
llmlb_op_gemv, the residual fold, RMSNorm, RoPE / KV-append and embedding cases, and the sampler's vocabularies
(tests/test_sampling_sm90_gpu.py).  Nothing executes; the log is the launch
plan of the test cases.  Every section is optional.
usage: kernel_case_sweep.py <cases.json>   ({"gemm": [[T, n_out, K, epi], ...], "wave_tail": [T, n_out, K, main_rows],
                                             "decode_splits": [...], "max_split": n,
                                             "decode": [[splits, n_heads, n_kv, batch], ...], "chain": [batch, ...],
                                             "gemv": [[n_out, K, tokens, epi, norm, out_stride], ...],
                                             "fold": [[T, H, n_parts, gain, part_stride], ...], "rmsnorm": [[T, H], ...],
                                             "rope": [[T, n_heads, n_kv], ...], "embed": [[T, H, vocab], ...],
                                             "sample": [[rows, vocab], ...]})"""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from llmlb_b200 import ffi  # noqa: E402

L = ffi.lib()
cu = ctypes.CDLL("libcudart.so.12")
cu.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
LOG = os.environ["FAKE_CUDART_LAUNCH_LOG"]


def dmalloc(n):
    p = ctypes.c_void_p()
    assert cu.cudaMalloc(ctypes.byref(p), n) == 0
    return p


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


cases = json.load(open(sys.argv[1]))
w, x, out = dmalloc(1 << 33), dmalloc(1 << 30), dmalloc(1 << 31)          # address space only: nothing is executed
parts = ctypes.c_uint32()
for T, n_out, k, epi in cases.get("gemm", []):
    mark("gemm %d %d %d %d" % (T, n_out, k, epi))
    n_cols = n_out // 2 if epi == 2 else n_out
    if epi == 4:
        ffi.check(L.llmlb_debug_gemm(w, x, out, T, n_out, k, epi, n_cols, 0, 0, cases["max_split"], ctypes.byref(parts), None))
    else:
        ffi.check(L.llmlb_op_gemm(w, x, out, T, n_out, k, epi, n_cols, 0, None))
if "wave_tail" in cases:
    T, n_out, k, rows = cases["wave_tail"]
    for epi in (2, 3):
        mark("wave tail %d" % epi)
        n_cols = n_out // 2 if epi == 2 else n_out
        for row0, n_rows in ((0, 0), (0, rows), (rows, n_out - rows)):
            ffi.check(L.llmlb_debug_gemm(w, x, out, T, n_out, k, epi, n_cols, row0, n_rows, cases["max_split"], ctypes.byref(parts), None))
rope, ws = dmalloc(1 << 20), dmalloc(256)
for sp in cases.get("decode_splits", []):
    mark("decode %d" % sp)
    ffi.check(L.llmlb_op_decode_attention(x, w, w, out, 66, out, out, 5, out, 32, 8, rope, sp, 5, ws, None))
for sp, nh, nkv, B in cases.get("decode", []):
    mark("decode case %d %d %d %d" % (sp, nh, nkv, B))
    ffi.check(L.llmlb_debug_decode_attention(x, w, w, out, 66, out, out, B, out, nh, nkv, rope, sp, B, ws, 0, None))


def chain_arg(name, l):
    """The decode layer chain's arguments: weights and pools in w, activations in x, block tables and lengths in out."""
    if name == "bt_stride":
        return 66
    return {"x": x, "qkv": x, "attn": x, "h": x, "bt": out, "rows": out, "seq_lens": out, "rope": rope, "ws": ws}.get(name, w)


for B in cases.get("chain", []):
    mark("chain B=%d" % B)
    import test_gemv_sm90_gpu as GV
    GV.chain_launches(L, B, 2, chain_arg, lambda: None)
if "decode_splits" in cases:
    mark("prefill")
    ffi.check(L.llmlb_op_prefill_attention_tc(x, 300, w, w, 80, out, 66, out, 3, out, 32, 8, None))
    ffi.check(L.llmlb_op_prefill_attention(x, w, w, out, 66, out, 3, out, 32, 8, None))
gain = dmalloc(1 << 20)
for n_out, k, n_tok, epi, norm, out_stride in cases.get("gemv", []):
    mark("gemv %d %d %d %d %d" % (n_out, k, n_tok, epi, norm))
    ffi.check(L.llmlb_op_gemv(w, x, gain if norm else None, 1e-5, out, n_tok, n_out, k, epi, out_stride, None))
for T, H, n_parts, g, stride in cases.get("fold", []):
    mark("fold %d %d %d %d %d" % (T, H, n_parts, g, stride))
    ffi.check(L.llmlb_debug_rmsnorm_parts(out, w, n_parts, stride, gain if g else None, x if g else None, T, H, 1e-5, None))
for T, H in cases.get("rmsnorm", []):
    mark("rmsnorm %d %d" % (T, H))
    ffi.check(L.llmlb_op_rmsnorm(out, gain, x, T, H, 1e-5, None))
for T, nh, nkv in cases.get("rope", []):
    mark("rope %d %d %d" % (T, nh, nkv))
    ffi.check(L.llmlb_op_rope_append(x, out, out, rope, w, w, T, nh, nkv, None))
for T, H, V in cases.get("embed", []):
    mark("embed %d %d" % (T, H))
    ffi.check(L.llmlb_op_embed(w, x, out, T, H, V, None))
for R, V in cases.get("sample", []):
    mark("sample %d %d" % (R, V))
    ffi.check(L.llmlb_op_sample(w, R, V, x, x, x, x, x, out, None))
