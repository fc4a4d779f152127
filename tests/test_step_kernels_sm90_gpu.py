"""-m gpu: the kernels of a wide step (more than 4 tokens) besides the projections and attention — the residual fold +
RMSNorm between projections (rmsnorm_parts_cluster_kernel for 5..256 tokens, rmsnorm_parts_kernel above), the final
RMSNorm (llmlb_op_rmsnorm), RoPE + KV append (llmlb_op_rope_append) and the embedding gather (llmlb_op_embed) — at every
configuration the engine launches, against references that leave no room for an indexing mistake.

  * fold: x + p0 + p1 + ... in fp32, ascending p, is reproduced bit for bit by torch (additions are never contracted).  The
    inputs spread over a wide exponent range, so adding the parts in another order changes bits.  The part stride is the
    engine's T * H, or padded with NaN gaps, so a kernel that derives the stride from T * H fails.
  * RMSNorm: y64 = x rsqrt(mean(x^2) + eps) g in fp64 from the folded x.  y must be the round-to-nearest-even bf16 of some
    z with |z - y64| <= delta |y64|, where delta (norm_rel_bound, about 2^-19) charges the kernel's summation of squares
    (serial per-thread sums, warp tree, 8-warp sum, 4-CTA sum), rsqrtf's 2 ulp, the eps add and the two fp32 products.
    All terms are positive, so the bound is relative; away from a bf16 rounding boundary y is exact.  Per-token scales 8x
    apart, gains that vary per column and an all-zero token make every (token, column) distinguishable.
  * RoPE: each rotated element must be the bf16 rounding of a value within 2^-23 (|a c| + |b s|) of the fp64 rotation of
    the bf16 inputs by the GPU table's fp32 (c, s) (any fp32 evaluation order, with or without FMA).  The K page slot must
    hold the rotated k, the V slot and the V third of qkv the input V, bit for bit; every other pool and qkv byte is
    unchanged.  Positions run up to 131071 in a Llama 3.1-scaled table; sequences are packed with cached context; the page
    table is a permutation over a NaN-poisoned pool; some rows have page -1 (rotate, do not append).
  * embedding: bit-exact, out-of-range ids read row 0.
Every output lands inside a NaN guard band that must come back unchanged, and inputs must come back unchanged too.  A chain
test restates forward_tokens for T > 4 over two Llama-3-8B layers with the debug entry points: each stage meets its own
reference on its actual inputs, and back-to-back launches are bit-identical to the same launches with a synchronize after
each.

FOLD_CASES, RMSNORM_CASES, ROPE_HEADS x ROPE_TOKENS and EMBED_CASES are plain data: tests/test_kernel_coverage_cpu.py runs
them over the fake CUDA runtime and checks that they launch every class of these kernels the engine launches.
"""
import math

import pytest

from test_kernels_sm90_gpu import (EPI_PARTIAL_F32, EPI_SILU_MUL, EPI_STORE_BF16, SENT16, SENT32, _check_random, _Out,
                                   _report, bits_equal)

# ---------------------------------------------------------------------------------------------------------------- cases --
HIDDENS = (512, 2048, 4096, 8192)                 # LLAMA_TINY, LLAMA_MID, Llama-3-8B, Llama-3-70B
FOLD_TOKENS = (5, 6, 17, 128, 255, 256, 257, 300, 640, 2048)     # the cluster kernel up to 256 rows, the plain one above
FOLD_PARTS = (0, 1, 2, 4, 8)                      # 8 = the engine's max_split
STRIDE_PAD = 1028                                 # floats between padded parts: a multiple of 4 (float4 loads), not of H
# (T, H, n_parts, gain, padded part stride)
FOLD_CASES = [(T, H, n, g, pad) for H in HIDDENS for T in FOLD_TOKENS for n in FOLD_PARTS for g in (True, False)
              for pad in ((False, True) if n >= 2 else (False,))]
RMSNORM_CASES = [(T, H) for H in HIDDENS for T in (1, 5, 257, 2048)]
# (n_heads, n_kv) at tp = 1: Llama-3-8B, Llama-3-70B, LLAMA_MID, LLAMA_TINY; tensor-parallel shards of 8B (tp 2 / 4 / 8:
# (16, 4), (8, 2), (4, 1)) and 70B ((32, 4), (16, 2), (8, 1))
ROPE_HEADS = [(32, 8), (64, 8), (16, 4), (8, 2), (4, 1), (32, 4), (16, 2), (8, 1)]
ROPE_TOKENS = (1, 5, 64, 65, 300, 2048)
ROPE_MAX_POS = 131072
EMBED_VOCAB = 128256
EMBED_CASES = [(T, H) for H in HIDDENS for T in (1, 5, 300, 2048)]
EPS = 1e-5
CLUSTER_MAX_TOKENS = 256                          # rmsnorm_parts_launch: 4-CTA clusters up to this many rows

# --------------------------------------------------------------------------------------------------- reference math --
U = 2.0 ** -24          # fp32 unit roundoff


def _gamma(k):
    return k * U / (1 - k * U)


def norm_rel_bound(H, cluster):
    """delta: the relative error of the kernels' y = x r g before its bf16 rounding, r = rsqrtf(sum(x^2) / H + eps).
    Sum of squares: each thread squares (1 rounding) and adds 4 terms per float4 it owns (one per float4 and lane in the
    cluster kernel: H / 16 per CTA, else H / 4, over 256 threads), then 5 warp-shuffle levels, the 8 warp partials and,
    in the cluster kernel, the 4 CTA partials: every term passes at most k roundings, all terms positive, so the sum is
    within gamma(k) relatively.  The division and the eps add: 2 more.  The square root halves it, rsqrtf adds 2 ulp
    (2^-22 relative), the products x r and (x r) g one rounding each."""
    per_thread = -(-(H // 16 if cluster else H // 4) // 256)
    k = 4 * per_thread + 1 + 5 + 7 + (3 if cluster else 0)
    ms = _gamma(k + 2)
    rs = ms / (2 * (1 - ms)) + 4 * U
    return (1 + rs) * (1 + U) ** 2 - 1


def fold_inputs(T, H, n_parts, seed, device):
    """x [T, H] and n_parts parts, fp32 over a wide exponent range (2^-6..2^6 times N(0, 1), parts 2^-12..2^6) with token t
    scaled by 8^(t % 4 - 1); token T // 2 is zero in x and in every part.  gain [H] bf16 around 1, random per column."""
    import torch
    gen = torch.Generator(device=device).manual_seed(seed)
    scale = torch.exp2(3.0 * (torch.arange(T, device=device) % 4 - 1).double()).float()[:, None]

    def spread(lo, hi):
        e = torch.randint(lo, hi, (T, H), generator=gen, device=device).float()
        return torch.randn(T, H, generator=gen, device=device) * torch.exp2(e) * scale
    x = spread(-6, 7)
    parts = [spread(-12, 7) for _ in range(n_parts)]
    for t in [x] + parts:
        t[T // 2] = 0
    gain = (1 + 0.25 * torch.randn(H, generator=gen, device=device)).to(torch.bfloat16)
    return x, parts, gain


def fold_ref(x, parts):
    """((x + p0) + p1) + ... in fp32: what the fold must produce bit for bit."""
    acc = x.clone()
    for p in parts:
        acc = acc + p
    return acc


def norm_ref(x, gain, eps):
    """y64 = x rsqrt(mean(x^2) + eps) g in fp64; eps is the fp32 value the kernel adds."""
    import torch
    xd = x.double()
    eps = float(torch.tensor(eps, dtype=torch.float32))
    return xd * (xd.pow(2).mean(-1, keepdim=True) + eps).rsqrt() * gain.double()


def bf16_dist(got, ref):
    """Distance (fp64) from ref to the reals that round to the bf16 values `got` (to nearest; a tie counts for both sides).
    NaN where got is NaN."""
    import torch
    bits = got.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    mag, neg = bits & 0x7FFF, bits >= 0x8000

    def val(m):
        return (m << 16).view(torch.float32).double()
    a = val(mag)
    up = val(mag + 1)
    dn = torch.where(mag > 0, val((mag - 1).clamp(min=0)), -val(torch.ones_like(mag)))
    lo, hi = (a + dn) / 2, (a + up) / 2
    lo, hi = torch.where(neg, -hi, lo), torch.where(neg, -lo, hi)
    return torch.clamp(torch.maximum(lo - ref, ref - hi), min=0)


def interval_check(got, ref, bound):
    """(elements of bf16 `got` that are not the rounding of any value within `bound` of ref, largest distance / bound over
    the elements with a nonzero bound)."""
    d = bf16_dist(got, ref)
    bad = ~(d <= bound)
    nz = bound > 0
    return int(bad.sum()), float((d[nz] / bound[nz]).max()) if bool(nz.any()) else 0.0


def check_norm(y, x_folded, gain, eps, H, cluster):
    """The y criterion: (mismatches, largest err / bound)."""
    y64 = norm_ref(x_folded, gain, eps)
    return interval_check(y, y64, norm_rel_bound(H, cluster) * y64.abs())


def rope_layout(T):
    """Positions and sequence index of the T rows of one prefill step.  One row: position 131071 (slot 63).  Else three
    sequences packed: T // 3 rows from position 0, T // 3 rows after 63 cached tokens (slot 63, then the next page), and the
    rest ending at position 131071."""
    if T == 1:
        return [ROPE_MAX_POS - 1], [0]
    n0 = n1 = T // 3
    n2 = T - n0 - n1
    pos = list(range(n0)) + list(range(63, 63 + n1)) + list(range(ROPE_MAX_POS - n2, ROPE_MAX_POS))
    return pos, [0] * n0 + [1] * n1 + [2] * n2


def rope_pages(pos, seq, seed, spare=3):
    """page_of_token over a permuted pool: each (sequence, position // 64) gets its own page; every 7th row (from row 3)
    gets -1.  Returns (page list, n_pages)."""
    import torch
    keys = sorted({(s, p // 64) for p, s in zip(pos, seq)})
    n_pages = len(keys) + spare
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
    where = {k: perm[i] for i, k in enumerate(keys)}
    return [-1 if t % 7 == 3 else where[(s, p // 64)] for t, (p, s) in enumerate(zip(pos, seq))], n_pages


def rope_check(qkv_in, qkv_out, pos, table, nh, nkv):
    """(mismatches, largest err / bound) of the rotated q and k heads, plus the V third (bit for bit)."""
    import torch
    T, nr = qkv_in.shape[0], nh + nkv
    x = qkv_in[:, : nr * 128].reshape(T, nr, 128).double()
    a, b = x[..., :64], x[..., 64:]
    cs = table[pos.long()].double()
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    ref = torch.cat([a * c - b * s, b * c + a * s], -1)
    # 2^-23: two roundings (products, difference) of at most 2^-24 of |a c| + |b s| each; the factor covers the second-order
    # term of the difference's rounding
    bound = 2.0 ** -23 * (1 + 2.0 ** -20) * torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], -1)
    n_bad, ratio = interval_check(qkv_out[:, : nr * 128].reshape(T, nr, 128), ref, bound)
    return n_bad + bits_equal(qkv_out[:, nr * 128:], qkv_in[:, nr * 128:]), ratio


def rope_pool_expected(kp, vp, qkv_in, qkv_out, pos, page, nh, nkv):
    """The pools after the append: rows with a page write the rotated k (as left in qkv) and the input v into slot pos % 64."""
    T = qkv_in.shape[0]
    kp, vp = kp.clone(), vp.clone()
    rows = (page >= 0).nonzero().flatten()
    pg, sl = page[rows].long(), (pos[rows] % 64).long()
    kp[pg, :, sl] = qkv_out[:, nh * 128:(nh + nkv) * 128].reshape(T, nkv, 128)[rows]
    vp[pg, :, sl] = qkv_in[:, (nh + nkv) * 128:].reshape(T, nkv, 128)[rows]
    return kp, vp


# ------------------------------------------------------------------------------------------------------- GPU tests --
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(built_lib):
    from llmlb_b200 import ffi
    return ffi.lib()


def _sentinel(n, dtype):
    import torch
    t = torch.empty(n, dtype=dtype, device="cuda")
    if dtype == torch.float32:
        t.view(torch.int32).fill_(SENT32)
    else:
        t.view(torch.int16).fill_(SENT16)
    return t


_FOLD_IDS = ["T%d-H%d-p%d-%s-%s" % (T, H, n, "gain" if g else "fold", "padded" if pad else "dense")
             for T, H, n, g, pad in FOLD_CASES]


@pytest.mark.parametrize("T,H,n_parts,gain,padded", FOLD_CASES, ids=_FOLD_IDS)
def test_fold_and_rmsnorm_against_fp64(L, T, H, n_parts, gain, padded):
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    x0, parts, g = fold_inputs(T, H, n_parts, T * 131 + H + n_parts * 7 + gain, "cuda")
    stride = T * H + (STRIDE_PAD if padded else 0)
    pbuf = _sentinel(max(1, n_parts) * stride + 64, torch.float32)      # NaN gaps between padded parts and after the last
    for i, part in enumerate(parts):
        pbuf[i * stride: i * stride + T * H] = part.flatten()
    pbuf0 = pbuf.clone()
    x = _Out(T, H, torch.float32, pad=0)
    x.slot(0).copy_(x0)
    y = _Out(T, H, torch.bfloat16, pad=0)
    ok(L.llmlb_debug_rmsnorm_parts(x.ptr(), p(pbuf), n_parts, stride, p(g) if gain else None, y.ptr() if gain else None, T, H,
                                   EPS, stream_ptr()))
    sync()
    assert x.untouched_outside(1) == 0 and y.untouched_outside(1 if gain else 0) == 0, "stray writes outside x / y"
    assert bits_equal(pbuf, pbuf0) == 0, "the parts changed"
    want = fold_ref(x0, parts)
    bad = bits_equal(x.slot(0), want)
    if bad:
        i = tuple((x.slot(0).view(torch.int32) != want.view(torch.int32)).nonzero()[0].tolist())
        pytest.fail("%d folded elements differ, first (token, column) %s: got %r want %r" % (bad, i, x.slot(0)[i].item(), want[i].item()))
    if gain:
        n_bad, ratio = check_norm(y.slot(0), want, g, EPS, H, T <= CLUSTER_MAX_TOKENS)
        assert n_bad == 0, "%d normalised elements outside the bound (largest err/bound %.3g)" % (n_bad, ratio)
        _report("fold + norm", ratio)


@pytest.mark.parametrize("T,H", RMSNORM_CASES, ids=["T%d-H%d" % c for c in RMSNORM_CASES])
def test_rmsnorm_against_fp64(L, T, H):
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    x0, _, g = fold_inputs(T, H, 0, T + H, "cuda")
    x = _Out(T, H, torch.float32, pad=0)
    x.slot(0).copy_(x0)
    y = _Out(T, H, torch.bfloat16, pad=0)
    ok(L.llmlb_op_rmsnorm(x.ptr(), p(g), y.ptr(), T, H, EPS, stream_ptr()))
    sync()
    assert y.untouched_outside(1) == 0 and x.untouched_outside(1) == 0 and bits_equal(x.slot(0), x0) == 0
    n_bad, ratio = check_norm(y.slot(0), x0, g, EPS, H, False)
    assert n_bad == 0, "%d elements outside the bound (largest err/bound %.3g)" % (n_bad, ratio)
    _report("final norm", ratio)


@pytest.fixture(scope="module")
def rope_table(built_lib):
    """The Llama 3.1 (llama3-scaled) table over 131072 positions, as the engine builds it."""
    import ctypes as C
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    from llmlb_b200 import ffi
    from rope_oracle import rope_freq_factors
    from rope_scaling_util import LLAMA31_8B, THETA
    f = (C.c_float * 64)(*[float(v) for v in rope_freq_factors(LLAMA31_8B, THETA)])
    tab = torch.empty(ROPE_MAX_POS, 64, 2, dtype=torch.float32, device="cuda")
    ok(ffi.lib().llmlb_op_rope_table_scaled(p(tab), ROPE_MAX_POS, THETA, f, stream_ptr()))
    sync()
    return tab


@pytest.mark.parametrize("T", ROPE_TOKENS)
@pytest.mark.parametrize("nh,nkv", ROPE_HEADS)
def test_rope_append_against_fp64(L, rope_table, nh, nkv, T):
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    seed = nh * 100 + nkv * 10 + T
    pos_l, seq = rope_layout(T)
    page_l, n_pages = rope_pages(pos_l, seq, seed)
    pos = torch.tensor(pos_l, dtype=torch.int32, device="cuda")
    page = torch.tensor(page_l, dtype=torch.int32, device="cuda")
    kp = _sentinel(n_pages * nkv * 64 * 128, torch.bfloat16).view(n_pages, nkv, 64, 128)
    vp = _sentinel(n_pages * nkv * 64 * 128, torch.bfloat16).view(n_pages, nkv, 64, 128)
    kp0, vp0 = kp.clone(), vp.clone()
    W = (nh + 2 * nkv) * 128
    qkv = _Out(T, W, torch.bfloat16, pad=0)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    qkv.slot(0).copy_((torch.randn(T, W, generator=gen, device="cuda") * 4).to(torch.bfloat16))
    qkv_in = qkv.slot(0).clone()
    ok(L.llmlb_op_rope_append(qkv.ptr(), p(pos), p(page), p(rope_table), p(kp), p(vp), T, nh, nkv, stream_ptr()))
    sync()
    assert qkv.untouched_outside(1) == 0, "stray writes outside qkv"
    n_bad, ratio = rope_check(qkv_in, qkv.slot(0), pos, rope_table, nh, nkv)
    assert n_bad == 0, "%d q / k / v elements wrong (largest err/bound %.3g)" % (n_bad, ratio)
    kw, vw = rope_pool_expected(kp0, vp0, qkv_in, qkv.slot(0), pos, page, nh, nkv)
    assert bits_equal(kp, kw) == 0, "K pool differs from the rotated k in its slots, or was written elsewhere"
    assert bits_equal(vp, vw) == 0, "V pool differs from the input v in its slots, or was written elsewhere"
    _report("RoPE", ratio)


_EMBED_TABLE = {}


@pytest.fixture(scope="module", autouse=True)
def _free_embed_table():
    yield
    _EMBED_TABLE.clear()


@pytest.mark.parametrize("T,H", EMBED_CASES, ids=["T%d-H%d" % c for c in EMBED_CASES])
def test_embed_is_bit_exact(L, T, H):
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    V = EMBED_VOCAB
    if H not in _EMBED_TABLE:
        _EMBED_TABLE.clear()
        gen = torch.Generator(device="cuda").manual_seed(H)
        _EMBED_TABLE[H] = torch.randn(V, H, generator=gen, device="cuda").to(torch.bfloat16)
    table = _EMBED_TABLE[H]
    ids = torch.randint(0, V, (T,), generator=torch.Generator().manual_seed(T), dtype=torch.int64)
    special = [V - 1] if T == 1 else [0, V - 1, -1, V, 2 ** 31 - 1]
    ids[: len(special)] = torch.tensor(special)
    ids = ids.to(torch.int32).cuda()
    x = _Out(T, H, torch.float32, pad=0)
    ok(L.llmlb_op_embed(p(table), p(ids), x.ptr(), T, H, V, stream_ptr()))
    sync()
    assert x.untouched_outside(1) == 0
    rows = torch.where((ids >= 0) & (ids < V), ids, torch.zeros_like(ids)).long()     # out-of-range ids read row 0
    assert bits_equal(x.slot(0), table[rows].float()) == 0


# ------------------------------------------------------------------------------------------------- wide-step chain --
CHAIN_TOKENS = (5, 33, 256, 257, 600)
CHAIN_LAYERS = 2
CHAIN_H, CHAIN_QKV, CHAIN_FFN = 4096, 6144, 14336     # Llama-3-8B
CHAIN_MAX_SPLIT = 8                                   # gemm_tc_launch's default in forward_tokens


@pytest.fixture(scope="module")
def wide_weights():
    import torch
    gen = torch.Generator(device="cuda").manual_seed(2025)

    def rnd(*shape, std=0.02):
        return (torch.randn(*shape, generator=gen, device="cuda") * std).to(torch.bfloat16)
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    return [dict(wqkv=rnd(Q, H), wo=rnd(H, H), wgu=rnd(2 * F, H), wdown=rnd(H, F),
                 g_attn=(1 + rnd(H, std=0.1).float()).to(torch.bfloat16), g_ffn=(1 + rnd(H, std=0.1).float()).to(torch.bfloat16))
            for _ in range(CHAIN_LAYERS)]


def _wide_stages(L, lw, buf, attn, T):
    """forward_tokens for T > 4 at tp = 1 as a list of (kind, inputs, launch) stages, attention replaced by the fixed
    input `attn`: per layer fold + attn_norm, QKV (bf16), O (fp32 partials), fold + ffn_norm, gate/up (SiLU), down
    (partials); then the fold of the last partials without a norm.  Each fold is given the n_parts the partial GEMM before
    it reported, as forward_tokens passes them on.  launch() returns the parts count (the fold's input, the GEMM's output)."""
    import ctypes as C
    from gpu_util import ok, p, stream_ptr
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    state = {"pending": 0}

    def fold(gain):
        def run():
            n = state["pending"]
            ok(L.llmlb_debug_rmsnorm_parts(p(buf["x"]), p(buf["parts"]), n, T * H, p(gain), p(buf["y"]) if gain is not None else None,
                                           T, H, EPS, stream_ptr()))
            state["pending"] = 0
            return n
        return ("fold", gain), run

    def gemm(w, xin, out, n_out, k, epi, stride):
        def run():
            n = C.c_uint32(0)
            ok(L.llmlb_debug_gemm(p(w), p(xin), p(out), T, n_out, k, epi, stride, 0, 0, CHAIN_MAX_SPLIT, C.byref(n), stream_ptr()))
            if epi == EPI_PARTIAL_F32:
                state["pending"] = n.value
            return n.value
        return ("gemm", w, xin, out, n_out, k, epi), run
    stages = []
    for l, w in enumerate(lw):
        stages += [fold(w["g_attn"]), gemm(w["wqkv"], buf["y"], buf["qkv"][l], Q, H, EPI_STORE_BF16, Q),
                   gemm(w["wo"], attn, buf["parts"], H, H, EPI_PARTIAL_F32, H), fold(w["g_ffn"]),
                   gemm(w["wgu"], buf["y"], buf["h"][l], 2 * F, H, EPI_SILU_MUL, F),
                   gemm(w["wdown"], buf["h"][l], buf["parts"], H, F, EPI_PARTIAL_F32, H)]
    stages.append(fold(None))
    return stages


class _View:
    """_check_random's view of a GEMM output: part / slot ks of a [T, n_cols] output."""

    def __init__(self, t, T, n_cols):
        self.t, self.T, self.n_cols = t, T, n_cols

    def slot(self, ks):
        return self.t.flatten()[ks * self.T * self.n_cols: (ks + 1) * self.T * self.n_cols].view(self.T, self.n_cols)


@pytest.mark.parametrize("T", CHAIN_TOKENS)
def test_wide_step_chain_meets_each_reference_and_is_bit_identical_back_to_back(L, wide_weights, T):
    """Two Llama-3-8B layers of a T-token prefill step.  With a synchronize after every stage, each stage is checked
    against its reference on the inputs it actually read.  Then every prefix of the stages is launched back to back (the
    GEMMs as programmatic dependents, as in the engine) and x, y, qkv, h and the parts must be bit-identical to the
    synchronised run after the same stage."""
    import torch
    from gpu_util import sync
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    gen = torch.Generator(device="cuda").manual_seed(T)
    x0 = torch.randn(T, H, generator=gen, device="cuda").to(torch.bfloat16).float()     # what the embedding writes
    attn = torch.randn(T, H, generator=gen, device="cuda").to(torch.bfloat16)
    buf = dict(x=torch.empty(T, H, device="cuda"), y=torch.empty(T, H, dtype=torch.bfloat16, device="cuda"),
               parts=torch.empty(CHAIN_MAX_SPLIT * T * H, device="cuda"),
               qkv=[torch.empty(T, Q, dtype=torch.bfloat16, device="cuda") for _ in range(CHAIN_LAYERS)],
               h=[torch.empty(T, F, dtype=torch.bfloat16, device="cuda") for _ in range(CHAIN_LAYERS)])
    names = ["x", "y", "parts"] + ["qkv%d" % l for l in range(CHAIN_LAYERS)] + ["h%d" % l for l in range(CHAIN_LAYERS)]

    def tensors():
        return [buf["x"], buf["y"], buf["parts"]] + buf["qkv"] + buf["h"]

    def reset():
        buf["x"].copy_(x0)
        buf["y"].view(torch.int16).fill_(SENT16)
        buf["parts"].view(torch.int32).fill_(SENT32)
        for t in buf["qkv"] + buf["h"]:
            t.view(torch.int16).fill_(SENT16)

    reset()
    init = [t.clone() for t in tensors()]
    stages = _wide_stages(L, wide_weights, buf, attn, T)
    snaps, counts = [], []
    for spec, run in stages:
        counts.append(run())
        sync()
        snaps.append([t.clone() for t in tensors()])
    # the parts each partial GEMM reports are the parts the next fold folds
    for i, (spec, _) in enumerate(stages):
        if spec[0] == "gemm" and spec[6] == EPI_PARTIAL_F32:
            assert 1 <= counts[i] <= CHAIN_MAX_SPLIT and counts[i + 1] == counts[i], (i, counts)
    assert counts[0] == 0
    # each stage against its reference, on the inputs it read (the snapshot before it)
    prev = init
    for i, (spec, _) in enumerate(stages):
        cur = snaps[i]
        before = dict(zip(names, prev))
        after = dict(zip(names, cur))
        if spec[0] == "fold":
            n = counts[i]
            parts = [_View(before["parts"], T, H).slot(k) for k in range(n)]
            want = fold_ref(before["x"], parts)
            assert bits_equal(after["x"], want) == 0, "stage %d: fold of %d parts" % (i, n)
            if spec[1] is not None:
                n_bad, ratio = check_norm(after["y"], want, spec[1], EPS, H, T <= CLUSTER_MAX_TOKENS)
                assert n_bad == 0, "stage %d: %d normalised elements outside the bound" % (i, n_bad)
                _report("fold + norm", ratio)
        else:
            _, w, xin, out, n_out, k, epi = spec
            src = attn if xin is attn else _snapshot_of(buf, xin, before)
            dst = _snapshot_of(buf, out, after)
            n_cols = n_out // 2 if epi == EPI_SILU_MUL else n_out
            _check_random(_View(dst, T, n_cols), counts[i] if epi == EPI_PARTIAL_F32 else 1, w, src, T, n_out, k, epi, None)
        prev = cur
    # back to back
    for depth in range(1, len(stages) + 1):
        reset()
        stages = _wide_stages(L, wide_weights, buf, attn, T)
        got_counts = [run() for _, run in stages[:depth]]
        sync()
        assert got_counts == counts[:depth]
        for name, got, want in zip(names, tensors(), snaps[depth - 1]):
            assert bits_equal(got, want) == 0, "back to back, %d stages: %s differs from the synchronised run" % (depth, name)


def _snapshot_of(buf, t, state):
    """The snapshot in `state` (name -> tensor) of the buffer t of buf."""
    for name in ("x", "y", "parts"):
        if t is buf[name]:
            return state[name]
    for l in range(CHAIN_LAYERS):
        if t is buf["qkv"][l]:
            return state["qkv%d" % l]
        if t is buf["h"][l]:
            return state["h%d" % l]
    raise KeyError("not a chain buffer")
