"""-m gpu: the decode GEMVs — the K-split kernel (gemv_ks.cu) and the row-owner kernel (gemv.cu) — at every configuration
the engine dispatches, against references that would notice a subtle indexing mistake.  Everything goes through
llmlb_op_gemv, which dispatches like the engine's gemv_decode: the K-split kernel where ks_pick finds a team shape, else the
row-owner kernel, one token per pass when the activations of all tokens do not fit its shared-memory stage.

Two kinds of input, as for the GEMMs (tests/test_kernels_sm90_gpu.py, whose helpers this file uses):
  * index probe.  The unit of K in both kernels is one lane's 16-byte load, 8 consecutive elements (an "8-group").  In
    gemv_ks, chunk k // 256 belongs to team warp (k // 256) % TW at loop slot (k // 256) // TW, and to lane (k % 256) // 8;
    in the row-owner kernel the lane is the same and the chunk is the trip.  Each token's activation is m-hot: one element
    (+-1) in each of m distinct 8-groups, the element within the group varying.  Over the rounds of a case every token hits
    every 8-group of K, each token in its own order.  probe_weights' entries have 8 significant bits and lie within 2^10 of
    each other in magnitude (multiples of 2^-13 below 2^4), so m <= 32 of them add exactly in fp32 (< 2^9 in steps of 2^-13:
    22 bits), a probe-valued residual included.  The fp32 epilogues must match bit for bit, the bf16 one after
    round-to-nearest-even, SiLU within its evaluation bound.
    NORM: x_t is +-c at the hits and 0 elsewhere, eps = 1 - m c^2 / K, so mean(x^2) + eps = 1 and rsqrtf gives 1 within a
    few ulp; gain_k = 2^e_k / c with e_k random in {-1, 0, 1}.  The normalised activation is then exactly +-2^e_k after the
    kernel's bf16 rounding, and with m <= 16 the products again add exactly (< 2^9 in steps of 2^-14: 23 bits, 24 with the
    residual).  The random exponents catch a gain read at the wrong k.
  * random data against fp64, with zeroed W rows, one W row x 2^10, a zeroed token and per-token scales 8x apart (a token
    that borrows another's RMS scale is off by 8x).  Elementwise bounds derived from |y| |W|^T.
Every output lands inside a NaN-sentinel guard band (rows before and after, out_stride = n_cols + PAD) that must come back
unchanged.  A chain test runs four Llama-3-8B decode layers, decode attention included, back to back and checks them bit for
bit against the same launches with a synchronize after each and against a CUDA-graph replay.

GEMV_CASES is plain data: tests/test_kernel_coverage_cpu.py runs it through llmlb_op_gemv over the fake CUDA runtime and
checks that it launches every GEMV class the engine launches at Llama-3-8B, LLAMA_MID and Llama-3-70B shapes.
"""
import math

import pytest

from test_kernels_sm90_gpu import (BF16_U, EPI_RESID_F32, EPI_SILU_MUL, EPI_STORE_BF16, EPI_STORE_F32, _Out, _report,
                                   bits_equal, gemm_acc_bound, probe_weights, silu_eval_rel, silu_mul_ref)
from test_step_kernels_sm90_gpu import rope_table  # noqa: F401 (fixture)

# ---------------------------------------------------------------------------------------------------------------- cases --
ALL = (EPI_STORE_BF16, EPI_RESID_F32, EPI_SILU_MUL, EPI_STORE_F32)
NO_SILU = (EPI_STORE_BF16, EPI_RESID_F32, EPI_STORE_F32)      # odd n_out: SiLU needs whole (gate, up) row pairs
BOTH = (False, True)                                           # bf16 activations / fp32 activations with fused RMSNorm

# (n_out, K, token counts, epilogues, norms).  The dispatch of each, as ks_pick and llmlb_op_gemv make it: K-split kernel
# (B, CW) with TW warps per team where TW * CW * 256 == K, 2 <= TW <= 16, B * CW <= 4; else the row-owner kernel.
GEMV_CASES = [
    # K-split, TW 16 CW 1 at B = 1..4: Llama-3-8B QKV / O / gate-up and the LM head
    (6144, 4096, (1, 2, 3, 4), ALL, BOTH),
    (28672, 4096, (1, 4), (EPI_SILU_MUL,), (True,)),
    (128256, 4096, (1, 4), (EPI_STORE_F32,), (True,)),
    (266, 4096, (1, 2, 3, 4), ALL, BOTH),          # 133 row pairs over 132 CTAs: one CTA range is two pairs long
    (263, 4096, (1, 3), NO_SILU, BOTH),            # odd n_out: the last row pair is half empty
    (1, 4096, (1, 4), NO_SILU, BOTH),
    (2, 4096, (1, 2), ALL, BOTH),
    (3, 4096, (1, 4), NO_SILU, BOTH),
    # Llama-3-8B down (K 14336): K-split TW 14 CW 4 at B = 1, the row-owner kernel at B = 2..4
    (4096, 14336, (1, 2, 3, 4), ALL, BOTH),
    # K-split TW 14 CW 2 at B = 1, 2 (two spare warps)
    (1002, 7168, (1, 2), ALL, BOTH),
    # Llama-3-70B (K 8192): K-split TW 16 CW 2 at B = 1, 2; the row-owner kernel with and without NORM at B = 3, 4
    (10240, 8192, (1, 2, 3, 4), ALL, BOTH),
    # Llama-3-70B down (K 28672): the row-owner kernel with 56 / 112 / 168 KiB of activations at B = 1..3, one token per
    # pass at B = 4.  One CTA per SM (over 100 registers x 512 threads) is 2112 warps; 8454 rows are 2114 row groups of 4,
    # so two warps go round their group loop a second time, onto the ragged last group of 2 rows
    (8454, 28672, (1, 2, 3, 4), ALL, BOTH),
    # LLAMA_MID (K 2048): K-split TW 8
    (3072, 2048, (1, 2, 3, 4), ALL, BOTH),
    # K-split teams with spare warps or few warps: TW 14 (K 3584), 7 (1792), 3 (768), 2 (512)
    (264, 3584, (1, 2, 3, 4), ALL, BOTH),
    (1002, 1792, (1, 2, 3, 4), ALL, BOTH),
    (266, 768, (1, 2, 3, 4), ALL, BOTH),
    (264, 512, (1, 2, 3, 4), ALL, BOTH),
    (263, 512, (1, 4), NO_SILU, BOTH),
    # the row-owner kernel at K % 256 != 0: a single 8-group, a lane's second 16-byte load only partly in range (264, 520),
    # a ragged last trip after 16 full ones (4104)
    (264, 8, (1, 2, 3, 4), ALL, BOTH),
    (263, 264, (1, 2, 3, 4), NO_SILU, BOTH),
    (266, 520, (1, 2, 3, 4), ALL, BOTH),
    (1002, 4104, (1, 2, 3, 4), ALL, BOTH),
    # K = 256 is one chunk: a K-split team of one warp would need 16 teams, so the row-owner kernel takes it
    (264, 256, (1, 2, 3, 4), ALL, BOTH),
]
PAD = 40                     # out_stride = n_cols + PAD, as _Out lays outputs out
M_PLAIN, M_NORM = 32, 16     # hits per token and round (see the module docstring)
PROBE_C = 0.25               # |x| at the hits of the NORM probe
TOKEN_SCALES = (1.0, 8.0, 0.0, 0.125)   # random data: token t is scaled by TOKEN_SCALES[t]


def gemv_params():
    return [(N, Kd, B, epi, norm) for N, Kd, toks, epis, norms in GEMV_CASES for B in toks for epi in epis for norm in norms]


def n_cols(N, epi):
    return N // 2 if epi == EPI_SILU_MUL else N


# --------------------------------------------------------------------------------------------------- reference math --
def probe_rounds(K, norm):
    G = K // 8
    return -(-G // min(M_NORM if norm else M_PLAIN, G))


def probe_plan(B, K, norm, seed):
    """The rounds of the m-hot probe: a list of (cols [B, m], signs [B, m]) on the CPU.  Token t walks the 8-groups in its
    own random order, m distinct groups per round; probe_rounds(K, norm) rounds hit every group.  The element within the
    group cycles through 0..7 along the walk, from a random start per token."""
    import torch
    G = K // 8
    m = min(M_NORM if norm else M_PLAIN, G)
    gen = torch.Generator().manual_seed(seed)
    perms = torch.stack([torch.randperm(G, generator=gen) for _ in range(B)])
    start = torch.randint(0, 8, (B, 1), generator=gen)
    plan = []
    for r in range(probe_rounds(K, norm)):
        j = r * m + torch.arange(m)
        cols = perms[:, j % G] * 8 + (start + j) % 8
        signs = torch.randint(0, 2, (B, m), generator=gen) * 2 - 1
        plan.append((cols, signs))
    return plan


def probe_norm_setup(K, m, seed, device):
    """NORM probe: gain exponents e_k in {-1, 0, 1}, the bf16 gain 2^e_k / c and eps = 1 - m c^2 / K."""
    import torch
    e = torch.randint(-1, 2, (K,), generator=torch.Generator().manual_seed(seed)).to(device)
    gain = torch.exp2(e.double() - math.log2(PROBE_C)).to(torch.bfloat16)
    return e, gain, 1.0 - m * PROBE_C ** 2 / K


def probe_x_and_ref(w, cols, signs, gain_exp=None):
    """The probe activation (bf16 +-1, or fp32 +-c when gain_exp is given: NORM) and its exact product acc [B, N] in fp32."""
    import torch
    B, m = cols.shape
    N, K = w.shape
    cols, signs = cols.to(w.device), signs.to(w.device)
    v = signs.double()
    if gain_exp is None:
        x = torch.zeros(B, K, dtype=torch.bfloat16, device=w.device)
        x.scatter_(1, cols, signs.to(torch.bfloat16))
    else:
        x = torch.zeros(B, K, dtype=torch.float32, device=w.device)
        x.scatter_(1, cols, signs.float() * PROBE_C)
        v = v * torch.exp2(gain_exp[cols].double())          # the normalised activation: exactly +-2^e_k
    acc = (w[:, cols.reshape(-1)].double().view(N, B, m) * v[None]).sum(-1).t()
    return x, acc.float() + 0.0                               # + 0.0: a sum of zeros is +0, as the kernels produce


def silu_probe_bound(ref, g):
    """The GEMM probe's SiLU bound (BF16_U + silu_eval_rel(g) (1 + BF16_U)) |ref|, plus what an m-hot sum can reach and two
    hits cannot: for g < -88 __expf(-g) overflows to inf and the kernel's silu is -0, an error of |ref|; a result in bf16's
    subnormal range is off by up to half its spacing, 2^-134."""
    import torch
    under = torch.where(g < -88, ref.abs(), torch.zeros_like(ref))
    return (BF16_U + silu_eval_rel(g) * (1 + BF16_U)) * ref.abs() + under + 2.0 ** -134


def probe_mismatches(got, acc, epi, prev=None):
    """The number of elements of `got` (a [B, n_cols] output) that the exact probe product `acc` rejects."""
    import torch
    if epi == EPI_STORE_F32:
        return bits_equal(got, acc)
    if epi == EPI_STORE_BF16:
        return bits_equal(got, acc.to(torch.bfloat16))
    if epi == EPI_RESID_F32:
        return bits_equal(got, prev + acc)
    ref, g, _ = silu_mul_ref(acc)
    return int((~((got.double() - ref).abs() <= silu_probe_bound(ref, g))).sum())


def rs_rel_err(K):
    """Relative error of the kernels' fp32 rsqrt(mean(x^2) + eps) and of y = x rs g before its bf16 rounding: the sum of K
    squares (K roundings of positive terms), the division and the eps add (2), halved by the square root; rsqrtf 2 ulp; the
    two products 2 roundings: ((K + 2) / 2 + 4 + 2) 2^-24 <= (K / 2 + 8) 2^-24."""
    return (K / 2 + 8) * 2.0 ** -24


TREE_ADDS = 5 + 16          # roundings after a lane's own sum: log2(32) shuffle levels, then up to 16 team partials


def random_ref(w, x, epi, prev=None, gain=None, eps=0.0):
    """fp64 reference and elementwise bound of the GEMV on random data: (ref, bound, group).
      acc = y W^T with y = x (bf16 input) or y = x rs g, rs = (mean(x^2) + eps)^-1/2 (NORM, fp32 input)
      |err acc| <= gemm_acc_bound(|y|, |W|)                          a lane's serial fp32 sums: the statistical sqrt(K)
                                                                     model of the GEMM tests, not a worst case
                 + TREE_ADDS 2^-24 |y| |W|^T                         the 5-level warp shuffle tree and the in-order sum of
                                                                     up to 16 team warps, at their worst case
                 + (2^-8 + rs_rel_err(K)) |y| |W|^T                 NORM: y rounded to bf16 after an inexact rs (may flip)
    then the epilogue: the residual add (2^-23 (|prev| + |y| |W|^T)), bf16 rounding (2^-8 of the result), or SiLU*up
    propagated through silu' <= 1.1 as for the GEMMs."""
    import torch
    K = w.shape[1]
    wd = w.double()
    wa = wd.abs()
    if gain is None:
        y = x.double()
    else:
        xd = x.double()
        y = xd * (xd.pow(2).mean(-1, keepdim=True) + eps).rsqrt() * gain.double()
    ya = y.abs()
    acc = y @ wd.t()
    yw = ya @ wa.t()
    b_acc = gemm_acc_bound(ya, wa, K) + TREE_ADDS * 2.0 ** -24 * yw
    if gain is not None:
        b_acc = b_acc + (BF16_U + rs_rel_err(K)) * yw
    if epi == EPI_SILU_MUL:
        ref, g, u = silu_mul_ref(acc)
        bg, bu = b_acc[:, 0::2], b_acc[:, 1::2]
        sg = (g / (1 + (-g).exp())).abs()
        prop = 1.1 * bg * (u.abs() + bu) + sg * bu
        bound = prop + (BF16_U + silu_eval_rel(g.abs() + bg) * (1 + BF16_U)) * (ref.abs() + prop)
        group = "SiLU"
    else:
        ref, bound = acc, b_acc
        if epi == EPI_RESID_F32:
            ref = acc + prev.double()
            bound = bound + 2.0 ** -23 * (prev.double().abs() + yw)
        if epi == EPI_STORE_BF16:
            bound = bound + BF16_U * (ref.abs() + bound)
        group = "bf16 out" if epi == EPI_STORE_BF16 else "fp32 out"
    return ref, bound, "GEMV NORM" if gain is not None else "GEMV " + group


def over_bound(got, ref, bound):
    """(elements over the bound (NaN counts), largest err / bound over the elements with a nonzero bound)."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    nz = bound > 0
    return int(bad.sum()), float((err[nz] / bound[nz]).max()) if bool(nz.any()) else 0.0


def random_w(N, K, seed, device):
    """Random bf16 W with zeroed rows 5, 102, ... and row N // 3 scaled by 2^10: a misplaced row shows up even where the
    true output is zero or small."""
    import torch
    w = torch.randn(N, K, generator=torch.Generator(device=device).manual_seed(seed), device=device).to(torch.bfloat16)
    w[5::97] = 0
    w[N // 3] *= 1024
    return w


def random_x(B, K, norm, seed, device):
    """Random x [B, K], token t scaled by TOKEN_SCALES[t] (bf16, or fp32 with NORM), and a bf16 gain around 1."""
    import torch
    gen = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(B, K, generator=gen, device=device) * torch.tensor(TOKEN_SCALES[:B], device=device)[:, None]
    gain = (1 + 0.25 * torch.randn(K, generator=gen, device=device)).to(torch.bfloat16)
    return (x if norm else x.to(torch.bfloat16)), gain


# ------------------------------------------------------------------------------------------------------- GPU tests --
pytestmark = pytest.mark.gpu
RANDOM_EPS = 1e-5


@pytest.fixture(scope="module")
def L(built_lib):
    from llmlb_b200 import ffi
    return ffi.lib()


_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _free_cache():
    yield
    _CACHE.clear()


def _cached(key, make):
    """One tensor per kind (the cases come grouped by shape): the largest W here is 1 GB."""
    if _CACHE.get(key[0], (None,))[0] != key:
        _CACHE.pop(key[0], None)
        _CACHE[key[0]] = (key, make())
    return _CACHE[key[0]][1]


def _probe_w(N, K):
    import torch

    def make():
        gen = torch.Generator(device="cuda").manual_seed(N * 31 + K)
        return torch.cat([probe_weights(min(8192, N - r), K, gen, "cuda") for r in range(0, N, 8192)])
    return _cached(("probe", N, K), make)


def _gemv(L, w, x, gain, eps, out, B, N, K, epi):
    from gpu_util import ok, p, stream_ptr
    ok(L.llmlb_op_gemv(p(w), p(x), p(gain), eps, out.ptr(), B, N, K, epi, out.stride, stream_ptr()))


def _out(B, N, epi):
    import torch
    return _Out(B, n_cols(N, epi), torch.bfloat16 if epi in (EPI_STORE_BF16, EPI_SILU_MUL) else torch.float32, pad=PAD)


_PARAMS = gemv_params()
_IDS = ["N%d-K%d-B%d-epi%d-%s" % (N, Kd, B, epi, "norm" if norm else "bf16x") for N, Kd, B, epi, norm in _PARAMS]


@pytest.mark.parametrize("N,K,B,epi,norm", _PARAMS, ids=_IDS)
def test_gemv_index_probe_is_exact(L, N, K, B, epi, norm):
    import torch
    from gpu_util import sync
    seed = N * 7919 + K * 31 + B * 5 + epi * 2 + norm
    w = _probe_w(N, K)
    plan = probe_plan(B, K, norm, seed)
    gain_exp, gain, eps = None, None, 0.0
    if norm:
        gain_exp, gain, eps = probe_norm_setup(K, plan[0][0].shape[1], seed, "cuda")
    prev = probe_weights(B, n_cols(N, epi), torch.Generator(device="cuda").manual_seed(seed), "cuda").float()
    for rnd, (cols, signs) in enumerate(plan):
        x, acc = probe_x_and_ref(w, cols, signs, gain_exp)
        out = _out(B, N, epi)
        if epi == EPI_RESID_F32:
            out.slot(0).copy_(prev)
        _gemv(L, w, x, gain, eps, out, B, N, K, epi)
        sync()
        where = "round %d of %d, token 0 hits columns %s" % (rnd, len(plan), sorted(cols[0].tolist())[:8])
        assert out.untouched_outside(1) == 0, "stray writes outside the output; " + where
        bad = probe_mismatches(out.slot(0), acc, epi, prev)
        if bad and epi != EPI_SILU_MUL:
            got = out.slot(0)
            want = (prev + acc if epi == EPI_RESID_F32 else acc).to(got.dtype)
            it = torch.int32 if got.dtype == torch.float32 else torch.int16
            i = tuple((got.contiguous().view(it) != want.contiguous().view(it)).nonzero()[0].tolist())
            where += "; first mismatch (token, row) %s: got %r want %r" % (i, got[i].item(), want[i].item())
        assert bad == 0, "%d mismatches; %s" % (bad, where)


@pytest.mark.parametrize("N,K,B,epi,norm", _PARAMS, ids=_IDS)
def test_gemv_random_data_within_fp64_bound(L, N, K, B, epi, norm):
    import torch
    from gpu_util import sync
    seed = N + K + B + epi + norm
    w = _cached(("random", N, K), lambda: random_w(N, K, N + K, "cuda"))
    x, gain = random_x(B, K, norm, seed, "cuda")
    out = _out(B, N, epi)
    prev = None
    if epi == EPI_RESID_F32:
        prev = torch.randn(B, N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
        out.slot(0).copy_(prev)
    _gemv(L, w, x, gain if norm else None, RANDOM_EPS, out, B, N, K, epi)
    sync()
    assert out.untouched_outside(1) == 0
    ref, bound, group = random_ref(w, x, epi, prev, gain if norm else None, float(torch.tensor(RANDOM_EPS).float()))
    got = out.slot(0)
    n_bad, ratio = over_bound(got, ref, bound)
    if n_bad:
        bad = ~((got.double() - ref).abs() <= bound)
        i = tuple(bad.nonzero()[0].tolist())
        pytest.fail("%d elements over the bound, first (token, row) %s: got %g want %g bound %g" % (
            n_bad, i, got[i].item(), ref[i].item(), bound[i].item()))
    _report(group, ratio)


# ------------------------------------------------------------------------------------------------ one decode layer --
CHAIN_LAYERS = 4
CHAIN_H, CHAIN_QKV, CHAIN_FFN = 4096, 6144, 14336     # Llama-3-8B
CHAIN_HEADS, CHAIN_KV = 32, 8
CHAIN_BATCHES = (1, 2, 3, 4)                          # decode_splits: 16 at B = 1, 2, 11 (a cluster of 8) at 3, 9 at 4
CHAIN_CTX = (300, 4097)                               # each layer's context per sequence (with the new token): in this range


@pytest.fixture(scope="module")
def chain_weights():
    import torch
    gen = torch.Generator(device="cuda").manual_seed(2024)

    def rnd(*shape, std=0.02):
        return (torch.randn(*shape, generator=gen, device="cuda") * std).to(torch.bfloat16)
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    return [dict(wqkv=rnd(Q, H), wo=rnd(H, H), wgu=rnd(2 * F, H), wdown=rnd(H, F),
                 g_attn=(1 + rnd(H, std=0.1).float()).to(torch.bfloat16), g_ffn=(1 + rnd(H, std=0.1).float()).to(torch.bfloat16))
            for _ in range(CHAIN_LAYERS)]


def chain_launches(L, B, depth, arg, stream, after=None):
    """The decode layer as forward_tokens launches it at B <= 4 sequences and tp = 1, layers 0..depth-1: QKV (NORM, bf16
    out), decode attention (a plain launch at layer 0, a programmatic dependent from layer 1 on, with the engine's split for
    B), O (residual into x), gate/up (NORM, SiLU), down (residual into x).  arg(name, l) is layer l's device pointer of
    wqkv, wo, wgu, wdown, g_attn, g_ffn, x, qkv, attn, h, kp, vp, bt, rows, seq_lens, rope, ws, or its bt_stride;
    after(launch index in the layer, l) runs after each launch."""
    from llmlb_b200 import ffi
    from test_decode_attention_sm90_gpu import decode_splits
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    splits = decode_splits(B, CHAIN_HEADS)

    def gemv(l, w, xin, gain, out, n_out, k, epi, stride):
        ffi.check(L.llmlb_op_gemv(arg(w, l), arg(xin, l), arg(gain, l) if gain else None, 1e-5, arg(out, l), B, n_out, k, epi, stride,
                                  stream()))

    def attention(l):
        ffi.check(L.llmlb_debug_decode_attention(arg("qkv", l), arg("kp", l), arg("vp", l), arg("bt", l), arg("bt_stride", l),
                                                 arg("rows", l), arg("seq_lens", l), B, arg("attn", l), CHAIN_HEADS, CHAIN_KV,
                                                 arg("rope", l), splits, B, arg("ws", l), int(l > 0), stream()))
    for l in range(depth):
        launches = [lambda: gemv(l, "wqkv", "x", "g_attn", "qkv", Q, H, EPI_STORE_BF16, Q), lambda: attention(l),
                    lambda: gemv(l, "wo", "attn", None, "x", H, H, EPI_RESID_F32, H),
                    lambda: gemv(l, "wgu", "x", "g_ffn", "h", 2 * F, H, EPI_SILU_MUL, F),
                    lambda: gemv(l, "wdown", "h", None, "x", H, F, EPI_RESID_F32, H)]
        for i, run in enumerate(launches):
            run()
            if after:
                after(i, l)


@pytest.mark.parametrize("B", CHAIN_BATCHES)
def test_decode_layer_chain_is_bit_identical_back_to_back_synchronised_and_graphed(L, chain_weights, rope_table, B):
    """Four layers, each with its own K/V pool and contexts of 300..4097 tokens, launched back to back on one stream as the
    engine does (the K-split GEMVs and, from layer 1 on, decode attention as programmatic dependents: attention's prologue
    prefetches K/V while the QKV GEMV runs and must read qkv only after it; the O GEMV streams its weights while attention
    runs) must give exactly what the same launches give with a synchronize after each, and so must a CUDA-graph replay of
    them — qkv, attn, h, the appended K/V of every layer and x after every layer.  Each layer's attention output and
    pools, from the synchronised run, meet the reference of tests/test_decode_attention_sm90_gpu.py on that layer's own qkv."""
    import torch
    from gpu_util import p, sync
    from test_decode_attention_sm90_gpu import Pool, check_launch, decode_splits, rope_rotate
    from test_kernels_sm90_gpu import SENT16
    H, Q, F = CHAIN_H, CHAIN_QKV, CHAIN_FFN
    gen = torch.Generator(device="cuda").manual_seed(B)
    x0 = torch.randn(B, H, generator=gen, device="cuda")
    x = torch.empty_like(x0)
    qkv = [torch.empty(B, Q, dtype=torch.bfloat16, device="cuda") for _ in range(CHAIN_LAYERS)]
    attn = [torch.empty(B, H, dtype=torch.bfloat16, device="cuda") for _ in range(CHAIN_LAYERS)]
    h = [torch.empty(B, F, dtype=torch.bfloat16, device="cuda") for _ in range(CHAIN_LAYERS)]
    lens = torch.randint(CHAIN_CTX[0], CHAIN_CTX[1] + 1, (CHAIN_LAYERS, B), generator=torch.Generator().manual_seed(B)).tolist()
    lens[0][0] = CHAIN_CTX[1]
    pools, ctx = [], []
    for l in range(CHAIN_LAYERS):
        pool = Pool(CHAIN_KV, lens[l], 100 * B + l)
        ck = [torch.randn(n - 1, CHAIN_KV, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens[l]]
        cv = [torch.randn(n - 1, CHAIN_KV, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens[l]]
        for i in range(B):
            pool.write(i, 0, ck[i], cv[i])
        pools.append(pool)
        ctx.append((ck, cv))
    pool0 = [(pl.kp.clone(), pl.vp.clone()) for pl in pools]
    seq_lens = [torch.tensor(n, dtype=torch.int32, device="cuda") for n in lens]
    ws = torch.zeros(256, dtype=torch.uint8, device="cuda")
    shared = dict(x=x, rope=rope_table, ws=ws)

    def arg(name, l):
        if name in chain_weights[l]:
            return p(chain_weights[l][name])
        if name in shared:
            return p(shared[name])
        if name in ("kp", "vp", "bt", "rows"):
            return p(getattr(pools[l], name))
        if name == "bt_stride":
            return pools[l].bt_stride
        return p({"qkv": qkv, "attn": attn, "h": h, "seq_lens": seq_lens}[name][l])

    def stream():
        from gpu_util import stream_ptr
        return stream_ptr()

    def reset():
        x.copy_(x0)
        for t in qkv + attn + h:
            t.view(torch.int16).fill_(SENT16)
        for pl, (k0, v0) in zip(pools, pool0):
            pl.kp.copy_(k0)
            pl.vp.copy_(v0)

    reset()
    snaps = []

    def after(i, l):
        torch.cuda.current_stream().synchronize()
        if i == 4:
            snaps.append(x.clone())
    chain_launches(L, B, CHAIN_LAYERS, arg, stream, after)
    sync()
    want = {"qkv": [t.clone() for t in qkv], "attn": [t.clone() for t in attn], "h": [t.clone() for t in h],
            "kp": [pl.kp.clone() for pl in pools], "vp": [pl.vp.clone() for pl in pools]}
    assert all(bool(torch.isfinite(t.float()).all()) for t in want["qkv"] + want["attn"] + want["h"] + snaps)
    assert all(bits_equal(snaps[l], snaps[l + 1]) > 0 for l in range(CHAIN_LAYERS - 1))    # every layer moves x
    splits, ratio = decode_splits(B, CHAIN_HEADS), 0.0
    for l, pl in enumerate(pools):
        rot = rope_rotate(L, want["qkv"][l], seq_lens[l] - 1, rope_table, CHAIN_HEADS, CHAIN_KV)
        sync()
        ratio = max(ratio, check_launch(L, rope_table, pl, pool0[l][0], pool0[l][1], want["qkv"][l], rot, want["attn"][l], ctx[l][0],
                                        ctx[l][1], seq_lens[l], CHAIN_HEADS, CHAIN_KV, splits, "layer %d" % l))
    _report("decode layer chain attention", ratio)

    def check(mode, depth):
        got = {"qkv": qkv, "attn": attn, "h": h, "kp": [pl.kp for pl in pools], "vp": [pl.vp for pl in pools]}
        for l in range(depth):
            for name in ("qkv", "attn", "h", "kp", "vp"):
                assert bits_equal(got[name][l], want[name][l]) == 0, "%s, %d layers: %s of layer %d differs" % (mode, depth, name, l)
        for l in range(depth, CHAIN_LAYERS):
            assert bits_equal(pools[l].kp, pool0[l][0]) == 0 and bits_equal(pools[l].vp, pool0[l][1]) == 0, (mode, depth, l)
        assert bits_equal(x, snaps[depth - 1]) == 0, "%s: x after layer %d differs" % (mode, depth - 1)

    for depth in range(1, CHAIN_LAYERS + 1):
        reset()
        chain_launches(L, B, depth, arg, stream)
        sync()
        check("back to back", depth)
    for depth in range(1, CHAIN_LAYERS + 1):     # the eager runs above made every shared-memory opt-in outside capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            chain_launches(L, B, depth, arg, stream)
        reset()
        g.replay()
        sync()
        check("graph replay", depth)
