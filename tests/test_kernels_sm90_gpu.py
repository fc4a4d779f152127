"""-m gpu: the Hopper wgmma projection GEMMs (gemm_tc.cu, gemm_tc2.cu) and the attention kernels at every configuration the
engine dispatches, against references that would notice a subtle indexing mistake.

GEMMs, two kinds of input:
  * index probe: every activation row is the sum of two one-hot vectors (x[t, a_t] = x[t, b_t] = 1, a_t and b_t in different
    64-wide K slabs and different k16 steps), so out[t, n] = W[n, a_t] + W[n, b_t] exactly in fp32 — every partial sum,
    K-split part and fold included.  The fp32 epilogues must match bit for bit, the bf16 one after round-to-nearest-even.
    Over the probe rounds of one case every k16 step of every slab is hit, the K tail included.
  * random data against x.double() @ w.double().T with an elementwise bound derived from |X| |W|^T.
Every output lands in a larger buffer (rows before and after, out_stride > n_cols) whose outside is a NaN bit pattern that must
come back unchanged.

GEMM_CASES, DECODE_SPLITS and PREFILL_IMPLS are plain data: tests/test_kernel_coverage_cpu.py runs them through the launch
planner over the fake CUDA runtime and checks that they launch every kernel instantiation and K-split class the engine does.
"""
import math

import pytest

# ---------------------------------------------------------------------------------------------------------------- cases --
EPI_STORE_BF16, EPI_RESID_F32, EPI_SILU_MUL, EPI_STORE_F32, EPI_PARTIAL_F32 = 0, 1, 2, 3, 4

# (tokens T, n_out, K, epilogues).  T hits every token tile width (BN 16 / 32 / 64 / 128 / 256) and both sides of each
# boundary; n_out is a multiple of 256, 128 mod 256, or ragged (+8, +120, +136); K % 64 is 0, 8 or 56.  Paths, as
# gemm_tc_launch picks them: 1-CTA gemm_tc without K-split, with the in-kernel store K-split, with the atomic residual
# split; the CTA-pair gemm_tc2 with the store epilogues and with the residual / partial split.
GEMM_CASES = [
    (5, 1032, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_PARTIAL_F32)),  # BN 16, store K-split, 8 parts
    (5, 16384, 64, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32, EPI_PARTIAL_F32)),   # one K slab: no split
    (16, 384, 568, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32)),
    (17, 8824, 1032, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                  # BN 32, 69 tiles: no split
    (17, 4096, 4096, (EPI_RESID_F32, EPI_PARTIAL_F32)),                               # BN 32, residual split
    (24, 4352, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                  # BN 32, store K-split
    (32, 4096, 14336, (EPI_PARTIAL_F32, EPI_RESID_F32)),                              # down projection, 4 parts
    (33, 640, 4152, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32)),
    (63, 2048, 8, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32)),      # K shorter than one slab
    (64, 6144, 4096, (EPI_STORE_BF16, EPI_STORE_F32)),
    (64, 1032, 14336, (EPI_RESID_F32, EPI_PARTIAL_F32)),                              # 8 parts
    (65, 1160, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                  # BN 128, store K-split
    (127, 8960, 520, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32)),   # BN 128, 70 tiles: no split
    (128, 4216, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32, EPI_PARTIAL_F32)),
    (129, 12416, 1032, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                # CTA pairs, half-empty last pair
    (129, 4096, 4096, (EPI_RESID_F32, EPI_PARTIAL_F32)),                              # CTA pairs, 4 parts
    (255, 1024, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                 # narrow: BN 256 with store K-split
    (256, 14336, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),
    (257, 6144, 4096, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32)),  # a 1-token second tile
    (300, 28672, 4096, (EPI_SILU_MUL,)),                                              # Llama-3-8B gate/up
    (300, 4096, 14336, (EPI_RESID_F32, EPI_PARTIAL_F32)),
    (512, 4104, 4152, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32)),                 # narrow, 2 parts
    (512, 6144, 4096, (EPI_STORE_BF16,)),
    (640, 6144, 1032, (EPI_STORE_BF16, EPI_SILU_MUL, EPI_STORE_F32, EPI_RESID_F32, EPI_PARTIAL_F32)),
    (640, 4096, 14336, (EPI_PARTIAL_F32,)),
]
GEMM_MAX_SPLIT = 8           # what the engine and llmlb_op_gemm allow the residual / partial split
# the engine's wave tail (engine.cu, proj()): Llama-3-8B gate/up at T = 600
WAVE_TAIL_CASE = (600, 28672, 4096)
DECODE_SPLITS = [1, 2, 4, 8, 16]
PREFILL_IMPLS = ["tc", "mma"]
SM_COUNT = 132


def wave_tail_rows(T, n_out, sms=SM_COUNT):
    """The row count of the main launch of proj()'s wave tail (the tail covers the rest), or None when proj() does not
    split this projection.  Restates engine.cu: CTA-pair tiles of 256 rows x 256 tokens in waves of sms / 2 pairs."""
    if T <= 128 or n_out % 256:
        return None
    t_tiles, m_pairs, pairs = -(-T // 256), n_out // 256, sms // 2
    waves, rem = divmod(m_pairs * t_tiles, pairs)
    if waves >= 2 and rem > 0 and rem % t_tiles == 0 and rem // t_tiles <= 2:
        return (m_pairs - rem // t_tiles) * 256
    return None


# --------------------------------------------------------------------------------------------------- reference math --
# Every tolerance below is a formula of the inputs.  Unit roundoff: fp32 carries 24 significant bits, bf16 8, so rounding
# to nearest is off by at most 2^-24 resp. 2^-8 of the value.  Tensor-core additions may truncate: 2^-23 per addition.
C_ACC = 2.0   # fp32 accumulation of K products: c * 2^-24 * sqrt(K) * sum_k |x_k| |w_k| (independent per-add rounding)
BF16_U = 2.0 ** -8


def probe_hits(T, K, rnd):
    """Probe round `rnd` of a T x K activation: per token (a_t, b_t), b_t = -1 when K has a single k16 step.  a_t walks the
    k16 steps in order over the rounds (rounds = ceil(steps / T) hit every step); b_t is in another 64-wide slab (when there
    is one) and another k16 position within its slab.  The column inside a step varies with the token."""
    steps = [(16 * s, min(16 * s + 16, K)) for s in range((K + 15) // 16)]
    n = len(steps)
    hits = []
    for t in range(T):
        j = rnd * T + t
        sa = j % n
        lo, hi = steps[sa]
        a = lo + (5 * j + rnd) % (hi - lo)
        b = -1
        for d in range(n):
            sb = (sa + n // 2 + 1 + d) % n
            if sb == sa or sb % 4 == sa % 4:
                continue
            if sb // 4 == sa // 4 and n > 4:
                continue
            lo, hi = steps[sb]
            b = lo + (3 * j + 1) % (hi - lo)
            break
        hits.append((a, b))
    return hits


def probe_rounds(T, K):
    return -(-((K + 15) // 16) // T)


def probe_weights(n_out, K, gen, device):
    """bf16 W whose entries are exact and within 2^9 of each other in magnitude: +-2^e (1 + m / 128), e in [-6, 3], about
    10 % zeros.  Two of them (and a residual of the same kind) add exactly in fp32."""
    import torch
    e = torch.randint(-6, 4, (n_out, K), generator=gen, device=device).double()
    m = torch.randint(0, 128, (n_out, K), generator=gen, device=device).double()
    s = torch.randint(0, 2, (n_out, K), generator=gen, device=device).double() * 2 - 1
    keep = (torch.randint(0, 10, (n_out, K), generator=gen, device=device) > 0).double()
    w = (s * keep * torch.exp2(e) * (1 + m / 128)).to(torch.bfloat16)
    return w.masked_fill_(w == 0, 0)     # +0, not -0: an accumulator that starts at +0 never produces -0


def probe_x_and_ref(w, T, K, rnd):
    """The probe activation of round `rnd` and its exact fp32 product out[t, n] = W[n, a_t] + W[n, b_t]."""
    import torch
    hits = probe_hits(T, K, rnd)
    a = torch.tensor([h[0] for h in hits], device=w.device)
    b = torch.tensor([h[1] for h in hits], device=w.device)
    x = torch.zeros(T, K, dtype=torch.bfloat16, device=w.device)
    x[torch.arange(T, device=w.device), a] = 1
    has_b = b >= 0
    x[torch.arange(T, device=w.device)[has_b], b[has_b]] = 1
    ref = w[:, a].t().float() + torch.where(has_b[:, None], w[:, b.clamp(min=0)].t().float(), torch.zeros((), device=w.device))
    return x, ref


def bits_equal(got, want):
    """Bit-for-bit equality of two tensors of the same dtype (NaN patterns included); returns the mismatch count."""
    import torch
    it = {torch.float32: torch.int32, torch.bfloat16: torch.int16}[got.dtype]
    return int((got.contiguous().view(it) != want.contiguous().view(it)).sum())


def silu_mul_ref(acc):
    """silu(g) * u of interleaved (gate, up) rows, in fp64: acc [T, n_out] -> ([T, n_out / 2] result, g, u)."""
    g, u = acc[:, 0::2].double(), acc[:, 1::2].double()
    return g / (1 + (-g).exp()) * u, g, u


def silu_eval_rel(g):
    """Relative error of the SiLU*up epilogue before its bf16 rounding: __expf at most 2 + floor(1.173 |x|) ulp (CUDA C
    Programming Guide; we use 2 + 2|x|), 1 + e^-g rounded once (at most 1/2 ulp), __fdividef 2 ulp, the product with u
    1/2 ulp: (5 + 2|g|) ulp of 2^-23."""
    return (5 + 2 * g.abs()) * 2.0 ** -23


def gemm_acc_bound(xa, wa, K):
    """c * 2^-24 * sqrt(K) * (|X| |W|^T): the fp32 accumulation error of K bf16 products (products are exact in fp32)."""
    return C_ACC * 2.0 ** -24 * math.sqrt(K) * (xa @ wa.t())


def attention_ref(q, k, v, q_pos, p_round):
    """Causal attention in fp64 and its elementwise error bound.
    q [n, nh, 128] (the values the kernel multiplies), k, v [S, nkv, 128] every key of the sequence, q_pos [n] positions.
    Returns ref [n, nh, 128] and bound [n, nh, 128]:
      |err| <= (p_round + (2 S_t + 16) 2^-23) sum_s p_s |v_s|          P rounded to bf16 (p_round = 2^-8 when the kernel
                                                                       does), fp32 P.V accumulation and per-block rescales
             + sum_s p_s e_s (|v_s| + |ref|)                            score errors, e_s = 2^-23 (130 A_s + 8 (|s| + |s_max|))
                                                                       + 2^-21 with A_s = sum_d |q_d| |k_sd| / sqrt(128):
                                                                       fp32 dot product, scale, max subtraction, exp2 ulps
             + 2^-8 |ref|                                               bf16 output
             + S_t 2^-126 max |v|                                       exp2 underflow flushed to zero"""
    import torch
    nh, nkv = q.shape[1], k.shape[1]
    g = nh // nkv
    S = k.shape[0]
    qd = q.double()
    kd, vd = k.double().repeat_interleave(g, 1), v.double().repeat_interleave(g, 1)
    sc = torch.einsum("thd,shd->hts", qd, kd) / math.sqrt(128)
    mask = torch.arange(S, device=q.device)[None, :] > q_pos.to(q.device)[:, None]
    sc = sc.masked_fill(mask[None], float("-inf"))
    p = torch.softmax(sc, -1)
    ref = torch.einsum("hts,shd->htd", p, vd)
    pv = torch.einsum("hts,shd->htd", p, vd.abs())
    A = torch.einsum("thd,shd->hts", qd.abs(), kd.abs()) / math.sqrt(128)
    smax = sc.amax(-1, keepdim=True)
    e = 2.0 ** -23 * (130 * A + 8 * (sc.masked_fill(mask[None], 0).abs() + smax.abs())) + 2.0 ** -21
    pe = (p * e).masked_fill(mask[None], 0)
    n_keys = (~mask).sum(-1).double()[None, :, None]
    bound = ((p_round + (2 * n_keys + 16) * 2.0 ** -23) * pv + torch.einsum("hts,shd->htd", pe, vd.abs())
             + pe.sum(-1, keepdim=True) * ref.abs() + BF16_U * ref.abs() + n_keys * 2.0 ** -126 * v.double().abs().max())
    return ref.permute(1, 0, 2), bound.permute(1, 0, 2)


# ------------------------------------------------------------------------------------------------------- GPU tests --
pytestmark = pytest.mark.gpu

SENT32, SENT16 = 0x7FC0BEEF, 0x7FC5        # NaN sentinels of the guard bands (fp32, bf16)
PRE, POST, PAD = 3, 5, 40                   # guard rows before / after the output, extra columns per row


def _lib():
    from llmlb_b200 import ffi
    return ffi.lib()


class _Out:
    """An output of `slots` x [T, n_cols] inside a sentinel-filled buffer of (PRE + slots T + POST) rows of n_cols + PAD."""

    def __init__(self, T, n_cols, dtype, slots=1, pad=PAD):
        import torch
        self.T, self.n_cols, self.slots, self.stride = T, n_cols, slots, n_cols + pad
        self.buf = torch.empty(PRE + slots * T + POST, self.stride, dtype=dtype, device="cuda")
        it = torch.int32 if dtype == torch.float32 else torch.int16
        self.sent = SENT32 if dtype == torch.float32 else SENT16
        self.buf.view(it).fill_(self.sent - (1 << 32) if it == torch.int32 and self.sent >= 1 << 31 else self.sent)
        self.it = it

    def ptr(self):
        import ctypes as C
        return C.c_void_p(self.buf[PRE].data_ptr())

    def slot(self, ks):
        return self.buf[PRE + ks * self.T: PRE + (ks + 1) * self.T, : self.n_cols]

    def untouched_outside(self, used_slots, col_ranges=None):
        """Number of elements outside slots [0, used_slots) x [0, n_cols) that lost their sentinel."""
        import torch
        inside = torch.zeros_like(self.buf, dtype=torch.bool)
        inside[PRE: PRE + used_slots * self.T, : self.n_cols] = True
        b = self.buf.view(self.it)
        want = torch.full_like(b, self.sent - (1 << 32) if self.it == torch.int32 and self.sent >= 1 << 31 else self.sent)
        return int(((b != want) & ~inside).sum())


def _call(L, w, x, out, T, n_out, K, epi, row0=0, n_rows=0, debug=False):
    import ctypes as C
    from gpu_util import ok, p, stream_ptr
    if not debug:
        ok(L.llmlb_op_gemm(p(w), p(x), out.ptr(), T, n_out, K, epi, out.stride, 0, stream_ptr()))
        return GEMM_MAX_SPLIT if epi == EPI_RESID_F32 else 1
    parts = C.c_uint32(0)
    ok(L.llmlb_debug_gemm(p(w), p(x), out.ptr(), T, n_out, K, epi, out.stride, row0, n_rows, GEMM_MAX_SPLIT, C.byref(parts),
                          stream_ptr()))
    return parts.value


def _gemm_out(T, n_out, epi):
    import torch
    n_cols = n_out // 2 if epi == EPI_SILU_MUL else n_out
    dt = torch.float32 if epi in (EPI_RESID_F32, EPI_STORE_F32, EPI_PARTIAL_F32) else torch.bfloat16
    return _Out(T, n_cols, dt, GEMM_MAX_SPLIT if epi == EPI_PARTIAL_F32 else 1)


def _fold(out, parts):
    acc = out.slot(0).clone()
    for ks in range(1, parts):
        acc += out.slot(ks)        # part order, as rmsnorm_parts folds them
    return acc


@pytest.fixture(scope="module")
def L(built_lib):
    return _lib()


_GEMM_PARAMS = [(T, N, K, epi) for T, N, K, epis in GEMM_CASES for epi in epis]


@pytest.mark.parametrize("T,N,K,epi", _GEMM_PARAMS, ids=["T%d-N%d-K%d-epi%d" % c for c in _GEMM_PARAMS])
def test_gemm_index_probe_is_bit_exact(L, T, N, K, epi):
    import torch
    from gpu_util import sync
    gen = torch.Generator(device="cuda").manual_seed(T * 7919 + N * 31 + K + epi)
    w = probe_weights(N, K, gen, "cuda")
    prev = probe_weights(T, N, gen, "cuda").float() if epi == EPI_RESID_F32 else None   # exact sums with the products
    for rnd in range(probe_rounds(T, K)):
        x, acc = probe_x_and_ref(w, T, K, rnd)
        out = _gemm_out(T, N, epi)
        if prev is not None:
            out.slot(0).copy_(prev)
        parts = _call(L, w, x, out, T, N, K, epi, debug=epi == EPI_PARTIAL_F32)
        sync()
        where = "round %d hits %s" % (rnd, probe_hits(T, K, rnd)[:4])
        used = parts if epi == EPI_PARTIAL_F32 else 1
        assert out.untouched_outside(used) == 0, "stray writes outside the output; " + where
        if epi == EPI_STORE_F32:
            assert bits_equal(out.slot(0), acc) == 0, where
        elif epi == EPI_STORE_BF16:
            assert bits_equal(out.slot(0), acc.to(torch.bfloat16)) == 0, where
        elif epi == EPI_RESID_F32:
            assert bits_equal(out.slot(0), prev + acc) == 0, where
        elif epi == EPI_PARTIAL_F32:
            assert 1 <= parts <= GEMM_MAX_SPLIT
            assert bits_equal(_fold(out, parts), acc) == 0, where
        else:
            ref, gg, _ = silu_mul_ref(acc)
            bound = (BF16_U + silu_eval_rel(gg) * (1 + BF16_U)) * ref.abs()
            err = (out.slot(0).double() - ref).abs()
            assert bool((err <= bound).all()), "%s: max err/bound %.3g" % (where, (err / bound.clamp(min=1e-300)).max().item())


_RATIOS = {}


def _report(group, ratio):
    _RATIOS[group] = max(_RATIOS.get(group, 0.0), ratio)
    print("largest err/bound so far, %s: %.4f" % (group, _RATIOS[group]))


def _random_gemm_inputs(T, N, K, seed):
    """Random bf16 inputs with zeroed W rows and x tokens and one W row scaled by 2^10: a misplaced row or token shows up
    even where the true output is zero or small."""
    from gpu_util import bf16_randn
    w = bf16_randn((N, K), seed=seed)
    x = bf16_randn((T, K), seed=seed + 1)
    w[5::97] = 0
    w[N // 3] *= 1024
    x[3::7] = 0
    return w, x


def _check_random(out, parts, w, x, T, N, K, epi, prev):
    import torch
    xa, wa = x.double().abs(), w.double().abs()
    acc = x.double() @ w.double().t()
    xw = xa @ wa.t()
    b_acc = gemm_acc_bound(xa, wa, K) + parts * 2.0 ** -23 * xw       # + the fold / atomic adds of the K-split parts
    if epi == EPI_SILU_MUL:
        ref, g, u = silu_mul_ref(acc)
        bg, bu = b_acc[:, 0::2], b_acc[:, 1::2]
        sg = (g / (1 + (-g).exp())).abs()
        # silu' <= 1.1: |silu(g') u' - silu(g) u| <= 1.1 bg (|u| + bu) + |silu(g)| bu
        prop = 1.1 * bg * (u.abs() + bu) + sg * bu
        bound = prop + (BF16_U + silu_eval_rel(g.abs() + bg) * (1 + BF16_U)) * (ref.abs() + prop)
        got = out.slot(0).double()
        group = "SiLU"
    else:
        ref = acc + (prev.double() if prev is not None else 0)
        bound = b_acc + (parts + 1) * 2.0 ** -23 * (prev.double().abs() if prev is not None else 0)
        if epi == EPI_STORE_BF16:
            bound = bound + BF16_U * (ref.abs() + bound)
        group = "GEMM random, bf16 out" if epi == EPI_STORE_BF16 else "GEMM random, fp32 out"
        got = (_fold(out, parts) if epi == EPI_PARTIAL_F32 else out.slot(0)).double()
    err = (got - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), "%d elements over the bound, first at %s: got %g want %g bound %g" % (
        int(bad.sum()), tuple(bad.nonzero()[0].tolist()), got[bad][0].item(), ref[bad][0].item(), bound[bad][0].item())
    # a zero bound (zeroed W row or x token) admits only an exact zero; report the ratio over the others
    nz = bound > 0
    _report(group, float((err[nz] / bound[nz]).max()) if bool(nz.any()) else 0.0)


@pytest.mark.parametrize("T,N,K,epi", _GEMM_PARAMS, ids=["T%d-N%d-K%d-epi%d" % c for c in _GEMM_PARAMS])
def test_gemm_random_data_within_fp64_bound(L, T, N, K, epi):
    import torch
    from gpu_util import sync
    w, x = _random_gemm_inputs(T, N, K, seed=T + N + K + epi)
    out = _gemm_out(T, N, epi)
    prev = None
    if epi == EPI_RESID_F32:
        prev = torch.randn(T, N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(T))
        out.slot(0).copy_(prev)
    parts = _call(L, w, x, out, T, N, K, epi, debug=epi == EPI_PARTIAL_F32)
    sync()
    assert out.untouched_outside(parts if epi == EPI_PARTIAL_F32 else 1) == 0
    _check_random(out, parts, w, x, T, N, K, epi, prev)


@pytest.mark.parametrize("epi", [EPI_SILU_MUL, EPI_STORE_F32])
def test_gemm_wave_tail_pair_equals_one_full_launch(L, epi):
    """proj()'s wave tail: the CTA-pair launch over rows [0, r) plus the 128-row K-split launch over [r, n_out) must give
    exactly what one launch over all rows gives (index probe), and stay within the fp64 bound on random data."""
    import torch
    from gpu_util import sync
    T, N, K = WAVE_TAIL_CASE
    r = wave_tail_rows(T, N)
    assert r == 28160
    gen = torch.Generator(device="cuda").manual_seed(600)
    w = probe_weights(N, K, gen, "cuda")
    for rnd in range(probe_rounds(T, K)):
        x, acc = probe_x_and_ref(w, T, K, rnd)
        full, pair = _gemm_out(T, N, epi), _gemm_out(T, N, epi)
        _call(L, w, x, full, T, N, K, epi, debug=True)
        _call(L, w, x, pair, T, N, K, epi, row0=0, n_rows=r, debug=True)
        _call(L, w, x, pair, T, N, K, epi, row0=r, n_rows=N - r, debug=True)
        sync()
        assert pair.untouched_outside(1) == 0 and full.untouched_outside(1) == 0
        assert bits_equal(pair.slot(0), full.slot(0)) == 0
        if epi == EPI_STORE_F32:
            assert bits_equal(pair.slot(0), acc) == 0
    w, x = _random_gemm_inputs(T, N, K, seed=601)
    pair = _gemm_out(T, N, epi)
    _call(L, w, x, pair, T, N, K, epi, row0=0, n_rows=r, debug=True)
    _call(L, w, x, pair, T, N, K, epi, row0=r, n_rows=N - r, debug=True)
    sync()
    assert pair.untouched_outside(1) == 0
    _check_random(pair, 1, w, x, T, N, K, epi, None)


# ------------------------------------------------------------------------------------------------- attention ------
POISON_K, POISON_V = 30.0, 1000.0


def _poison(shape, mag, gen, device="cuda"):
    """Large finite bf16 values +-mag (1 +- 1/8): what a reused page holds past a sequence's horizon.  The kernels rely on
    0 * finite = 0 for masked scores, so the poison is finite, never NaN."""
    import torch
    s = torch.randint(0, 2, shape, generator=gen, device=device).float() * 2 - 1
    f = 1 + (torch.rand(shape, generator=gen, device=device) - 0.5) / 4
    return (s * f * mag).to(torch.bfloat16)


class _Pages:
    """A paged K/V pool [n_pages][nkv][64][128] full of poison, with a shuffled block table per sequence."""

    def __init__(self, nkv, horizons, seed, spare=3):
        import torch
        self.gen = torch.Generator(device="cuda").manual_seed(seed)
        self.bt_stride = max((h + 63) // 64 for h in horizons) + 1
        self.n_pages = len(horizons) * self.bt_stride + spare
        shape = (self.n_pages, nkv, 64, 128)
        self.kp, self.vp = _poison(shape, POISON_K, self.gen), _poison(shape, POISON_V, self.gen)
        perm = torch.randperm(self.n_pages, generator=torch.Generator().manual_seed(seed))[: len(horizons) * self.bt_stride]
        self.bt = perm.view(len(horizons), self.bt_stride).to(torch.int32).cuda()

    def write(self, i, pos0, k, v):
        """K/V of sequence i for positions [pos0, pos0 + len(k))."""
        import torch
        pos = torch.arange(pos0, pos0 + k.shape[0], device="cuda")
        pages = self.bt[i][(pos // 64).long()].long()
        self.kp[pages, :, pos % 64] = k
        self.vp[pages, :, pos % 64] = v


def _qkv_rows(n, nh, nkv, scale, gen):
    import torch
    W = (nh + 2 * nkv) * 128
    x = torch.randn(n, W, generator=gen, device="cuda")
    x[:, : nh * 128] *= scale
    return x.to(torch.bfloat16)


# prefill scenarios: each call is a list of (sequence, first position, new rows); a sequence's context is whatever earlier
# calls (or the scenario's pre-filled context) appended.  "chunked": one sequence's prompt over two calls.
PREFILL_SCENARIOS = {
    "ragged": [[(0, 0, 150), (1, 70, 37), (2, 3, 128), (3, 200, 129), (4, 0, 1)]],
    "long": [[(0, 3900, 196)]],
    "chunked": [[(0, 0, 300), (1, 0, 77)], [(0, 300, 400)]],
}


ATTN_GQA = [(8, 8), (8, 2), (8, 1), (32, 8), (64, 8)]
ATTN_SCALES = [1, 4, 16]     # q x scale: scores from nearly flat (N(0, 1)) to nearly one-hot (N(0, 256))


def _attn_check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                   # a NaN output is over any bound
    assert not bool(bad.any()), "%s: %d elements over the bound, first (row, head, d) %s: got %g want %g bound %g" % (
        what, int(bad.sum()), tuple(bad.nonzero()[0].tolist()), got[bad][0].item(), ref[bad][0].item(), bound[bad][0].item())
    return float((err / bound).max())


@pytest.mark.parametrize("scenario", sorted(PREFILL_SCENARIOS))
@pytest.mark.parametrize("scale", ATTN_SCALES)
@pytest.mark.parametrize("nh,nkv", ATTN_GQA)
@pytest.mark.parametrize("impl", PREFILL_IMPLS)
def test_prefill_attention_against_fp64(L, impl, nh, nkv, scale, scenario):
    """Poisoned pages (every slot past a sequence's horizon and every unused page holds K ~ +-30, V ~ +-1e3), tiles listed
    out of order and starting mid-page, a 4096-token horizon (32 KV blocks), a prompt prefilled over two calls."""
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    seed = nh * 1000 + nkv * 100 + scale + len(scenario)
    calls = PREFILL_SCENARIOS[scenario]
    horizon = {}
    for call in calls:
        for i, pos0, n in call:
            horizon[i] = max(horizon.get(i, 0), pos0 + n)
    seqs = sorted(horizon)
    pages = _Pages(nkv, [horizon[i] for i in seqs], seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    K = {i: torch.randn(horizon[i], nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for i in seqs}
    V = {i: torch.randn(horizon[i], nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for i in seqs}
    for i in seqs:                       # context cached before the first call
        first = min(pos0 for call in calls for j, pos0, _ in call if j == i)
        if first:
            pages.write(i, 0, K[i][:first], V[i][:first])
    tile = 128 if impl == "tc" else 64
    ratio = 0.0
    for ci, call in enumerate(calls):
        for i, pos0, n in call:          # the rows of this call append their K/V first (rope_append does in the engine)
            pages.write(i, pos0, K[i][pos0: pos0 + n], V[i][pos0: pos0 + n])
        T = sum(n for _, _, n in call)
        qkv = _qkv_rows(T, nh, nkv, scale, gen)
        tiles, row0 = [], 0
        for i, pos0, n in call:
            for j in range(0, n, tile):
                tiles.append([row0 + j, min(tile, n - j), pos0 + j, i])
            row0 += n
        order = torch.randperm(len(tiles), generator=torch.Generator().manual_seed(seed + ci)).tolist()
        tiles_t = torch.tensor([tiles[k] for k in order], dtype=torch.int32, device="cuda")
        out = _Out(T, nh * 128, torch.bfloat16, pad=0)      # the kernels write dense [T, nh * 128] rows
        if impl == "tc":
            ok(L.llmlb_op_prefill_attention_tc(p(qkv), T, p(pages.kp), p(pages.vp), pages.n_pages, p(pages.bt), pages.bt_stride,
                                               p(tiles_t), len(tiles), out.ptr(), nh, nkv, stream_ptr()))
        else:
            ok(L.llmlb_op_prefill_attention(p(qkv), p(pages.kp), p(pages.vp), p(pages.bt), pages.bt_stride, p(tiles_t), len(tiles),
                                            out.ptr(), nh, nkv, stream_ptr()))
        sync()
        assert out.untouched_outside(1) == 0
        row0 = 0
        for i, pos0, n in call:
            q = qkv[row0: row0 + n, : nh * 128].view(n, nh, 128)
            ref, bound = attention_ref(q, K[i][: pos0 + n], V[i][: pos0 + n], torch.arange(pos0, pos0 + n, device="cuda"), BF16_U)
            got = out.slot(0)[row0: row0 + n].view(n, nh, 128)
            ratio = max(ratio, _attn_check(got, ref, bound, "call %d sequence %d" % (ci, i)))
            row0 += n
    _report("prefill " + impl, ratio)


DECODE_LENS = [1, 63, 64, 65, 4097]      # tokens INCLUDING the new one: split boundaries mid-page and on page edges


@pytest.mark.parametrize("scale", ATTN_SCALES)
@pytest.mark.parametrize("nh,nkv", [(8, 2), (8, 1), (32, 8), (64, 8)])
@pytest.mark.parametrize("splits", DECODE_SPLITS)
def test_decode_attention_against_fp64(L, splits, nh, nkv, scale):
    """Decode attention (cluster of `splits` CTAs per sequence and head group; 1 = the tensor-core kernel) over poisoned
    pages, then a second launch with another batch composition sharing the same workspace.  The RoPE table is the
    identity (cos 1, sin 0), so the q and k the kernel uses are exactly the bf16 inputs."""
    import torch
    from gpu_util import ok, p, stream_ptr, sync
    seed = splits * 1000 + nh * 10 + nkv + scale
    lens = DECODE_LENS
    pages = _Pages(nkv, lens, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    Kc = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
    Vc = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
    for i, n in enumerate(lens):
        if n > 1:
            pages.write(i, 0, Kc[i], Vc[i])
    rope = torch.zeros(max(lens) + 1, 64, 2, dtype=torch.float32, device="cuda")
    rope[..., 0] = 1
    ws = torch.zeros(L.llmlb_op_decode_attention_ws(len(lens), nh, splits), dtype=torch.uint8, device="cuda")
    ratio = 0.0
    p_round = BF16_U if splits == 1 else 0.0       # only the tensor-core kernel rounds P to bf16
    for batch in ([0, 1, 2, 3, 4], [4, 2, 0]):     # two compositions through one workspace
        B = len(batch)
        qkv = _qkv_rows(B, nh, nkv, scale, gen)
        seq_lens = torch.tensor([lens[i] for i in batch], dtype=torch.int32, device="cuda")
        bt_rows = torch.tensor(batch, dtype=torch.int32, device="cuda")
        out = _Out(B, nh * 128, torch.bfloat16, pad=0)
        ok(L.llmlb_op_decode_attention(p(qkv), p(pages.kp), p(pages.vp), p(pages.bt), pages.bt_stride, p(bt_rows), p(seq_lens), B,
                                       out.ptr(), nh, nkv, p(rope), splits, len(lens), p(ws), stream_ptr()))
        sync()
        assert out.untouched_outside(1) == 0
        for b, i in enumerate(batch):
            n = lens[i]
            row = qkv[b]
            q = row[: nh * 128].view(1, nh, 128)
            kn = row[nh * 128:(nh + nkv) * 128].view(1, nkv, 128)
            vn = row[(nh + nkv) * 128:].view(1, nkv, 128)
            k, v = torch.cat([Kc[i], kn]), torch.cat([Vc[i], vn])
            ref, bound = attention_ref(q, k, v, torch.tensor([n - 1], device="cuda"), p_round)
            ratio = max(ratio, _attn_check(out.slot(0)[b].view(1, nh, 128), ref, bound, "batch %s sequence %d (len %d)" % (batch, i, n)))
            page = pages.bt[i, (n - 1) // 64]          # the new token's K / V were appended to its page slot
            assert torch.equal(pages.kp[page, :, (n - 1) % 64], kn[0]) and torch.equal(pages.vp[page, :, (n - 1) % 64], vn[0])
    _report("decode", ratio)
