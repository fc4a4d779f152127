"""-m gpu: the sampling kernel (sample_kernel, llmlb_op_sample) draw by draw against an fp64 reference of its definition, at
every vocabulary the engine launches it with, and at the draws where its fp32 arithmetic can go wrong.

  * reference (fp64, independent of the kernel's arithmetic): p_i = exp((l_i - l_max) / T); top-k keeps the k largest with
    ties at the threshold kept; top-p (top_p < 1) keeps p_i >= v, v the value at which the descending kept mass first
    reaches top_p x the kept mass (top_p = 0: the maximum(s) alone); the draw is the first index in vocab order whose
    cumulative kept mass exceeds u x the kept mass, u = (mix64(mix64(seed) + step) >> 40) / 2^24 (oracle.sampling_ref).
  * checker, every row and draw: the token is kept, can have e > 0 in fp32 (p (1 + eta) >= 2^-150: __expf returns
    denormals down to 2^-149), and its CDF interval contains u x M widened by delta.  delta charges (a) each kept e_j its
    error p_j eta_j + 2^-149, eta_j = 2^-23 (3 + 3 |x_j|): __expf's 2 + floor(1.173 |x|) ulp plus three fp32 roundings in
    x = (l - l_max) / T, which move e by |x| 2^-24 each; and (b) fp32 summation, gamma(span / 32 + 48) M: the lane sums
    over a warp span (span / 32 rows), the 5-level butterfly, the 32-warp chain, the 5-level row scan, the run carried over
    span / 32 rows and the product u x total.  Tokens within those errors of a top-k or top-p threshold are ambiguous:
    either side is accepted, and the number of draws that needed that is counted and asserted small.
  * directed draws: (seed, step) pairs found on the CPU whose u lands at the lowest and highest 64 values, at the CDF
    position of warp-span ends and of 32-element row boundaries, and inside the gaps between the kernel's two fp32 orders
    (lane sums + butterfly decide which warp holds the target; a row scan carried across rows searches inside it).  The
    gaps are located by emulating both orders in numpy (FP32Draw), on crafted rows that widen them to ~10^-6 of the mass
    and put them at a mid-CDF warp and at the last warp, where vocab - 1 is banned.
  * greedy (T <= 0 or NaN), exact: lowest index on ties, ties across warps, -inf entries, all-equal rows.
  * chi^2 at V = 128256 against the textbook distribution with the mass spread over all 32 warp spans, so that the run
    carried across rows is tested against something that does not restate the kernel.
  * determinism and row independence: a second launch is bit-identical; a row at another index or in another batch draws
    the same token (tensor-parallel ranks sample the same logits independently and must agree).

VOCABS, the case builders and the checker are plain code: tests/test_kernel_coverage_cpu.py runs the vocabularies over the
fake CUDA runtime against the engine's launch plans, and applies the checker on the CPU to models of the kernel that are
wrong in the ways a sampler goes wrong.
"""
import math

import numpy as np
import pytest

from oracle.sampling_ref import uniform
from oracle.synth import _mix64

# ---------------------------------------------------------------------------------------------------------------- cases --
VOCAB_LLAMA3 = 128256          # Llama-3-8B and Llama-3-70B
VOCAB_MID = 4096               # LLAMA_MID
VOCAB_TINY = 2048              # LLAMA_TINY
VOCAB_ODD = 32003              # not a multiple of 32: the i < vocab tails of the last row and the last warp
VOCABS = (VOCAB_LLAMA3, VOCAB_MID, VOCAB_TINY, VOCAB_ODD)
TIED_K = 3                     # rows of kind "tiedk": values 6, 5, then 4 three times (ranks 3..5 tie)
TOP_PS = (0.0, 1e-6, 0.5, 0.9, 1.0 - 2.0 ** -24, 1.0)
TEMPS = (1.4e-45, 1e-38, 1e-30, 1e-6, 0.05, 0.2, 0.7, 1.0, 3.0, 1e4)
TINY_TEMPS = (1.4e-45, 1e-38, 1e-30)        # every surviving token is an arg-max
ROW_KINDS = ("lm", "flat", "onehot_first", "onehot_last", "last_warp", "banned", "tiedk")
BAN = -100.0                   # logit_bias -100, in rows whose max logit is >= 10: exp(-110) is below fp32's least denormal
LIVE = 10.0                    # offset of the live logits in rows with banned tokens
SEED = 0x5EED
U = 2.0 ** -24
DENORM = 2.0 ** -148            # fp32 denormals are spaced 2^-149: values this close may round together


def top_ks(V):
    return (0, 1, 2, TIED_K, V - 1, V, V + 5)


def param_sets(V):
    """(T, top_k, top_p): one axis at a time around (1, 0, 1), and a few combinations."""
    out = [(1.0, k, 1.0) for k in top_ks(V)] + [(1.0, 0, p) for p in TOP_PS] + [(t, 0, 1.0) for t in TEMPS]
    return out + [(0.7, 40, 0.9), (0.2, 0, 0.95), (1.3, 1000, 0.5), (0.05, TIED_K, 0.0), (3.0, V - 1, 1.0 - 2.0 ** -24)]


def span_of(V):
    """Elements per warp span in the draw: 32 warps over ceil(V / 1024) rows of 32 each."""
    return ((V + 1023) // 1024) * 32


def make_row(kind, V, seed):
    rs = np.random.RandomState(seed)
    if kind == "lm":
        return (rs.randn(V) * 2.5).astype(np.float32)
    if kind == "flat":
        return np.full(V, 1.5, np.float32)
    if kind in ("onehot_first", "onehot_last"):
        l = (rs.randn(V) * 0.5 - 30).astype(np.float32)
        l[0 if kind == "onehot_first" else V - 1] = 0.0
        return l
    if kind == "last_warp":
        l = np.full(V, BAN, np.float32)
        w0 = 31 * span_of(V)
        l[w0:] = rs.randn(V - w0) * 2 + LIVE
        return l
    if kind == "banned":
        l = (rs.randn(V) * 2.5 + LIVE).astype(np.float32)
        l[rs.rand(V) < 0.1] = BAN
        l[[0, V - 1]] = BAN
        return l
    if kind == "tiedk":
        l = (rs.randn(V) * 0.5 - 10).astype(np.float32)
        pos = rs.permutation(V)[:5]
        l[pos] = (6.0, 5.0, 4.0, 4.0, 4.0)
        return l
    raise ValueError(kind)


def crafted_gap_row(V, warp):
    """A row whose warp `warp` holds e = 1 at its first element and ~2^-30 everywhere else in its span: the row scan
    absorbs the small terms into the 1 while the lane sums keep them, so its warp total exceeds what the search can reach by
    ~span x 2^-30.  Two tokens with e ~ 1/4 sit in other warps (mass before and after); everything else is banned,
    vocab - 1 included."""
    sp = span_of(V)
    l = np.full(V, BAN, np.float32)
    w0, w1 = warp * sp, min(V, (warp + 1) * sp)
    l[w0:w1] = np.float32(LIVE - 30 * math.log(2))
    l[w0] = LIVE
    for w in ((3, 28) if warp not in (3, 28) else (5, 20)):
        l[w * sp + 7] = np.float32(LIVE - 2 * math.log(2))
    l[V - 1] = BAN
    return l


# ------------------------------------------------------------------------------------------------------- RNG counters --
N_STEPS = 1 << 24
_STEPS = {}


def step_table():
    """(values, steps): the distinct u x 2^24 that steps 0..2^24-1 give under SEED, ascending, and a step for each."""
    if not _STEPS:
        with np.errstate(over="ignore"):
            h = _mix64(_mix64(np.uint64(SEED)) + np.arange(N_STEPS, dtype=np.uint64))
        ui = (h >> np.uint64(40)).astype(np.int64)
        _STEPS[0] = np.unique(ui, return_index=True)
    return _STEPS[0]


def u_of(step):
    return np.float64(uniform(SEED, np.asarray(step, dtype=np.uint64)))


def steps_near(ui, below):
    """A step whose u x 2^24 is the nearest available value <= ui (below) or >= ui."""
    vals, steps = step_table()
    ui = np.clip(np.asarray(ui, np.int64), 0, 2 ** 24 - 1)
    j = np.searchsorted(vals, ui, side="right") - 1 if below else np.searchsorted(vals, ui, side="left")
    return steps[np.clip(j, 0, len(vals) - 1)]


def steps_in(lo, hi, n):
    """Up to n steps whose u x 2^24 lies in [lo, hi), spread over the range."""
    vals, steps = step_table()
    a, b = np.searchsorted(vals, lo), np.searchsorted(vals, hi)
    idx = np.unique(np.linspace(a, b - 1, n).round().astype(np.int64)) if b > a else np.zeros(0, np.int64)
    return steps[idx]


def extreme_steps(n=2):
    return np.concatenate([steps_in(0, 64, n), steps_in(2 ** 24 - 64, 2 ** 24, n)])


# ------------------------------------------------------------------------------------------------ fp64 reference + check --
def gamma(n):
    return n * U / (1 - n * U)


def eta_of(x):
    """Relative error bound of the kernel's e = __expf(fl(fl(l - l_max) * fl(1 / T))) at exponent x <= 0."""
    return 2.0 ** -23 * (3 + 3 * np.minimum(np.abs(x), 300.0))


class Ref:
    """The fp64 reference of one row's sampling, with the sets the kernel surely keeps (sure) and may keep either way
    (amb), and the acceptance test for a drawn token."""

    def __init__(self, logits, T, k, p):
        l = logits.astype(np.float64)
        V = l.size
        self.V, self.T = V, float(T)
        lmax = l.max()
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            x = np.where(l == lmax, 0.0, (l - lmax) / np.float64(np.float32(T)))
        pr = np.exp(x)
        eta = eta_of(x)
        self.pr, self.eta, self.is_max = pr, eta, l == lmax
        sure, amb = np.ones(V, bool), np.zeros(V, bool)
        if 0 < k < V:
            vk = np.partition(pr, V - k)[V - k]                  # the k-th largest
            ek = eta_of(math.log(vk)) if vk > 0 else eta_of(300.0)
            band = np.abs(pr - vk) <= 2.01 * ek * vk + DENORM
            if np.unique(pr[band]).size <= 1:                    # only the k-th value's own tie group: ranks are stable
                sure = pr >= vk
            else:
                sure, amb = pr > vk * (1 + 2.01 * ek) + DENORM, band
        if p < 1.0:
            k_lo, k_hi = sure, sure | amb
            m_hi = pr[k_hi].sum()
            m_lo = pr[k_lo].sum()
            # the kernel's kept-mass sums: its e errors, 2^-40 fixed point per token, the top-k-ambiguous mass
            err = (pr * eta)[k_hi].sum() + V * 2.0 ** -40 + pr[amb].sum() + 1e-15 * m_hi
            w = 2.01 * eta
            s_lo = self._mass_above(pr[k_lo], pr * (1 + w) + DENORM)
            s_hi = self._mass_above(pr[k_hi], pr * (1 - w) - DENORM) - self._mass_equal(pr[k_hi], pr)
            t_lo, t_hi = p * (m_lo - err), p * (m_hi + err)
            keep = self.is_max | (s_hi + err < t_lo)
            drop = ~self.is_max & (s_lo - err >= t_hi)
            sure, amb = k_lo & keep, k_hi & ~(k_lo & keep) & ~drop
        self.sure, self.amb = sure, amb
        self.pos = pr * (1 + eta) >= 2.0 ** -150
        self.c_lo = np.cumsum(np.where(sure, pr, 0.0))
        self.c_hi = np.cumsum(np.where(sure | amb, pr, 0.0))
        self.m_lo, self.m_hi = self.c_lo[-1], self.c_hi[-1]
        self.delta = (pr * eta + 2.0 ** -149)[sure | amb].sum() + gamma(span_of(V) // 32 + 48) * self.m_hi

    @staticmethod
    def _mass_above(vals, thr):
        a = np.sort(vals)
        suffix = np.concatenate([np.cumsum(a[::-1])[::-1], [0.0]])
        return suffix[np.searchsorted(a, thr, side="right")]

    @staticmethod
    def _mass_equal(vals, v):
        a = np.sort(vals)
        return (np.searchsorted(a, v, side="right") - np.searchsorted(a, v, side="left")) * v

    def check(self, t, u):
        """(ok, ambiguous, reason) for token t drawn with uniform u."""
        if not 0 <= t < self.V:
            return False, False, "token out of range"
        if not (self.sure[t] or self.amb[t]):
            return False, False, "a token the filters drop"
        if not self.pos[t]:
            return False, False, "a token with zero mass"
        d = self.delta

        def inside(c, m, prev):
            return prev - d <= u * m <= c[t] + d

        ok_lo = self.sure[t] and inside(self.c_lo, self.m_lo, self.c_lo[t] - self.pr[t])
        ok_hi = inside(self.c_hi, self.m_hi, self.c_hi[t] - self.pr[t])
        prev_lo = self.c_lo[t] - (self.pr[t] if self.sure[t] else 0.0)
        ok_mix = prev_lo - d <= u * self.m_hi and u * self.m_lo <= self.c_hi[t] + d
        ok = ok_lo or ok_hi or ok_mix
        return ok, bool(self.amb[t]) or not (ok_lo and ok_hi), "" if ok else "u x M outside the token's CDF interval"

    def directed_steps(self, rs, n_rows=8):
        """Steps whose u lands at the CDF position of every warp-span end and of n_rows random 32-element row
        boundaries (the value at or just below, and at or just above), and at the extremes."""
        sp = span_of(self.V)
        ends = [min(self.V, (w + 1) * sp) - 1 for w in range(32) if w * sp < self.V]
        rows = rs.choice(np.arange(31, self.V, 32), min(n_rows, self.V // 32), replace=False)
        pos = self.c_lo[np.array(ends + list(rows))] / self.m_lo * 2 ** 24
        pos = pos[pos < 2 ** 24 - 1]
        ui = np.floor(pos).astype(np.int64)
        return np.concatenate([steps_near(ui, True), steps_near(ui + 1, False), extreme_steps()])


# ----------------------------------------------------------------------------------------- the kernel's fp32 orders --
def kernel_e(logits, T):
    """A numpy stand-in for the kernel's e: fp32 (l - l_max) x (1 / T), np.exp for __expf (denormals kept, as the
    kernel's are)."""
    lg = logits.astype(np.float32)
    d = lg - lg.max()
    with np.errstate(over="ignore", divide="ignore", invalid="ignore", under="ignore"):
        inv_t = np.float32(1.0) / np.float32(T)
        z = np.where(d < 0, d * inv_t, np.float32(0)).astype(np.float32)
        return np.exp(z).astype(np.float32)


def _f32(a):
    return np.asarray(a, dtype=np.float32)


class FP32Draw:
    """The kernel's draw over kept masses e (float32, 0 where dropped), operation for operation in fp32: per warp span,
    lane sums over its rows then the xor butterfly (wsum); the chain of warp totals (before, total); target = u x total;
    inside the warp that holds the target, a Hillis-Steele scan per 32-element row with `run` carried across rows, and the
    first e > 0 lane with run + inc > target."""

    def __init__(self, e, carry=True):
        V = e.size
        self.V, self.sp = V, span_of(V)
        R = self.sp // 32
        E = np.zeros(32 * self.sp, np.float32)
        E[:V] = e
        self.E = E = E.reshape(32, R, 32)
        lane = np.zeros((32, 32), np.float32)
        for r in range(R):
            lane = _f32(lane + E[:, r])
        for o in (16, 8, 4, 2, 1):
            lane = _f32(lane + lane[:, np.arange(32) ^ o])
        self.wsum = lane[:, 0]
        self.before = np.zeros(33, np.float32)
        for w in range(32):
            self.before[w + 1] = _f32(self.before[w] + self.wsum[w])
        inc = E.copy()
        for o in (1, 2, 4, 8, 16):
            t = inc.copy()
            inc[..., o:] = _f32(t[..., o:] + t[..., :-o])
        self.inc = inc
        run = np.zeros((32, R), np.float32)
        cur = self.before[:32].copy()
        for r in range(R):
            run[:, r] = cur
            if carry:
                cur = _f32(cur + inc[:, r, 31])
        self.run = run
        self.reach = np.where(E > 0, _f32(run[..., None] + inc), -np.inf).reshape(32, -1).max(1)

    def target(self, u):
        return _f32(_f32(u) * self.before[32])

    def draw(self, u, fallback=None):
        """The token, or fallback(warp) when the crossing warp's search finds none (warp None: no warp crosses)."""
        tg = self.target(u)
        ws = [w for w in range(32) if self.before[w] <= tg < self.before[w + 1]]
        if not ws:
            return fallback(None)
        w = ws[0]
        hit = (self.E[w] > 0) & (_f32(self.run[w][:, None] + self.inc[w]) > tg)
        if hit.any():
            return w * self.sp + int(np.argmax(hit.reshape(-1)))
        return fallback(w)

    def last_positive(self, w):
        nz = np.nonzero(self.E[w].reshape(-1) > 0)[0]
        return w * self.sp + int(nz[-1])

    def gap_u_ints(self, w):
        """The u x 2^24 values whose target falls in warp w's interval but beyond what its search reaches."""
        tot = float(self.before[32])
        lo, hi = float(self.reach[w]), float(self.before[w + 1])
        if not (lo < hi and self.wsum[w] > 0):
            return np.zeros(0, np.int64)
        cand = np.arange(max(0, int(lo / tot * 2 ** 24) - 4), min(2 ** 24, int(hi / tot * 2 ** 24) + 5))
        tg = _f32(_f32(cand * U) * self.before[32])
        return cand[(tg >= self.reach[w]) & (tg < self.before[w + 1]) & (tg >= self.before[w])]


def gap_steps(e, per_warp=4):
    """Steps whose u lands in a gap of some warp (the middle of each gap), by the fp32 emulation of the kernel's orders."""
    d = FP32Draw(e)
    vals, steps = step_table()
    out = []
    for w in range(32):
        ui = d.gap_u_ints(w)
        if ui.size >= 3:
            ui = ui[ui.size // 4: ui.size - ui.size // 4]      # away from the gap's edges
        ui = ui[np.isin(ui, vals)]
        if ui.size:
            sel = ui[np.linspace(0, ui.size - 1, min(per_warp, ui.size)).round().astype(np.int64)]
            out.append(steps[np.searchsorted(vals, sel)])
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def check_draws(ref, toks, steps, where=""):
    """Asserts every draw; returns the number that needed an ambiguous band."""
    n_amb = 0
    for t, s in zip(np.asarray(toks).tolist(), np.asarray(steps).tolist()):
        ok, amb, why = ref.check(t, u_of(s))
        # delta = sum_j p_j eta_j + gamma(span / 32 + 48) M (module docstring)
        assert ok, "%s step %d u=%.9f: token %d is %s (delta %.3g of M; sure %s amb %s p %.3g)" % (
            where, s, u_of(s), t, why, ref.delta / ref.m_hi, ref.sure[t] if 0 <= t < ref.V else None,
            ref.amb[t] if 0 <= t < ref.V else None, ref.pr[t] / ref.m_hi if 0 <= t < ref.V else 0)
        n_amb += amb
    return n_amb


def case_list(V):
    """[(kind, row seed, T, k, p)] of the draw tests at vocab V."""
    return [(kind, 100 + i, T, k, p) for i, kind in enumerate(ROW_KINDS) for T, k, p in param_sets(V)]


# ------------------------------------------------------------------------------------------------------------- GPU --
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(built_lib):
    from llmlb_b200 import ffi
    return ffi.lib()


def _sample(L, logits, T, k, p, steps, seed=SEED):
    """One llmlb_op_sample launch over rows logits [R, V] (torch, on the GPU) with per-row parameters; returns tokens."""
    import torch
    from gpu_util import dev, ok, p as ptr, stream_ptr, sync
    R, V = logits.shape
    d = lambda a, dt: torch.as_tensor(np.array(a), dtype=dt).reshape(R).to(dev())
    t, tp, tk = d(np.broadcast_to(T, R), torch.float32), d(np.broadcast_to(p, R), torch.float32), d(np.broadcast_to(k, R), torch.int32)
    sd = d(np.broadcast_to(seed, R).astype(np.int64), torch.int64)
    st = d(np.broadcast_to(steps, R).astype(np.int64), torch.int64)
    out = torch.full((R,), -7, dtype=torch.int32, device=dev())
    ok(L.llmlb_op_sample(ptr(logits), R, V, ptr(t), ptr(tp), ptr(tk), ptr(sd), ptr(st), ptr(out), stream_ptr()))
    sync()
    return out.cpu().numpy()


@pytest.mark.parametrize("V", VOCABS)
def test_sample_every_draw_against_fp64(L, V):
    """Every row kind x parameter set at vocab V, ~50 draws each: random, extreme u, and u at the CDF positions of every
    warp-span end and of random row boundaries."""
    import torch
    from gpu_util import dev
    cases = case_list(V)
    rows = {kind: make_row(kind, V, seed) for kind, seed, _, _, _ in cases}
    logits = torch.from_numpy(np.stack([rows[c[0]] for c in cases])).to(dev())
    rs = np.random.RandomState(V)
    refs, plans = [], []
    for kind, seed, T, k, p in cases:
        ref = Ref(rows[kind], T, k, p)
        refs.append(ref)
        plans.append(np.concatenate([ref.directed_steps(rs), rs.randint(0, N_STEPS, 8)]))
    n = max(len(s) for s in plans)
    plans = np.stack([np.resize(s, n) for s in plans])          # wrap shorter plans around
    T, K, P = (np.array([c[i] for c in cases]) for i in (2, 3, 4))
    toks = np.stack([_sample(L, logits, T, K, P, plans[:, j]) for j in range(n)], 1)
    n_amb = 0
    for i, (kind, _, t, k, p) in enumerate(cases):
        n_amb += check_draws(refs[i], toks[i], plans[i], "V %d %s T %g k %d p %r" % (V, kind, t, k, p))
        if t in TINY_TEMPS:
            assert refs[i].is_max[toks[i]].all(), (kind, t, toks[i])
    # ambiguous draws: a token within fp32 error of a top-k / top-p threshold, or a draw that only passes with it
    assert n_amb <= max(4, toks.size // 500), (n_amb, toks.size)


GAP_CASES = [(VOCAB_LLAMA3, "mid"), (VOCAB_LLAMA3, "last"), (VOCAB_ODD, "mid")]   # V = 32003's last warp has 259 elements


@pytest.mark.parametrize("V,where", GAP_CASES)
def test_sample_draws_inside_the_fp32_gaps(L, V, where):
    """u inside the gap between the crossing warp's total (lane sums + butterfly) and what its row scan reaches: the draw
    must still be a kept token with e > 0 inside that warp.  The kernel once fell back to vocab - 1 there (banned here)."""
    import torch
    from gpu_util import dev
    warp = 16 if where == "mid" else (V - 1) // span_of(V)
    row = crafted_gap_row(V, warp)
    e = kernel_e(row, 1.0)
    d = FP32Draw(e)
    gap = d.gap_u_ints(warp)
    assert gap.size >= 8, gap.size                     # the crafted row opens a gap of several u values
    steps = gap_steps(e, per_warp=16)
    assert steps.size >= 4
    lm = make_row("lm", V, 7)
    lm_steps = gap_steps(kernel_e(lm, 1.0))             # natural gaps of an LM-like row (by np.exp's e: most are real)
    toks = _sample(L, torch.from_numpy(np.stack([row] * steps.size)).to(dev()), 1.0, 0, 1.0, steps)
    ref = Ref(row, 1.0, 0, 1.0)
    check_draws(ref, toks, steps, "crafted %s gap" % where)
    sp = span_of(V)
    assert ((toks // sp) == warp).all(), toks
    if lm_steps.size:
        toks = _sample(L, torch.from_numpy(np.stack([lm] * lm_steps.size)).to(dev()), 1.0, 0, 1.0, lm_steps)
        check_draws(Ref(lm, 1.0, 0, 1.0), toks, lm_steps, "LM gap")


@pytest.mark.parametrize("V", VOCABS)
def test_sample_greedy_exact(L, V):
    """T <= 0 or NaN: the arg-max, lowest index on ties; ties in different warps with the later index in a lower warp
    (element i goes to thread i % 1024), -inf entries, an all-equal row and an all -inf row (token 0)."""
    import torch
    from gpu_util import dev
    rs = np.random.RandomState(3)
    rows = [(rs.randn(V) * 3).astype(np.float32) for _ in range(4)]
    r = rows[1]
    i1 = 261                                            # thread 261: warp 8
    i2 = 1024 * ((V - 1) // 1024) + 3                   # thread 3: warp 0, a later index
    r[[i1, i2]] = 50.0
    r = rows[2]
    r[rs.rand(V) < 0.3] = -np.inf
    r[V - 1] = 40.0
    r[V // 2] = 40.0
    rows[3][:] = -np.inf
    rows[3][V - 1] = -1e30
    rows.append(np.full(V, 0.25, np.float32))
    rows.append(np.full(V, -np.inf, np.float32))
    want = [int(np.argmax(x)) for x in rows]
    assert want[1] == i1 and want[2] == V // 2 and want[4] == 0 and want[5] == 0
    lg = torch.from_numpy(np.stack(rows)).to(dev())
    for T in (0.0, -1.0, float("nan")):
        got = _sample(L, lg, T, 5, 0.5, np.arange(len(rows)))
        assert got.tolist() == want, (T, got.tolist(), want)
    from gpu_util import ok, p as ptr, stream_ptr, sync
    out = torch.full((len(rows),), -7, dtype=torch.int32, device=dev())
    ok(L.llmlb_op_sample(ptr(lg), len(rows), V, None, None, None, None, None, ptr(out), stream_ptr()))   # no parameters: greedy
    sync()
    assert out.tolist() == want


def chi_square_row(V=VOCAB_LLAMA3, n_live=2000, seed=21):
    """n_live tokens with randn logits spread over the whole vocabulary (every warp span, many rows of each), the rest
    banned."""
    rs = np.random.RandomState(seed)
    l = np.full(V, BAN, np.float32)
    live = np.sort(rs.choice(V, n_live, replace=False))
    l[live] = rs.randn(n_live) * 0.8 + LIVE
    return l, live


@pytest.mark.parametrize("T,top_k", [(1.0, 0), (0.8, 1000)])
def test_sample_distribution_chi_square_128256(L, T, top_k):
    """~10^5 draws (2048 copies of one row, 50 step counters each) against softmax(l / T) over the top_k in fp64."""
    import torch
    from scipy import stats
    from gpu_util import dev
    V, R, N = VOCAB_LLAMA3, 2048, 50                    # logits 2048 x 128256 x 4 B = 1.05 GB
    l, live = chi_square_row()
    assert len({int(i) // span_of(V) for i in live}) == 32
    pr = np.exp((l.astype(np.float64) - l.max()) / T)
    keep = np.ones(V, bool)
    if top_k:
        srt = np.sort(pr)[::-1]
        assert srt[top_k - 1] > srt[top_k] * (1 + 1e-4)     # no token near the threshold
        keep = pr >= srt[top_k - 1]
    want = np.where(keep, pr, 0.0)
    want /= want.sum()
    logits = torch.from_numpy(l).to(dev()).repeat(R, 1).contiguous()
    counts = np.zeros(V)
    for j in range(N):
        toks = _sample(L, logits, T, top_k, 1.0, np.arange(R) + j * R, seed=77)
        counts += np.bincount(toks, minlength=V)
    del logits
    assert counts[~keep].sum() == 0 and counts[want == 0].sum() == 0
    idx = np.argsort(-want)
    exp, obs = want[idx] * R * N, counts[idx]
    cut = int(np.searchsorted(-exp, -5.0))
    if cut < len(exp):
        exp, obs = np.append(exp[:cut], exp[cut:].sum()), np.append(obs[:cut], obs[cut:].sum())
    nz = exp > 0
    chi2, pval = stats.chisquare(obs[nz], exp[nz])
    assert pval > 1e-4, (chi2, pval, int(nz.sum()))


def test_sample_is_deterministic_and_rows_are_independent(L):
    """The same launch twice is bit-identical; each row draws the same token at another index and in another batch."""
    import torch
    from gpu_util import dev
    V = VOCAB_LLAMA3
    cases = [c for c in case_list(V) if c[2] in (0.2, 0.7, 1.0)][:48]
    rows = np.stack([make_row(c[0], V, c[1]) for c in cases])
    T, K, P = (np.array([c[i] for c in cases]) for i in (2, 3, 4))
    steps = np.random.RandomState(5).randint(0, N_STEPS, len(cases))
    lg = torch.from_numpy(rows).to(dev())
    a = _sample(L, lg, T, K, P, steps)
    b = _sample(L, lg, T, K, P, steps)
    assert np.array_equal(a, b)
    perm = np.random.RandomState(6).permutation(len(cases))
    c = _sample(L, lg[torch.from_numpy(perm).to(dev())].contiguous(), T[perm], K[perm], P[perm], steps[perm])
    assert np.array_equal(c, a[perm])
    other = torch.from_numpy(make_row("lm", V, 999)).to(dev())[None].repeat(5, 1)
    big = torch.cat([other, lg[10:20], other]).contiguous()
    pad = lambda x, v: np.concatenate([[v] * 5, x[10:20], [v] * 5])
    d = _sample(L, big, pad(T, 1.0), pad(K, 0), pad(P, 1.0), pad(steps, 0))
    assert np.array_equal(d[5:15], a[10:20])
