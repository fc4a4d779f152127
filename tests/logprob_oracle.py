"""Token log-probabilities for the tests (test infrastructure, not product): the definition at llmlb_token_logprobs in
include/llmlb_b200.h in float64, the top-n selection (descending z, ties by ascending id), and a checker whose bound is
derived from the kernel's arithmetic (llmlb_b200/csrc/logprob.cu):

  d_j  = fl32(z_j - m)                 the checker forms the same float32 difference, so its rounding is known exactly
  s    = fl32(sum_j expf(d_j))         expf within 2 ulp (CUDA's documented bound): relative 2^-22 per term; the fp64
                                       sum adds at most (vocab + 32) 2^-53 relative and the rounding to fp32 2^-24
  ls   = logf(s)                       within 1 ulp of log(s)
  lp_j = fl32(d_j - ls)                half an ulp of the result

so |lp_j - lp64_j| <= |d_j - (z_j - m)| + |log S_d - log S| + 1.01 (5 2^-24 + (V + 32) 2^-53) + ulp(log s) + ulp(lp_j) / 2,
where S_d = sum exp(d_j) and S = sum exp(z_j - m) are evaluated in float64 (both known to the checker).  A -inf logit
must give exactly -inf.  The selection involves no arithmetic, so its ids must match exactly.

kernel_model() restates the kernel in numpy (float32 operations, float64 sum, correctly rounded exp and log); its knobs
plant the defects the checker must reject."""
import numpy as np

MAX_TOP = 20
EPS = 2.0 ** -24
# the vocabularies the GPU op test (tests/test_logprobs_gpu.py) runs: those the engine samples at Llama-3-8B / 70B, LLAMA_MID
# and LLAMA_TINY, one that is not a multiple of 32, and one below 20
VOCABS = (128256, 4096, 2048, 32003, 7)


def lm_row(V, rs):
    """Logits shaped like a language model's: a normal bulk and a few tokens well above it."""
    z = (rs.randn(V) * 2.0).astype(np.float32)
    k = min(V, 8)
    z[rs.choice(V, k, replace=False)] += rs.uniform(6, 12, k).astype(np.float32)
    return z


def log_softmax64(z):
    """float64 log_softmax of a float32 row; -inf entries stay -inf."""
    z = np.asarray(z, dtype=np.float32).astype(np.float64)
    m = z.max()
    with np.errstate(invalid="ignore", over="ignore"):
        return (z - m) - np.log(np.exp(z - m).sum())


def top_ids(z, n):
    """The min(n, 20, vocab) largest z, by descending z with ties by ascending id (-0 and +0 are a tie)."""
    z = np.asarray(z, dtype=np.float32).astype(np.float64)
    order = np.lexsort((np.arange(z.size), -z))
    return order[:min(int(n), MAX_TOP, z.size)]


def _ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


def bound(z):
    """(lp64, per-element bound) for row z, as derived in the module docstring."""
    z32 = np.asarray(z, dtype=np.float32)
    z64 = z32.astype(np.float64)
    m32 = z32.max()
    with np.errstate(invalid="ignore", over="ignore"):
        d32 = (z32 - m32).astype(np.float64)                 # the kernel's float32 differences, exactly
        d64 = z64 - np.float64(m32)
        S_d, S = np.exp(d32).sum(), np.exp(d64).sum()
        lp64 = d64 - np.log(S)
        ls = np.log(S_d)
        b = (np.abs(d32 - d64) + abs(np.log(S_d) - np.log(S)) + 1.01 * (5 * EPS + (z32.size + 32) * 2.0 ** -53)
             + 1.01 * _ulp32(ls) + 0.5 * 1.01 * _ulp32(d32 - ls))
    return lp64, b


def check(z, n, token, rec):
    """Checks one record {logprob, n_top, ids, vals} of row z (requested n alternatives, sampled token).  Returns
    (ok, reason)."""
    lp64, b = bound(z)
    z32 = np.asarray(z, dtype=np.float32)
    want = top_ids(z32, n)
    n_top, ids, vals, lp = int(rec["n_top"]), np.asarray(rec["ids"]), np.asarray(rec["vals"], dtype=np.float32), np.float32(rec["logprob"])
    if n_top != len(want):
        return False, "n_top %d, want %d" % (n_top, len(want))
    if not np.array_equal(ids[:n_top], want):
        return False, "ids %s, want %s" % (ids[:n_top].tolist(), want.tolist())

    def ok_val(v, j):
        if np.isneginf(z32[j]):
            return bool(np.isneginf(v))
        return bool(np.isfinite(v) and abs(float(v) - lp64[j]) <= b[j])
    for k in range(n_top):
        if not ok_val(vals[k], ids[k]):
            return False, "top %d (id %d): %r vs %r, bound %g" % (k, ids[k], float(vals[k]), lp64[ids[k]], b[ids[k]])
    if not ok_val(lp, token):
        return False, "token %d: %r vs %r, bound %g" % (token, float(lp), lp64[token], b[token])
    hit = np.nonzero(ids[:n_top] == token)[0]
    if hit.size and np.float32(vals[hit[0]]).view(np.uint32) != lp.view(np.uint32):
        return False, "the sampled token's value differs from its list entry"
    return True, ""


def kernel_model(z, n, token, expf_ulps=None, drop_last_span=False, ties_high=False, temperature=None):
    """The kernel in numpy: float32 differences, correctly rounded exp and log, float64 sum.  Knobs: expf_ulps(d) -> the
    error, in ulp, subtracted from every term (__expf's documented bound is 2 + floor(1.173 |d|)); drop_last_span leaves
    the last warp span (32 ceil(V / 1024) elements) out of the sum; ties_high breaks ties by the highest id; temperature
    takes logprobs of z / T."""
    z32 = np.asarray(z, dtype=np.float32)
    if temperature is not None:
        z32 = (z32 * np.float32(1.0 / temperature)).astype(np.float32)
    V = z32.size
    m = z32.max()
    with np.errstate(invalid="ignore", over="ignore"):
        d = (z32 - m).astype(np.float32)
        e = np.exp(d.astype(np.float64)).astype(np.float32)
        if expf_ulps is not None:
            e = (e - np.float32(expf_ulps(d)) * np.spacing(e)).astype(np.float32)
        if drop_last_span:
            e[V - min(V, 32 * ((V + 1023) // 1024)):] = 0
        s = np.float32(e.astype(np.float64).sum())
        ls = np.float32(np.log(np.float64(s)))
        lp = (d - ls).astype(np.float32)
    if ties_high:
        order = np.lexsort((-np.arange(V), -z32.astype(np.float64)))
    else:
        order = np.lexsort((np.arange(V), -z32.astype(np.float64)))
    ids = order[:min(int(n), MAX_TOP, V)]
    return dict(logprob=lp[token], n_top=ids.size, ids=ids, vals=lp[ids])


def expf_documented_ulps(d):
    """__expf's documented maximum error, in ulp (CUDA C Programming Guide, intrinsic functions)."""
    return 2 + np.floor(1.173 * np.abs(d.astype(np.float64)))
