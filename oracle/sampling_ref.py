"""Oracle restatement of the sampler definition in llmlb_b200/csrc/sampling.cu (test
infrastructure, not product).  The reference forwards `temperature`/`top_p`/`top_k` untouched to
its endpoints (llmlb/src/api/openai.rs:761-1005 passes the payload through; benchmark payload at
llmlb/src/api/benchmarks.rs:484-522), so the semantics restated here are the usual
OpenAI/llama.cpp ones: temperature scaling, top-k, then nucleus over the kept set, then an
inverse-CDF draw in vocabulary order with a counter RNG."""
import numpy as np

from .synth import _mix64


def uniform(seed, step):
    with np.errstate(over="ignore"):
        h = _mix64(_mix64(np.uint64(seed)) + np.uint64(step))
    return np.float32(np.uint32(h >> np.uint64(40))) * np.float32(1.0 / 16777216.0)


def kept_mask(logits, temperature, top_k, top_p):
    lg = logits.astype(np.float32)
    d = lg - lg.max()
    with np.errstate(over="ignore", invalid="ignore"):
        inv_t = np.float32(1.0) / np.float32(temperature)      # inf below T ~ 3e-39: the max still maps to 0
        z = np.where(d < 0, d * inv_t, np.float32(0)).astype(np.float32)
    e = np.exp(z).astype(np.float32)
    keep = np.ones_like(e, dtype=bool)
    if 0 < top_k < e.size:
        kth = np.sort(e)[::-1][top_k - 1]
        keep &= e >= kth
    if top_p < 1.0:                          # top_p <= 0: target 0, the maximum(s) alone
        ek = np.where(keep, e, 0).astype(np.float64)
        order = np.argsort(-ek, kind="stable")
        cs = np.cumsum(ek[order])
        target = np.float64(np.float32(top_p) * np.float32(ek.sum()))
        idx = int(np.searchsorted(cs, target, side="left"))
        idx = min(idx, e.size - 1)
        v = ek[order][idx]
        keep &= e >= np.float32(v)
    return e, keep


def sample(logits, temperature, top_k, top_p, seed, step):
    """Returns (token, margin): margin = relative distance of the draw from the nearest CDF
    edge; tiny margins mark draws where fp32 summation order may legitimately flip the answer."""
    if not temperature > 0:
        return int(np.argmax(logits)), 1.0
    e, keep = kept_mask(logits, temperature, top_k, top_p)
    ek = np.where(keep, e, 0).astype(np.float64)
    cs = np.cumsum(ek)
    total = cs[-1]
    target = np.float64(uniform(seed, step)) * total
    tok = int(np.searchsorted(cs, target, side="right"))
    tok = min(tok, e.size - 1)
    while not keep[tok] and tok + 1 < e.size:
        tok += 1
    lo = cs[tok] - ek[tok]
    margin = min(target - lo, cs[tok] - target) / total
    return tok, float(margin)
