"""Frequency / presence penalties and logit bias for the sampler oracle (test infrastructure, not product): the
definition in OpenAI's API reference (text-generation guide, "frequency and presence penalties"), restated in float32
in the operation order of penalize_kernel (llmlb_b200/csrc/penalty.cu).  Its output feeds oracle.sampling_ref.sample
unchanged, as the kernel's output feeds sample_kernel."""
import numpy as np


def penalize(logits, counts, frequency_penalty, presence_penalty, bias):
    """z[j] = (logit[j] - (c[j] * frequency_penalty + (c[j] > 0 ? presence_penalty : 0))) + bias[j], one float32 rounding
    per operation and no fused multiply-add.  counts: int [vocab], times each token was generated so far; bias:
    {token id: value}, added to those ids only.  Both penalties 0 and no bias return the logits unchanged."""
    z = np.array(logits, dtype=np.float32, copy=True)
    f, p = np.float32(frequency_penalty), np.float32(presence_penalty)
    if f != 0 or p != 0:
        c = np.asarray(counts)
        pen = (c.astype(np.float32) * f).astype(np.float32) + np.where(c > 0, p, np.float32(0)).astype(np.float32)
        z = (z - pen.astype(np.float32)).astype(np.float32)
    if bias:
        ids = np.array(list(bias.keys()), dtype=np.int64)
        z[ids] = (z[ids] + np.array(list(bias.values()), dtype=np.float32)).astype(np.float32)
    return z
