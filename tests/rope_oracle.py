"""RoPE frequency scaling for the model oracle (test infrastructure): oracle/llama_ref.py's LlamaRef with
cfg["rope_scaling"] = {"rope_type": "llama3", "factor", "low_freq_factor", "high_freq_factor",
"original_max_position_embeddings"} or {"rope_type": "linear", "factor"}.  Each inv_freq[j] is divided by a fixed
factor f[j] (rope_freq_factors; llama.cpp's rope_freqs), computed in fp64 — equal in real arithmetic to
transformers' _compute_llama3_parameters / _compute_linear_scaling_rope_parameters.  Without rope_scaling the
model is exactly LlamaRef.  Pinned to transformers on tests/golden/llama_rope_scaling_golden.npz
(tests/test_rope_scaling_cpu.py).

forward_tail evaluates only the last positions of a one-layer model (K/V for every position, queries, attention
and MLP only where checked), so that a 120K-token parity check stays cheap on a CPU."""
import math

import numpy as np
import torch

from oracle.llama_ref import LlamaRef, _bf16_round


def rope_freq_factors(rope_scaling, rope_theta, head_dim=128):
    """Per-frequency RoPE divisors f[j] (float64, head_dim/2 of them) for a llama3 or linear `rope_scaling`
    dict; None for no scaling.  Any other type raises ValueError."""
    if not rope_scaling:
        return None
    kind = rope_scaling.get("rope_type", rope_scaling.get("type"))
    n = head_dim // 2
    if kind in (None, "default", "none"):
        return None
    if kind == "linear":
        return np.full(n, float(rope_scaling["factor"]), dtype=np.float64)
    if kind != "llama3":
        raise ValueError("unsupported RoPE scaling type %r" % (kind,))
    factor = float(rope_scaling["factor"])
    low, high = float(rope_scaling["low_freq_factor"]), float(rope_scaling["high_freq_factor"])
    old = float(rope_scaling["original_max_position_embeddings"])
    inv = 1.0 / (float(rope_theta) ** (np.arange(0, head_dim, 2, dtype=np.float64) / head_dim))
    wavelen = 2 * math.pi / inv
    f = np.ones(n, dtype=np.float64)
    lo = wavelen > old / low                      # low frequencies: divided by `factor`
    mid = ~lo & ~(wavelen < old / high)           # medium: interpolated between 1 and `factor`
    f[lo] = factor
    smooth = (old / wavelen[mid] - low) / (high - low)
    f[mid] = 1.0 / ((1 - smooth) / factor + smooth)
    return f



class ScaledLlamaRef(LlamaRef):
    def __init__(self, cfg, state_dict, **kw):
        super().__init__(cfg, state_dict, **kw)
        f = rope_freq_factors(cfg.get("rope_scaling"), cfg["rope_theta"], cfg["head_dim"])
        if f is not None:
            self.inv_freq = self.inv_freq / torch.from_numpy(f)

    @torch.no_grad()
    def forward_tail(self, ids, n_last):
        """One-layer model only: feeds `ids` from position 0 and returns the logits of the last `n_last`
        positions.  K and V are computed for every position (and cached, so forward() continues the
        sequence), but queries, attention and the MLP only for the last n_last rows: a 100K-token
        context costs a few projections instead of a T x T attention."""
        c = self.cfg
        if c["n_layers"] != 1:
            raise ValueError("forward_tail needs a one-layer model")
        if getattr(self.w["model.embed_tokens.weight"], "dtype", None) in ("bf16_bits", "q4_0"):
            raise ValueError("forward_tail needs torch weights")
        nh, nkv, hd = c["n_heads"], c["n_kv_heads"], c["head_dim"]
        self.reset()
        ids = torch.as_tensor(ids, dtype=torch.long)
        T = ids.numel()
        n_last = min(int(n_last), T)
        p = "model.layers.0."
        x_all = self.w["model.embed_tokens.weight"][ids].to(torch.float32)
        K = torch.empty(T, nkv, hd)
        V = torch.empty(T, nkv, hd)
        for s0 in range(0, T, 8192):   # bounded working set
            y = self._norm(x_all[s0:s0 + 8192], self.w[p + "input_layernorm.weight"])
            k = self._mm(y, self.w[p + "self_attn.k_proj.weight"]).view(-1, nkv, hd)
            v = self._mm(y, self.w[p + "self_attn.v_proj.weight"]).view(-1, nkv, hd)
            if self.emulate:
                k, v = _bf16_round(k), _bf16_round(v)
            k = self._rope(k, torch.arange(s0, s0 + k.shape[0]))
            K[s0:s0 + k.shape[0]] = _bf16_round(k) if self.emulate else k
            V[s0:s0 + v.shape[0]] = v
        self.k_cache[0], self.v_cache[0] = K, V
        positions = torch.arange(T - n_last, T)
        x = x_all[T - n_last:]
        y = self._norm(x, self.w[p + "input_layernorm.weight"])
        q = self._mm(y, self.w[p + "self_attn.q_proj.weight"]).view(n_last, nh, hd)
        if self.emulate:
            q = _bf16_round(q)
        q = self._rope(q, positions)
        if self.emulate:
            q = _bf16_round(q)
        g = nh // nkv
        qg = q.view(n_last, nkv, g, hd)
        scores = torch.einsum("tkgd,skd->kgts", qg, K) / math.sqrt(hd)
        mask = torch.arange(T)[None, :] > positions[:, None]
        scores = scores.masked_fill(mask[None, None], float("-inf"))
        pr = torch.softmax(scores, dim=-1)
        a = torch.einsum("kgts,skd->tkgd", pr, V).reshape(n_last, nh * hd)
        if self.emulate:
            a = _bf16_round(a)
        x = x + self._mm(a, self.w[p + "self_attn.o_proj.weight"])
        y = self._norm(x, self.w[p + "post_attention_layernorm.weight"])
        hmid = torch.nn.functional.silu(self._mm(y, self.w[p + "mlp.gate_proj.weight"])) * self._mm(y, self.w[p + "mlp.up_proj.weight"])
        if self.emulate:
            hmid = _bf16_round(hmid)
        x = x + self._mm(hmid, self.w[p + "mlp.down_proj.weight"])
        self.pos = T
        y = self._norm(x, self.w["model.norm.weight"])
        return self._mm(y, self.w["lm_head.weight"])
