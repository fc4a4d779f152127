"""RoPE frequency scaling pinned against Hugging Face transformers' LlamaForCausalLM (fp32, CPU, eager
attention) on the tiny geometry: Llama 3.1-style llama3 scaling (factor 8, low/high frequency factors
1 / 4, original context 8192) and linear scaling (factor 4).  The prompts are a few hundred tokens
long so that the scaled low and medium frequencies turn far enough to move the logits.  Writes
tests/golden/llama_rope_scaling_golden.npz; run in the build container:

    python tests/golden/make_llama_rope_scaling_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.synth import synth_state_dict  # noqa: E402

TINY = dict(hidden=512, n_layers=2, n_heads=8, n_kv_heads=2, head_dim=128, ffn=1024, vocab=2048,
            rope_theta=500000.0, rms_eps=1e-5)
SCALINGS = {
    "llama3": {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
               "original_max_position_embeddings": 8192},
    "linear": {"rope_type": "linear", "factor": 4.0},
}
PROMPT_LEN = 384


def main():
    from transformers import LlamaConfig, LlamaForCausalLM
    M = TINY
    out = {}
    sd = {k: torch.from_numpy(v.copy()) for k, v in synth_state_dict(M, seed=11).items()}
    for name, rs in SCALINGS.items():
        cfg = LlamaConfig(hidden_size=M["hidden"], num_hidden_layers=M["n_layers"], num_attention_heads=M["n_heads"],
                          num_key_value_heads=M["n_kv_heads"], head_dim=M["head_dim"], intermediate_size=M["ffn"],
                          vocab_size=M["vocab"], rope_theta=M["rope_theta"], rms_norm_eps=M["rms_eps"],
                          rope_scaling=dict(rs), max_position_embeddings=131072, tie_word_embeddings=False,
                          attention_bias=False, mlp_bias=False, hidden_act="silu")
        cfg._attn_implementation = "eager"
        assert cfg.rope_parameters["rope_type"] == rs["rope_type"]
        model = LlamaForCausalLM(cfg).to(torch.float32).eval()
        missing, unexpected = model.load_state_dict(sd, strict=False)
        assert not unexpected and all("rotary" in m or "inv_freq" in m for m in missing), (missing, unexpected)
        rng = np.random.RandomState({"llama3": 31, "linear": 41}[name])
        prompt = rng.randint(0, M["vocab"], size=PROMPT_LEN).astype(np.int64)
        ids = torch.from_numpy(prompt)[None]
        with torch.no_grad():
            full = model(ids).logits[0].float().numpy()
            gen = model.generate(ids, max_new_tokens=10, do_sample=False, use_cache=True, pad_token_id=0, eos_token_id=None)[0, len(prompt):].numpy()
        out["prompt_" + name] = prompt.astype(np.int32)
        out["logits_" + name] = full[-6:].astype(np.float32)
        out["greedy_" + name] = gen.astype(np.int32)
    np.savez_compressed(os.path.join(os.path.dirname(__file__), "llama_rope_scaling_golden.npz"), **out)
    print("wrote", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
