"""Helpers shared by the RoPE-scaling tests: the scaling configs of real Llama checkpoints, llama.cpp's converter
arithmetic for rope_freqs.weight, and writers of small Llama 3.1-style checkpoints (GGUF with rope_freqs.weight,
safetensors with a config.json beside it)."""
import json
import math
import os

import numpy as np

THETA = 500000.0
# rope_scaling of the published config.json files
LLAMA31_8B = {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192, "rope_type": "llama3"}
LLAMA32_3B = {"factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192, "rope_type": "llama3"}
LLAMA33_70B = {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192, "rope_type": "llama3"}
LINEAR2 = {"rope_type": "linear", "factor": 2.0}
LINEAR4 = {"rope_type": "linear", "factor": 4.0}
SCALINGS = {"llama3.1-8b": LLAMA31_8B, "llama3.2-3b": LLAMA32_3B, "llama3.3-70b": LLAMA33_70B, "linear2": LINEAR2, "linear4": LINEAR4}


def convert_rope_factors(rs, theta=THETA, head_dim=128):
    """rope_freqs.weight as llama.cpp's convert_hf_to_gguf.py (LlamaModel.generate_extra_tensors) computes it:
    fp32 base frequencies, Python-float band arithmetic, stored as float32."""
    import torch
    factor, low, high = rs.get("factor", 8.0), rs.get("low_freq_factor", 1.0), rs.get("high_freq_factor", 4.0)
    old = rs.get("original_max_position_embeddings", 8192)
    freqs = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim))
    out = []
    for freq in freqs:
        wavelen = 2 * math.pi / freq
        if wavelen < old / high:
            out.append(1)
        elif wavelen > old / low:
            out.append(factor)
        else:
            smooth = (old / wavelen - low) / (high - low)
            out.append(1 / ((1 - smooth) / factor + smooth))
    return np.array(out, dtype=np.float32)


def write_llama_gguf(path, M, sd, rope_freqs=None, scaling_type=None, scaling_factor=None):
    """A whole Llama as one .gguf (F32 tensors, Q/K rows permuted as the converter does), optionally with
    rope_freqs.weight and {arch}.rope.scaling.type / .factor metadata."""
    import gguf
    from gguf_util import _to_gguf_name
    w = gguf.GGUFWriter(str(path), "llama")
    w.add_uint32("llama.block_count", M["n_layers"]); w.add_uint32("llama.embedding_length", M["hidden"])
    w.add_uint32("llama.feed_forward_length", M["ffn"]); w.add_uint32("llama.attention.head_count", M["n_heads"])
    w.add_uint32("llama.attention.head_count_kv", M["n_kv_heads"]); w.add_float32("llama.rope.freq_base", M["rope_theta"])
    w.add_float32("llama.attention.layer_norm_rms_epsilon", M["rms_eps"])
    w.add_uint32("llama.attention.key_length", M["head_dim"])
    if scaling_type is not None:
        w.add_string("llama.rope.scaling.type", scaling_type)
    if scaling_factor is not None:
        w.add_float32("llama.rope.scaling.factor", scaling_factor)
    for name, t in sd.items():
        t = np.asarray(t, dtype=np.float32)
        if name.endswith("q_proj.weight") or name.endswith("k_proj.weight"):
            nh = M["n_heads"] if "q_proj" in name else M["n_kv_heads"]
            t = np.ascontiguousarray(t.reshape(nh, 2, t.shape[0] // nh // 2, t.shape[1]).swapaxes(1, 2).reshape(t.shape))
        w.add_tensor(_to_gguf_name(name), t)
    if rope_freqs is not None:
        w.add_tensor("rope_freqs.weight", np.asarray(rope_freqs, dtype=np.float32))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()


def hf_config(M, rope_scaling=None, **over):
    """config.json of a Hugging Face Llama checkpoint in the classic form (rope_theta + rope_scaling)."""
    c = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "hidden_size": M["hidden"], "num_hidden_layers": M["n_layers"],
         "num_attention_heads": M["n_heads"], "num_key_value_heads": M["n_kv_heads"], "head_dim": M["head_dim"],
         "intermediate_size": M["ffn"], "vocab_size": M["vocab"], "rope_theta": M["rope_theta"], "rms_norm_eps": M["rms_eps"],
         "max_position_embeddings": 131072, "rope_scaling": rope_scaling, "tie_word_embeddings": False, "torch_dtype": "bfloat16"}
    c.update(over)
    return c


def write_safetensors_dir(d, M, sd, config=None):
    """model.safetensors (bf16) in directory d, with config.json (a dict) beside it when given; returns the shard path."""
    from llmlb_b200 import weights
    from oracle.synth import f32_to_bf16_bits
    os.makedirs(d, exist_ok=True)
    p = os.path.join(str(d), "model.safetensors")
    weights.write_safetensors(p, {k: f32_to_bf16_bits(np.asarray(v, dtype=np.float32)) for k, v in sd.items()})
    if config is not None:
        with open(os.path.join(str(d), "config.json"), "w") as f:
            json.dump(config, f)
    return p


def native_ckpt(lib_path):
    """ctypes handle of the host library's checkpoint surface, RoPE factors included."""
    import ctypes as C
    lib = C.CDLL(lib_path)
    lib.llmlb_ckpt_open.restype = C.c_void_p
    lib.llmlb_ckpt_open.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32]
    lib.llmlb_ckpt_close.argtypes = [C.c_void_p]
    lib.llmlb_ckpt_geometry.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
    lib.llmlb_ckpt_rope_freq_factors.restype = C.c_uint32
    lib.llmlb_ckpt_rope_freq_factors.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_uint32]
    return lib


def native_open(K, path):
    """-> (geometry dict, float32 factors or None); raises ValueError with the reader's message."""
    import ctypes as C
    err = C.create_string_buffer(512)
    h = K.llmlb_ckpt_open(str(path).encode(), err, 512)
    if not h:
        raise ValueError(err.value.decode())
    try:
        u7, f2 = (C.c_uint32 * 7)(), (C.c_float * 2)()
        known = K.llmlb_ckpt_geometry(h, u7, f2)
        geo = dict(zip(["hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "ffn", "vocab"], list(u7)))
        geo.update(rope_theta=f2[0], rms_eps=f2[1], known=bool(known))
        n = K.llmlb_ckpt_rope_freq_factors(h, None, 0)
        buf = np.zeros(max(n, 1), dtype=np.float32)
        assert K.llmlb_ckpt_rope_freq_factors(h, buf.ctypes.data_as(C.POINTER(C.c_float)), n) == n
        return geo, (buf[:n] if n else None)
    finally:
        K.llmlb_ckpt_close(h)
