"""GGUF checkpoints through the C ABI (SURVEY.md §8 f4, "GGUF-q4 dequant-on-load"): a
dependency-free GGUF v2/v3 reader, block dequantisers for the formats Llama GGUF files use
(F32, F16, BF16, Q8_0, Q4_0, Q4_1, Q5_0, Q5_1, Q4_K, Q5_K, Q6_K), the llama.cpp -> Hugging Face
tensor-name map with the Q/K row un-permutation, and `load_gguf`, which expands every tensor to
bf16 on the host and feeds `llmlb_engine_load_tensor` (the engine computes in bf16; quantised
execution is a later row).  Block layouts are ggml's (ggml-common.h); the arithmetic is pinned
against llama.cpp's own `gguf` Python package in tests/test_gguf.py.

The reference never reads model files itself — its endpoints (xLLM / llama.cpp / Ollama) do; this
is the loader an in-process endpoint needs to take the same .gguf artefacts.
"""
import mmap
import os
import struct

import numpy as np

GGUF_MAGIC = 0x46554747  # "GGUF"
QK_K = 256

# ggml type id -> (name, elements per block, bytes per block)
GGML_TYPES = {
    0: ("F32", 1, 4), 1: ("F16", 1, 2), 2: ("Q4_0", 32, 18), 3: ("Q4_1", 32, 20), 6: ("Q5_0", 32, 22), 7: ("Q5_1", 32, 24),
    8: ("Q8_0", 32, 34), 12: ("Q4_K", QK_K, 144), 13: ("Q5_K", QK_K, 176), 14: ("Q6_K", QK_K, 210), 30: ("BF16", 1, 2),
}
_SCALAR = {0: "<B", 1: "<b", 2: "<H", 3: "<h", 4: "<I", 5: "<i", 6: "<f", 7: "<?", 10: "<Q", 11: "<q", 12: "<d"}


class GGUFError(ValueError):
    pass


class _Cursor:
    def __init__(self, buf):
        self.buf, self.pos = buf, 0

    def take(self, fmt):
        size = struct.calcsize(fmt)
        if self.pos + size > len(self.buf):
            raise GGUFError("truncated GGUF header")
        (v,) = struct.unpack_from(fmt, self.buf, self.pos)
        self.pos += size
        return v

    def string(self):
        n = self.take("<Q")
        if self.pos + n > len(self.buf):
            raise GGUFError("truncated GGUF string")
        s = bytes(self.buf[self.pos:self.pos + n]).decode("utf-8", errors="replace")
        self.pos += n
        return s

    def value(self, vtype):
        if vtype in _SCALAR:
            return self.take(_SCALAR[vtype])
        if vtype == 8:
            return self.string()
        if vtype == 9:
            etype, count = self.take("<I"), self.take("<Q")
            if etype in _SCALAR and etype != 7:        # homogeneous numeric array: one unpack
                fmt = "<%d%s" % (count, _SCALAR[etype][1])
                size = struct.calcsize(fmt)
                vals = list(struct.unpack_from(fmt, self.buf, self.pos))
                self.pos += size
                return vals
            return [self.value(etype) for _ in range(count)]
        raise GGUFError("unknown GGUF value type %d" % vtype)


def read_gguf(path):
    """-> (metadata dict, tensors list of dicts {name, shape (row-major: outermost first), type,
    offset (absolute), nbytes}, mmap).  The caller closes the mmap."""
    f = open(path, "rb")
    mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    f.close()
    cur = _Cursor(mm)
    if cur.take("<I") != GGUF_MAGIC:
        mm.close()
        raise GGUFError("not a GGUF file: " + str(path))
    version = cur.take("<I")
    if version not in (2, 3):
        mm.close()
        raise GGUFError("unsupported GGUF version %d" % version)
    n_tensors, n_kv = cur.take("<Q"), cur.take("<Q")
    meta = {}
    for _ in range(n_kv):
        key = cur.string()
        meta[key] = cur.value(cur.take("<I"))
    infos = []
    for _ in range(n_tensors):
        name = cur.string()
        nd = cur.take("<I")
        dims = [cur.take("<Q") for _ in range(nd)]          # ggml order: innermost first
        ttype, off = cur.take("<I"), cur.take("<Q")
        infos.append((name, dims, ttype, off))
    align = int(meta.get("general.alignment", 32))
    base = (cur.pos + align - 1) // align * align
    tensors = []
    for name, dims, ttype, off in infos:
        if ttype not in GGML_TYPES:
            mm.close()
            raise GGUFError("tensor %s: unsupported ggml type %d" % (name, ttype))
        _, per, bsz = GGML_TYPES[ttype]
        n = int(np.prod(dims)) if dims else 1
        if dims and dims[0] % per:
            mm.close()
            raise GGUFError("tensor %s: row length %d is not a multiple of the block size %d" % (name, dims[0], per))
        nbytes = n // per * bsz
        if base + off + nbytes > len(mm):
            mm.close()
            raise GGUFError("tensor %s: data past the end of the file" % name)
        tensors.append({"name": name, "shape": list(reversed(dims)), "type": ttype, "offset": base + off, "nbytes": nbytes})
    return meta, tensors, mm


# ---- block dequantisers: raw bytes -> float32, one row of the result per block ------------------
def _f16(raw2):
    return np.ascontiguousarray(raw2).view(np.float16).astype(np.float32)


def _k_scales(s12):
    """The 12-byte scale field of Q4_K / Q5_K: eight 6-bit scales and eight 6-bit minima.
    Sub-blocks 0..3 sit in the low 6 bits of bytes 0..3 / 4..7; sub-blocks 4..7 take their low 4 bits
    from bytes 8..11 and their top 2 bits from the spare top bits of bytes 0..3 / 4..7."""
    a, b, c = s12[:, 0:4], s12[:, 4:8], s12[:, 8:12]
    sc = np.concatenate([a & 63, (c & 15) | ((a >> 6) << 4)], axis=1)
    mn = np.concatenate([b & 63, (c >> 4) | ((b >> 6) << 4)], axis=1)
    return sc.astype(np.float32), mn.astype(np.float32)


def _deq_q8_0(blk):
    d = _f16(blk[:, 0:2])
    return d * blk[:, 2:34].view(np.int8).astype(np.float32)


def _nibbles(qs):
    """[n, k] bytes -> [n, 2k]: the k low nibbles first, then the k high nibbles (ggml's Q4/Q5 order)."""
    return np.concatenate([qs & 15, qs >> 4], axis=1)


def _deq_q4_0(blk):
    d = _f16(blk[:, 0:2])
    return d * (_nibbles(blk[:, 2:18]).astype(np.int8) - np.int8(8)).astype(np.float32)


def _deq_q4_1(blk):
    d, m = _f16(blk[:, 0:2]), _f16(blk[:, 2:4])
    return d * _nibbles(blk[:, 4:20]).astype(np.float32) + m


def _fifth_bits(qh4):
    """4 bytes = 32 bits, bit j belongs to element j"""
    bits = np.ascontiguousarray(qh4).view("<u4")                       # [n, 1]
    return ((bits >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(np.uint8)


def _deq_q5_0(blk):
    d = _f16(blk[:, 0:2])
    q = _nibbles(blk[:, 6:22]) | (_fifth_bits(blk[:, 2:6]) << 4)
    return d * (q.astype(np.int8) - np.int8(16)).astype(np.float32)


def _deq_q5_1(blk):
    d, m = _f16(blk[:, 0:2]), _f16(blk[:, 2:4])
    q = _nibbles(blk[:, 8:24]) | (_fifth_bits(blk[:, 4:8]) << 4)
    return d * q.astype(np.float32) + m


def _deq_q4_k(blk):
    n = blk.shape[0]
    d, dmin = _f16(blk[:, 0:2]), _f16(blk[:, 2:4])
    sc, mn = _k_scales(blk[:, 4:16])
    qs = blk[:, 16:144].reshape(n, 4, 32)                              # 4 groups of 32 bytes = 64 elements each
    q = np.stack([qs & 15, qs >> 4], axis=2).reshape(n, 8, 32).astype(np.float32)   # sub-block 2g: low, 2g+1: high
    return ((d * sc)[:, :, None] * q - (dmin * mn)[:, :, None]).reshape(n, QK_K)


def _deq_q5_k(blk):
    n = blk.shape[0]
    d, dmin = _f16(blk[:, 0:2]), _f16(blk[:, 2:4])
    sc, mn = _k_scales(blk[:, 4:16])
    qh = blk[:, 16:48]                                                 # bit s of byte l: 5th bit of element l of sub-block s
    qs = blk[:, 48:176].reshape(n, 4, 32)
    lo = np.stack([qs & 15, qs >> 4], axis=2).reshape(n, 8, 32)
    hi = ((qh[:, None, :] >> np.arange(8, dtype=np.uint8)[None, :, None]) & 1).astype(np.uint8)
    q = (lo | (hi << 4)).astype(np.float32)
    return ((d * sc)[:, :, None] * q - (dmin * mn)[:, :, None]).reshape(n, QK_K)


def _deq_q6_k(blk):
    n = blk.shape[0]
    ql = blk[:, 0:128].reshape(n, 2, 64)                               # two halves of 128 elements
    qh = blk[:, 128:192].reshape(n, 2, 32)
    sc = blk[:, 192:208].view(np.int8).astype(np.float32)             # 16 sub-blocks of 16 elements
    d = _f16(blk[:, 208:210])
    # within a half: elements 0..31 / 32..63 take the low nibbles of ql[0..31] / ql[32..63], elements
    # 64..95 / 96..127 the high nibbles; their top two bits are bit pairs 0,1,2,3 of qh[0..31]
    low = np.concatenate([ql[:, :, 0:32] & 15, ql[:, :, 32:64] & 15, ql[:, :, 0:32] >> 4, ql[:, :, 32:64] >> 4], axis=2)
    top = np.concatenate([(qh >> s) & 3 for s in (0, 2, 4, 6)], axis=2)
    q = ((low | (top << 4)).astype(np.int8) - np.int8(32)).reshape(n, 16, 16).astype(np.float32)
    return ((d * sc)[:, :, None] * q).reshape(n, QK_K)


_DEQ = {8: _deq_q8_0, 2: _deq_q4_0, 3: _deq_q4_1, 6: _deq_q5_0, 7: _deq_q5_1, 12: _deq_q4_k, 13: _deq_q5_k, 14: _deq_q6_k}


def dequantize(raw, ggml_type, n_elements):
    """raw: uint8 array of the tensor's bytes -> float32 [n_elements]"""
    if ggml_type not in GGML_TYPES:
        raise GGUFError("unsupported ggml type %d" % ggml_type)
    name, per, bsz = GGML_TYPES[ggml_type]
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if n_elements % per or raw.size != n_elements // per * bsz:
        raise GGUFError("%s: %d bytes do not hold %d elements" % (name, raw.size, n_elements))
    if ggml_type == 0:
        return raw.view("<f4").astype(np.float32)
    if ggml_type == 1:
        return raw.view("<f2").astype(np.float32)
    if ggml_type == 30:
        return (raw.view("<u2").astype(np.uint32) << np.uint32(16)).view(np.float32)
    return _DEQ[ggml_type](raw.reshape(-1, bsz)).reshape(-1)


def to_bf16_bits(x):
    """float32 -> bf16 bit patterns, round to nearest even (NaN stays NaN)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((u + (np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1)))) >> np.uint32(16)).astype(np.uint16)
    nan = (u & np.uint32(0x7FFFFFFF)) > np.uint32(0x7F800000)
    r[nan] = (u[nan] >> np.uint32(16)).astype(np.uint16) | np.uint16(0x40)
    return r


# ---- llama.cpp naming / layout -> the Hugging Face names the engine's loader speaks --------------
_LAYER_MAP = {
    "attn_norm": "input_layernorm", "attn_q": "self_attn.q_proj", "attn_k": "self_attn.k_proj", "attn_v": "self_attn.v_proj",
    "attn_output": "self_attn.o_proj", "ffn_norm": "post_attention_layernorm", "ffn_gate": "mlp.gate_proj",
    "ffn_up": "mlp.up_proj", "ffn_down": "mlp.down_proj",
}


def hf_name(gguf_name):
    """'blk.3.attn_q.weight' -> 'model.layers.3.self_attn.q_proj.weight'; None for tensors the
    engine has no use for (rope_freqs, ...)."""
    if gguf_name == "token_embd.weight":
        return "model.embed_tokens.weight"
    if gguf_name == "output_norm.weight":
        return "model.norm.weight"
    if gguf_name == "output.weight":
        return "lm_head.weight"
    parts = gguf_name.split(".")
    if len(parts) == 4 and parts[0] == "blk" and parts[1].isdigit() and parts[3] == "weight" and parts[2] in _LAYER_MAP:
        return "model.layers.%s.%s.weight" % (parts[1], _LAYER_MAP[parts[2]])
    return None


def unpermute_qk(w, n_head):
    """llama.cpp's converter stores Q/K rows so that a head's rotary pairs are adjacent (2i, 2i+1);
    the engine (like Hugging Face) rotates (i, i + head_dim/2).  Inverse of convert_hf_to_gguf's
    `permute`: rows [head][pair][half] -> [head][half][pair]."""
    rows, cols = w.shape
    hd = rows // n_head
    return w.reshape(n_head, hd // 2, 2, cols).swapaxes(1, 2).reshape(rows, cols)


def geometry(meta, tensors):
    """Model geometry dict (the keys of ffi.LLAMA3_8B) from llama.* metadata."""
    arch = meta.get("general.architecture", "llama")
    g = lambda k, d=None: meta.get("%s.%s" % (arch, k), d)
    hidden, heads = int(g("embedding_length")), int(g("attention.head_count"))
    emb = [t for t in tensors if t["name"] == "token_embd.weight"]
    vocab = emb[0]["shape"][0] if emb else int(g("vocab_size", len(meta.get("tokenizer.ggml.tokens", []))))
    # head width: metadata when present, else the q projection's own shape (rows / heads)
    q = [t for t in tensors if t["name"].endswith("attn_q.weight")]
    hd_default = q[0]["shape"][0] // heads if q and q[0]["shape"][1] == hidden else hidden // heads
    return {"hidden": hidden, "n_layers": int(g("block_count")), "n_heads": heads, "n_kv_heads": int(g("attention.head_count_kv", heads)),
            "head_dim": int(g("attention.key_length", hd_default)), "ffn": int(g("feed_forward_length")), "vocab": int(vocab),
            "rope_theta": float(g("rope.freq_base", 10000.0)), "rms_eps": float(g("attention.layer_norm_rms_epsilon", 1e-5))}


def rope_scaling(meta, tensors, mm):
    """RoPE frequency scaling a GGUF file states: (type, float32 divisors [head_dim/2] or None).
    `rope_freqs.weight` (F32, what convert_hf_to_gguf.py writes for Llama 3.1+) is returned bit for bit
    as type "rope_freqs"; `{arch}.rope.scaling.type = linear` multiplies every divisor by its factor;
    "none" or no key is no scaling.  Any other type raises GGUFError."""
    arch = meta.get("general.architecture", "llama")
    n = geometry(meta, tensors)["head_dim"] // 2
    kind, f = "none", None
    rf = [t for t in tensors if t["name"] == "rope_freqs.weight"]
    if rf:
        t = rf[0]
        if t["type"] != 0 or t["shape"] != [n] or n == 0:
            raise GGUFError("rope_freqs.weight must be %d F32 values (head_dim / 2)" % n)
        f = np.frombuffer(mm, dtype="<f4", count=n, offset=t["offset"]).astype(np.float32)
        if not (np.isfinite(f).all() and (f > 0).all()):
            raise GGUFError("rope_freqs.weight holds a factor that is not finite and > 0")
        kind = "rope_freqs"
    stype = meta.get(arch + ".rope.scaling.type")
    if stype not in (None, "", "none"):
        if stype != "linear":
            raise GGUFError("unsupported RoPE scaling type %r: only linear and rope_freqs.weight are served" % (stype,))
        factor = float(meta.get(arch + ".rope.scaling.factor", 0.0))
        if not (np.isfinite(factor) and factor > 0):
            raise GGUFError("RoPE scaling: factor must be finite and > 0")
        lin = np.full(n, factor, dtype=np.float32)
        f = lin if f is None else f * lin      # llama.cpp applies both
        kind = "linear"
    return kind, f


def read_rope_scaling(path):
    """rope_scaling() of the file at `path`."""
    meta, tensors, mm = read_gguf(os.fspath(path))
    try:
        return rope_scaling(meta, tensors, mm)
    finally:
        mm.close()


def iter_hf_tensors(path):
    """Yields (hf_name, bf16 bits [rows, cols]) for every tensor the engine can take, dequantised and
    with Q/K rows back in Hugging Face order.  A tied output head (no output.weight) is served
    from the embedding."""
    meta, tensors, mm = read_gguf(path)
    try:
        arch = meta.get("general.architecture", "llama")
        n_head = int(meta.get(arch + ".attention.head_count", 1))
        n_kv = int(meta.get(arch + ".attention.head_count_kv", n_head))
        names = {t["name"] for t in tensors}
        for t in tensors:
            name = hf_name(t["name"])
            if name is None:
                continue
            shape = t["shape"]
            rows, cols = (shape[0], shape[1]) if len(shape) == 2 else (1, shape[0])
            raw = np.frombuffer(mm, dtype=np.uint8, count=t["nbytes"], offset=t["offset"])
            w = dequantize(raw, t["type"], rows * cols).reshape(rows, cols)
            if t["name"].endswith("attn_q.weight"):
                w = unpermute_qk(w, n_head)
            elif t["name"].endswith("attn_k.weight"):
                w = unpermute_qk(w, n_kv)
            bits = to_bf16_bits(w).reshape(rows, cols)
            yield name, bits
            if name == "model.embed_tokens.weight" and "output.weight" not in names:
                yield "lm_head.weight", bits
            del raw, w
    finally:
        mm.close()


def load_gguf(engine, path):
    """Feeds a .gguf checkpoint to the engine; returns the Hugging Face names loaded."""
    from . import ffi
    loaded = []
    for name, bits in iter_hf_tensors(os.fspath(path)):
        try:
            engine.load_tensor(name, bits)
            loaded.append(name)
        except ffi.LlmlbError as e:
            if e.code != ffi.E_NOT_FOUND:
                raise
    return loaded


# ---- the tokenizer a .gguf carries (tokenizer.ggml.*) -> tokenizer.json for the native tokenizer ----
LLAMA3_SPLIT_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*"
                        r"|\s*[\r\n]+|\s+(?!\S)|\s+")
_TOKEN_CONTROL, _TOKEN_USER_DEFINED = 3, 4      # llama.cpp token types that are matched as whole strings


def tokenizer_json_from_gguf(meta):
    """A Hugging Face style tokenizer.json (dict) from GGUF metadata: model "gpt2" (byte-level BPE)
    with the "llama-bpe" pre-tokenizer — what Llama-3 GGUF files carry.  Tokens of type CONTROL /
    USER_DEFINED become added tokens (control ones flagged special), the rest the BPE vocabulary;
    `tokenizer.ggml.bos_token_id` becomes the begin-of-text token of the post-processor."""
    model = meta.get("tokenizer.ggml.model")
    if model != "gpt2":
        raise GGUFError("tokenizer.ggml.model is %r: only byte-level BPE (gpt2) is supported" % (model,))
    pre = meta.get("tokenizer.ggml.pre", "llama-bpe")
    if pre not in ("llama-bpe", "llama3", "llama-v3"):
        raise GGUFError("tokenizer.ggml.pre is %r: only the Llama-3 pre-tokenizer is implemented" % (pre,))
    tokens = meta.get("tokenizer.ggml.tokens")
    merges = meta.get("tokenizer.ggml.merges")
    if not isinstance(tokens, list) or not isinstance(merges, list):
        raise GGUFError("tokenizer.ggml.tokens / merges missing")
    types = meta.get("tokenizer.ggml.token_type") or [1] * len(tokens)
    vocab, added = {}, []
    for i, (tok, ty) in enumerate(zip(tokens, types)):
        if ty in (_TOKEN_CONTROL, _TOKEN_USER_DEFINED):
            added.append({"id": i, "content": tok, "single_word": False, "lstrip": False, "rstrip": False,
                          "normalized": False, "special": ty == _TOKEN_CONTROL})
        else:
            vocab[tok] = i
    out = {
        "version": "1.0", "truncation": None, "padding": None, "added_tokens": added, "normalizer": None,
        "pre_tokenizer": {"type": "Sequence", "pretokenizers": [
            {"type": "Split", "pattern": {"Regex": LLAMA3_SPLIT_PATTERN}, "behavior": "Isolated", "invert": False},
            {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": False}]},
        "post_processor": None,
        "decoder": {"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True},
        "model": {"type": "BPE", "dropout": None, "unk_token": None, "continuing_subword_prefix": None,
                  "end_of_word_suffix": None, "fuse_unk": False, "byte_fallback": False, "ignore_merges": True,
                  "vocab": vocab, "merges": list(merges)},
    }
    bos = meta.get("tokenizer.ggml.bos_token_id")
    if isinstance(bos, int) and 0 <= bos < len(tokens):
        out["post_processor"] = {"type": "TemplateProcessing",
                                 "single": [{"SpecialToken": {"id": tokens[bos], "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}}],
                                 "pair": [], "special_tokens": {tokens[bos]: {"id": tokens[bos], "ids": [bos], "tokens": [tokens[bos]]}}}
    return out
