"""The HTTP shim's start-up checks that need no GPU: unreadable / malformed checkpoints and
`--model auto` without a describing file stop the process with a message before the engine is
touched."""
import os
import subprocess

import pytest

from llmlb_b200 import build

BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "llmlb_b200", "llmlb_b200_server")


@pytest.fixture(scope="module")
def server_bin():
    build.build()
    build.build_host()
    assert os.path.exists(BIN)
    return BIN


def run(server_bin, *args):
    return subprocess.run([server_bin, "--port", "1", *args], capture_output=True, text=True, timeout=120)


def test_bad_checkpoints_are_rejected_before_the_engine_starts(server_bin, tmp_path):
    r = run(server_bin, "--weights", str(tmp_path / "missing.gguf"))
    assert r.returncode == 2 and "cannot read" in r.stderr
    bad = tmp_path / "bad.gguf"
    bad.write_bytes(b"GGUF" + (7).to_bytes(4, "little") + b"\0" * 64)
    r = run(server_bin, "--weights", str(bad))
    assert r.returncode == 2 and "unsupported version" in r.stderr
    r = run(server_bin, "--model", "auto")
    assert r.returncode == 2 and "--model auto needs --weights" in r.stderr


# ---- `--dry-run`: everything the start-up decides without a GPU (geometry, weight plan, tokenizer) ----
def _bits(seed=2):
    import numpy as np
    from llmlb_b200.ffi import LLAMA_TINY
    from oracle.synth import f32_to_bf16_bits, synth_state_dict
    sd = synth_state_dict(LLAMA_TINY, seed=seed)
    return LLAMA_TINY, {k: f32_to_bf16_bits(np.asarray(v, dtype=np.float32)) for k, v in sd.items()}


def test_dry_run_single_gguf_takes_head_dim_from_the_q_projection(server_bin, tmp_path):
    """The file has hidden 512 and 8 heads of 128 and no attention.key_length: hidden / heads = 64 is
    the wrong head width (this is what failed on the GPU in round 1)."""
    import json
    pytest.importorskip("gguf")
    from gguf_util import write_tiny_llama_gguf
    p = tmp_path / "tiny.gguf"
    M = write_tiny_llama_gguf(p)
    r = run(server_bin, "--dry-run", "--model", "auto", "--weights", str(p))
    assert r.returncode == 0, r.stderr
    j = json.loads(r.stdout)
    assert j["dry_run"] and j["model"] == {k: M[k] for k in ("hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "ffn", "vocab")}
    assert j["tensors_to_load"] == 3 + 9 * M["n_layers"] and j["tokenizer_entries"] == M["vocab"] and j["stop_ids"] == 3


def test_dry_run_sharded_safetensors_merge_geometry_and_need_every_weight(server_bin, tmp_path):
    import json
    from llmlb_b200 import weights
    M, bits = _bits()
    a = {k: v for k, v in bits.items() if ".layers.1." not in k and k not in ("model.norm.weight", "lm_head.weight")}
    b = {k: v for k, v in bits.items() if k not in a}
    pa, pb = tmp_path / "model-00001-of-00002.safetensors", tmp_path / "model-00002-of-00002.safetensors"
    weights.write_safetensors(pa, a); weights.write_safetensors(pb, b)
    r = run(server_bin, "--dry-run", "--model", "auto", "--weights", str(pa), "--weights", str(pb))
    assert r.returncode == 0, r.stderr
    j = json.loads(r.stdout)
    assert j["model"]["n_layers"] == 2 and j["model"]["vocab"] == M["vocab"] and j["tensors_to_load"] == len(bits) and not j["lm_head_tied"]
    # the first shard alone used to start a truncated, partly synthetic model: now it is refused
    r = run(server_bin, "--dry-run", "--model", "auto", "--weights", str(pa))
    assert r.returncode == 2 and ("do not describe the whole model" in r.stderr or "are in none of the files" in r.stderr)
    # explicit geometry + a shard missing: the missing weights are named
    r = run(server_bin, "--dry-run", "--model", "tiny", "--weights", str(pa))
    assert r.returncode == 2 and "are in none of the files" in r.stderr and "model.layers.1." in r.stderr


def test_dry_run_tied_head_unexpected_and_misshapen_tensors(server_bin, tmp_path):
    import json
    import numpy as np
    from llmlb_b200 import weights
    M, bits = _bits(seed=4)
    tied = {k: v for k, v in bits.items() if k != "lm_head.weight"}
    p = tmp_path / "tied.safetensors"
    weights.write_safetensors(p, tied)
    r = run(server_bin, "--dry-run", "--model", "auto", "--weights", str(p))
    assert r.returncode == 0, r.stderr
    j = json.loads(r.stdout)
    assert j["lm_head_tied"] and j["tensors_to_load"] == len(bits)     # lm_head is loaded from the embedding
    extra = dict(bits); extra["model.layers.0.mlp.experts.0.w1.weight"] = np.zeros((4, 8), dtype=np.uint16)
    q = tmp_path / "extra.safetensors"
    weights.write_safetensors(q, extra)
    r = run(server_bin, "--dry-run", "--model", "tiny", "--weights", str(q))
    assert r.returncode == 2 and "unexpected tensor model.layers.0.mlp.experts.0.w1.weight" in r.stderr
    ok = dict(bits); ok["model.layers.0.self_attn.rotary_emb.inv_freq"] = np.zeros((64,), dtype=np.uint16)   # a known non-weight buffer
    q2 = tmp_path / "buf.safetensors"
    weights.write_safetensors(q2, ok)
    assert run(server_bin, "--dry-run", "--model", "tiny", "--weights", str(q2)).returncode == 0
    bad = dict(bits); bad["model.layers.1.mlp.down_proj.weight"] = bits["model.layers.1.mlp.down_proj.weight"][:, :-8]
    q3 = tmp_path / "shape.safetensors"
    weights.write_safetensors(q3, bad)
    r = run(server_bin, "--dry-run", "--model", "tiny", "--weights", str(q3))
    assert r.returncode == 2 and "model.layers.1.mlp.down_proj.weight is" in r.stderr
