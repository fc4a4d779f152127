"""RoPE frequency scaling (llama3 / linear) on the CPU: the oracle against Hugging Face transformers, the native and
oracle factor functions against transformers' ROPE_INIT_FUNCTIONS, both GGUF readers against llama.cpp's converter
arithmetic, config.json beside safetensors shards, and the server's start-up report."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from rope_oracle import ScaledLlamaRef as LlamaRef, rope_freq_factors
from oracle.synth import synth_state_dict
from rope_scaling_util import (LINEAR4, LLAMA31_8B, SCALINGS, THETA, convert_rope_factors, hf_config, native_ckpt, native_open,
                               write_llama_gguf, write_safetensors_dir)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "llama_rope_scaling_golden.npz")
SMALL = dict(hidden=256, n_layers=1, n_heads=4, n_kv_heads=1, head_dim=128, ffn=512, vocab=384, rope_theta=THETA, rms_eps=1e-5)


def _golden_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk_rope", os.path.join(HERE, "golden", "make_llama_rope_scaling_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


# ---- 1. the oracle against transformers' LlamaForCausalLM with rope_scaling ----
@pytest.mark.parametrize("name", ["llama3", "linear"])
def test_oracle_with_rope_scaling_matches_transformers(name):
    mk = _golden_module()
    g = np.load(GOLD)
    sd = synth_state_dict(mk.TINY, seed=11)
    r = LlamaRef(dict(mk.TINY, rope_scaling=mk.SCALINGS[name]), sd)
    lg = r.forward(g["prompt_" + name]).numpy()[-6:]
    assert np.abs(lg - g["logits_" + name]).max() < 3e-5
    toks, _ = r.greedy(g["prompt_" + name], len(g["greedy_" + name]))
    assert toks == g["greedy_" + name].tolist()
    # the fixture discriminates: the same oracle without scaling misses it by far more than the tolerance
    plain = LlamaRef(mk.TINY, sd).forward(g["prompt_" + name]).numpy()[-6:]
    assert np.abs(plain - g["logits_" + name]).max() > 100 * 3e-5


def test_oracle_without_scaling_keeps_its_inv_freq_bit_for_bit():
    hd = 128
    want = 1.0 / (THETA ** (torch.arange(0, hd, 2, dtype=torch.float64) / hd))
    for cfg in (dict(SMALL), dict(SMALL, rope_scaling=None), dict(SMALL, rope_scaling={"rope_type": "default"})):
        assert torch.equal(LlamaRef(cfg, {}).inv_freq, want)
    with pytest.raises(ValueError, match="yarn"):
        rope_freq_factors({"rope_type": "yarn", "factor": 4.0}, THETA)


def test_oracle_tail_path_equals_the_full_forward():
    """forward_tail (K/V everywhere, queries only for the last rows) against forward() at a short length, then decode
    steps continue from the cache it leaves."""
    sd = synth_state_dict(SMALL, seed=3)
    cfg = dict(SMALL, rope_scaling=LLAMA31_8B)
    p = np.random.RandomState(4).randint(0, SMALL["vocab"], size=700)
    full = LlamaRef(cfg, sd)
    want = full.forward(p).numpy()
    tail = LlamaRef(cfg, sd)
    got = tail.forward_tail(p, 7).numpy()
    assert got.shape == (7, SMALL["vocab"]) and np.abs(got - want[-7:]).max() < 1e-4
    for t in (5, 77, 300):
        a, b = full.forward([t]).numpy(), tail.forward([t]).numpy()
        assert np.abs(a - b).max() < 1e-4
    with pytest.raises(ValueError):
        LlamaRef(dict(SMALL, n_layers=2), synth_state_dict(dict(SMALL, n_layers=2), seed=3)).forward_tail(p, 2)


# ---- 2. factor functions (native host code and oracle) against transformers' ROPE_INIT_FUNCTIONS ----
@pytest.fixture(scope="module")
def K():
    from llmlb_b200 import build
    return native_ckpt(build.build_host())


def _transformers_inv_freq(rs):
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    c = LlamaConfig(hidden_size=4096, num_attention_heads=32, head_dim=128, rope_theta=THETA, rope_scaling=dict(rs),
                    max_position_embeddings=131072)
    inv, attn = ROPE_INIT_FUNCTIONS[rs["rope_type"]](c, "cpu")
    assert attn == 1.0
    return inv.double().numpy()


def _bands(rs, inv_base):
    """high (0) / medium (1) / low (2) band of each frequency by transformers' own test"""
    if rs["rope_type"] == "linear":
        return np.full(64, 2)
    wavelen = 2 * np.pi / inv_base
    old = rs["original_max_position_embeddings"]
    low, high = wavelen > old / rs["low_freq_factor"], wavelen < old / rs["high_freq_factor"]
    return np.where(low, 2, np.where(high, 0, 1))


def _bands_of(f, rs):
    return np.where(f == 1.0, 0, np.where(f == rs["factor"], 2, 1))


@pytest.mark.parametrize("name", sorted(SCALINGS))
def test_factor_functions_match_transformers(K, tmp_path, name):
    rs = SCALINGS[name]
    tf = _transformers_inv_freq(rs)
    base32 = (1.0 / (THETA ** (torch.arange(0, 128, 2, dtype=torch.int64).float() / 128))).double().numpy()   # transformers' base
    base64 = 1.0 / (THETA ** (np.arange(0, 128, 2, dtype=np.float64) / 128))
    M = dict(SMALL)
    p = write_safetensors_dir(tmp_path, M, synth_state_dict(M, seed=1), hf_config(M, rope_scaling=rs))
    _, native = native_open(K, p)
    oracle = rope_freq_factors(rs, THETA)
    assert native is not None and native.shape == (64,) and oracle.shape == (64,)
    want_bands = _bands(rs, base32)
    assert np.array_equal(_bands_of(native.astype(np.float64), rs), want_bands)
    assert np.array_equal(_bands_of(oracle, rs), want_bands)
    if rs["rope_type"] == "llama3":
        assert set(want_bands.tolist()) == {0, 1, 2}       # all three bands are exercised
    # inv_freq: transformers computes in fp32 (a float power, then up to two float operations), ours in fp64 divided by the
    # fp32-stored factor: within four fp32 roundings (2^-23 each)
    fp32 = 4 * 2.0 ** -23
    np.testing.assert_allclose(base64 / native.astype(np.float64), tf, rtol=fp32, atol=0)
    np.testing.assert_allclose(base64 / oracle, tf, rtol=fp32, atol=0)
    np.testing.assert_allclose(native, oracle.astype(np.float32), rtol=1.2e-7, atol=0)


# ---- 3. GGUF readers ----
def _py_gguf(path):
    from llmlb_b200 import gguf as G
    meta, tensors, mm = G.read_gguf(path)
    try:
        return G.geometry(meta, tensors), G.rope_scaling(meta, tensors, mm), [G.hf_name(t["name"]) for t in tensors]
    finally:
        mm.close()


def test_gguf_rope_freqs_read_bit_for_bit_by_both_readers(K, tmp_path):
    pytest.importorskip("gguf")
    M = dict(SMALL)
    sd = synth_state_dict(M, seed=2)
    plain, scaled = tmp_path / "plain.gguf", tmp_path / "llama31.gguf"
    write_llama_gguf(plain, M, sd)
    for name in ("llama3.1-8b", "llama3.2-3b"):
        ff = convert_rope_factors(SCALINGS[name])
        write_llama_gguf(scaled, M, sd, rope_freqs=ff)
        geo, (kind, f), names = _py_gguf(scaled)
        assert kind == "rope_freqs" and f.dtype == np.float32 and np.array_equal(f.view(np.uint32), ff.view(np.uint32))
        ngeo, nf = native_open(K, scaled)
        assert np.array_equal(nf.view(np.uint32), ff.view(np.uint32))
        assert names.count(None) == 1                                  # rope_freqs stays out of the weight list
        # the converter's fp32 arithmetic and ours agree to float rounding
        np.testing.assert_allclose(ff, rope_freq_factors(SCALINGS[name], THETA), rtol=1e-6)
        # geometry: exactly what a file without scaling gives
        pgeo, (pkind, pf), _ = _py_gguf(plain)
        assert geo == pgeo and (pkind, pf) == ("none", None)
        pngeo, pnf = native_open(K, plain)
        assert ngeo == pngeo and pnf is None


def test_gguf_scaling_metadata_linear_honoured_others_refused(K, tmp_path):
    pytest.importorskip("gguf")
    from llmlb_b200 import gguf as G
    M = dict(SMALL)
    sd = synth_state_dict(M, seed=2)
    p = tmp_path / "lin.gguf"
    write_llama_gguf(p, M, sd, scaling_type="linear", scaling_factor=4.0)
    _, (kind, f), _ = _py_gguf(p)
    _, nf = native_open(K, p)
    assert kind == "linear" and np.array_equal(f, np.full(64, 4.0, np.float32)) and np.array_equal(nf, f)
    p = tmp_path / "none.gguf"
    write_llama_gguf(p, M, sd, scaling_type="none")
    assert _py_gguf(p)[1] == ("none", None) and native_open(K, p)[1] is None
    for bad in ("yarn", "longrope", "dynamic", "something-new"):
        p = tmp_path / ("%s.gguf" % bad)
        write_llama_gguf(p, M, sd, scaling_type=bad, scaling_factor=4.0)
        with pytest.raises(G.GGUFError, match="unsupported RoPE scaling type"):
            _py_gguf(p)
        with pytest.raises(ValueError, match="unsupported RoPE scaling type '%s'" % bad):
            native_open(K, p)
    p = tmp_path / "short.gguf"                                        # rope_freqs of the wrong length
    write_llama_gguf(p, M, sd, rope_freqs=np.ones(32, np.float32))
    with pytest.raises(G.GGUFError, match="rope_freqs"):
        _py_gguf(p)
    with pytest.raises(ValueError, match="rope_freqs"):
        native_open(K, p)


# ---- 4. safetensors with config.json ----
def test_safetensors_config_json_both_forms_mismatch_and_absence(K, tmp_path):
    from transformers import LlamaConfig
    M = dict(SMALL)
    sd = synth_state_dict(M, seed=6)
    want = rope_freq_factors(LLAMA31_8B, 6e5)
    # the classic form (Llama 3.1 config.json), with a theta and eps of its own
    geo, f = native_open(K, write_safetensors_dir(tmp_path / "classic", M, sd, hf_config(M, rope_scaling=LLAMA31_8B, rope_theta=6e5, rms_norm_eps=1e-6)))
    assert geo["rope_theta"] == np.float32(6e5) and geo["rms_eps"] == np.float32(1e-6) and geo["known"]
    np.testing.assert_allclose(f, want, rtol=1.2e-7)
    # the older key `type`
    old = dict(LLAMA31_8B); old["type"] = old.pop("rope_type")
    np.testing.assert_allclose(native_open(K, write_safetensors_dir(tmp_path / "type", M, sd, hf_config(M, rope_scaling=old, rope_theta=6e5)))[1], want, rtol=1.2e-7)
    # transformers 5's rope_parameters, as LlamaConfig itself writes it
    c = LlamaConfig(hidden_size=M["hidden"], num_hidden_layers=M["n_layers"], num_attention_heads=M["n_heads"], num_key_value_heads=M["n_kv_heads"],
                    head_dim=128, intermediate_size=M["ffn"], vocab_size=M["vocab"], rope_theta=6e5, rms_norm_eps=1e-6,
                    rope_scaling=dict(LINEAR4), max_position_embeddings=131072)
    d = tmp_path / "tf5"
    write_safetensors_dir(d, M, sd)
    c.save_pretrained(str(d))
    cj = json.load(open(d / "config.json"))
    assert "rope_parameters" in cj and "rope_scaling" not in cj and "rope_theta" not in cj     # the form under test
    geo, f = native_open(K, d / "model.safetensors")
    assert geo["rope_theta"] == np.float32(6e5) and np.array_equal(f, np.full(64, 4.0, np.float32))
    # no scaling in the config: no factors, the config's theta
    geo, f = native_open(K, write_safetensors_dir(tmp_path / "noscale", M, sd, hf_config(M, rope_theta=1e4)))
    assert f is None and geo["rope_theta"] == np.float32(1e4)
    # a config that contradicts the tensor shapes is an error
    for key, val in (("hidden_size", 512), ("num_attention_heads", 8), ("num_key_value_heads", 2), ("intermediate_size", 1024),
                     ("vocab_size", 999)):
        with pytest.raises(ValueError, match=key):
            native_open(K, write_safetensors_dir(tmp_path / ("bad_" + key), M, sd, hf_config(M, **{key: val})))
    two = dict(M, n_layers=2)
    with pytest.raises(ValueError, match="num_hidden_layers"):      # the file holds layer 1, the config says one layer
        native_open(K, write_safetensors_dir(tmp_path / "layers", two, synth_state_dict(two, seed=6), hf_config(two, num_hidden_layers=1)))
    with pytest.raises(ValueError, match="head_dim 64"):
        native_open(K, write_safetensors_dir(tmp_path / "hd64", M, sd, hf_config(M, head_dim=64)))
    with pytest.raises(ValueError, match="unsupported RoPE scaling type 'yarn'"):
        native_open(K, write_safetensors_dir(tmp_path / "yarn", M, sd, hf_config(M, rope_scaling={"rope_type": "yarn", "factor": 4.0})))
    # without config.json: exactly today's values
    geo, f = native_open(K, write_safetensors_dir(tmp_path / "bare", M, sd))
    assert f is None and geo["rope_theta"] == np.float32(5e5) and geo["rms_eps"] == np.float32(1e-5)
    assert {k: geo[k] for k in ("hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "ffn", "vocab")} == \
        {k: M[k] for k in ("hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "ffn", "vocab")}


# ---- 5. the server's start-up report ----
@pytest.fixture(scope="module")
def server_bin():
    from llmlb_b200 import build
    build.build()
    build.build_host()
    path = os.path.join(os.path.dirname(HERE), "llmlb_b200", "llmlb_b200_server")
    assert os.path.exists(path)
    return path


def _dry_run(server_bin, *weights):
    args = [server_bin, "--port", "1", "--dry-run", "--model", "auto"]
    for w in weights:
        args += ["--weights", str(w)]
    return subprocess.run(args, capture_output=True, text=True, timeout=120)


def test_server_dry_run_reports_the_scaling_and_refuses_yarn(server_bin, tmp_path):
    pytest.importorskip("gguf")
    M = dict(SMALL)
    sd = synth_state_dict(M, seed=8)
    g = tmp_path / "llama31.gguf"
    write_llama_gguf(g, M, sd, rope_freqs=convert_rope_factors(LLAMA31_8B))
    r = _dry_run(server_bin, g)
    assert r.returncode == 0, r.stderr
    j = json.loads(r.stdout)
    assert j["rope_scaling"] == {"type": "rope_freqs", "factors": 64, "min_factor": 1.0, "max_factor": 8.0} and j["rope_theta"] == THETA
    p = write_safetensors_dir(tmp_path / "st", M, sd, hf_config(M, rope_scaling=LLAMA31_8B))
    r = _dry_run(server_bin, p)
    assert r.returncode == 0, r.stderr
    assert json.loads(r.stdout)["rope_scaling"] == {"type": "llama3", "factors": 64, "min_factor": 1.0, "max_factor": 8.0}
    r = _dry_run(server_bin, write_safetensors_dir(tmp_path / "plain", M, sd))
    assert r.returncode == 0 and json.loads(r.stdout)["rope_scaling"] == {"type": "none"}
    r = _dry_run(server_bin, write_safetensors_dir(tmp_path / "yarn", M, sd, hf_config(M, rope_scaling={"rope_type": "yarn", "factor": 4.0})))
    assert r.returncode == 2 and "unsupported RoPE scaling type 'yarn'" in r.stderr
    # files that disagree about the scaling
    other = write_safetensors_dir(tmp_path / "lin", M, {"model.norm.weight": sd["model.norm.weight"]}, hf_config(M, rope_scaling=LINEAR4))
    r = _dry_run(server_bin, p, other)
    assert r.returncode == 2 and "disagree about RoPE" in r.stderr
