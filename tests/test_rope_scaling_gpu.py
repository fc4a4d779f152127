"""-m gpu: RoPE frequency scaling on the H100 — the scaled RoPE table against fp64, the attention kernels at 32K-128K
contexts (where llama3-scaled models are served) against fp64 on poisoned pages, engine parity with llama3 scaling
across the 8192-token original context and at a 120K-token context, and the server serving a Llama 3.1-style GGUF and
a safetensors directory with config.json exactly as the engine does with the same factors."""
import http.client
import json
import os
import socket
import subprocess
import time

import numpy as np
import pytest
import torch

import test_kernels_sm90_gpu as K9
from llmlb_b200 import ffi
from rope_oracle import ScaledLlamaRef as LlamaRef, rope_freq_factors
from oracle.synth import synth_state_dict
from rope_scaling_util import LINEAR4, LLAMA31_8B, THETA, convert_rope_factors, hf_config, write_llama_gguf, write_safetensors_dir

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TINY = ffi.LLAMA_TINY
LOGIT_TOL = 0.03          # tests/test_engine_gpu.py: bf16 engine vs the fp32 oracle


@pytest.fixture(scope="module")
def L(built_lib):
    return ffi.lib()


def _f32(x):
    return (ffi.f32 * 64)(*[float(v) for v in x])


# ---- 1. the RoPE table ----
TABLE_POS = [0, 1, 8191, 8192, 65535, 131071]


@pytest.mark.parametrize("kind", ["llama3", "linear", "none"])
def test_scaled_rope_table_against_fp64(L, kind):
    from gpu_util import ok, p, stream_ptr, sync
    n = 131072
    f = {"llama3": rope_freq_factors(LLAMA31_8B, THETA), "linear": rope_freq_factors(LINEAR4, THETA), "none": None}[kind]
    f32 = None if f is None else f.astype(np.float32)
    tab = torch.empty(n, 64, 2, dtype=torch.float32, device="cuda")
    ok(L.llmlb_op_rope_table_scaled(p(tab), n, THETA, None if f32 is None else _f32(f32), stream_ptr()))
    sync()
    inv = 1.0 / (np.float64(np.float32(THETA)) ** (np.arange(0, 128, 2, dtype=np.float64) / 128))
    if f32 is not None:
        inv = inv / f32.astype(np.float64)
    got = tab[TABLE_POS].cpu().numpy()
    ang = np.array(TABLE_POS, dtype=np.float64)[:, None] * inv[None, :]
    # fp64 angles rounded once to fp32: one fp32 ulp (2^-24 near 1) for a last-bit difference of pow / cos in fp64
    assert np.abs(got[..., 0] - np.cos(ang).astype(np.float32)).max() <= 2.0 ** -24
    assert np.abs(got[..., 1] - np.sin(ang).astype(np.float32)).max() <= 2.0 ** -24
    if f is not None:   # the scaled table really differs from the plain one where the divisors are not 1
        plain = torch.empty_like(tab)
        ok(L.llmlb_op_rope_table(p(plain), n, THETA, stream_ptr()))
        sync()
        assert not torch.equal(plain[8192], tab[8192])


def test_unit_factors_are_byte_identical_to_the_plain_table(L):
    from gpu_util import ok, p, stream_ptr, sync
    n = 131072
    a, b, c = (torch.full((n, 64, 2), float("nan"), dtype=torch.float32, device="cuda") for _ in range(3))
    ok(L.llmlb_op_rope_table(p(a), n, THETA, stream_ptr()))
    ok(L.llmlb_op_rope_table_scaled(p(b), n, THETA, _f32([1.0] * 64), stream_ptr()))
    ok(L.llmlb_op_rope_table_scaled(p(c), n, THETA, None, stream_ptr()))
    sync()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)) and torch.equal(a.view(torch.int32), c.view(torch.int32))
    bad = [1.0] * 64
    bad[3] = 0.0
    assert L.llmlb_op_rope_table_scaled(p(a), n, THETA, _f32(bad), stream_ptr()) == ffi.E_INVALID_ARG


# ---- 2. attention kernels at long contexts (the harness of test_kernels_sm90_gpu.py) ----
LONG_DECODE_LENS = [32768, 131072, 65]


@pytest.mark.parametrize("nh,nkv", [(8, 2), (32, 8)])
@pytest.mark.parametrize("splits", K9.DECODE_SPLITS)
def test_decode_attention_at_long_contexts_against_fp64(L, splits, nh, nkv):
    """Decode attention over 32K and 128K contexts on poisoned pages (cluster of 2-16 CTAs, 1 = the tensor-core kernel),
    with an identity RoPE table so that the q and k the kernel uses are the bf16 inputs."""
    from gpu_util import ok, p, stream_ptr, sync
    seed = 7000 + splits * 10 + nkv
    lens = LONG_DECODE_LENS
    pages = K9._Pages(nkv, lens, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    Kc = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
    Vc = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
    for i, n in enumerate(lens):
        pages.write(i, 0, Kc[i], Vc[i])
    rope = torch.zeros(max(lens) + 1, 64, 2, dtype=torch.float32, device="cuda")
    rope[..., 0] = 1
    ws = torch.zeros(L.llmlb_op_decode_attention_ws(len(lens), nh, splits), dtype=torch.uint8, device="cuda")
    p_round = K9.BF16_U if splits == 1 else 0.0
    ratio = 0.0
    for scale in (1, 16):
        B = len(lens)
        qkv = K9._qkv_rows(B, nh, nkv, scale, gen)
        seq_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
        bt_rows = torch.arange(B, dtype=torch.int32, device="cuda")
        out = K9._Out(B, nh * 128, torch.bfloat16, pad=0)
        ok(L.llmlb_op_decode_attention(p(qkv), p(pages.kp), p(pages.vp), p(pages.bt), pages.bt_stride, p(bt_rows), p(seq_lens), B,
                                       out.ptr(), nh, nkv, p(rope), splits, B, p(ws), stream_ptr()))
        sync()
        assert out.untouched_outside(1) == 0
        for b, n in enumerate(lens):
            row = qkv[b]
            q = row[: nh * 128].view(1, nh, 128)
            kn = row[nh * 128:(nh + nkv) * 128].view(1, nkv, 128)
            vn = row[(nh + nkv) * 128:].view(1, nkv, 128)
            k, v = torch.cat([Kc[b], kn]), torch.cat([Vc[b], vn])
            ref, bound = K9.attention_ref(q, k, v, torch.tensor([n - 1], device="cuda"), p_round)
            ratio = max(ratio, K9._attn_check(out.slot(0)[b].view(1, nh, 128), ref, bound, "len %d scale %d" % (n, scale)))
    K9._report("decode long", ratio)


@pytest.mark.parametrize("nh,nkv", [(8, 2), (8, 1)])
@pytest.mark.parametrize("impl", K9.PREFILL_IMPLS)
def test_prefill_attention_q_tiles_past_100k_against_fp64(L, impl, nh, nkv):
    """Prefill q tiles at positions above 100K over a cached context that long: one sequence whose chunk starts at
    100003 (mid-page), one that ends at 131072; tiles listed out of order."""
    from gpu_util import ok, p, stream_ptr, sync
    call = [(0, 100003, 200), (1, 131072 - 130, 130)]
    seed = 9100 + nh + nkv
    horizons = [pos0 + n for _, pos0, n in call]
    pages = K9._Pages(nkv, horizons, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    K = [torch.randn(h, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for h in horizons]
    V = [torch.randn(h, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for h in horizons]
    for i, h in enumerate(horizons):
        pages.write(i, 0, K[i], V[i])
    tile = 128 if impl == "tc" else 64
    T = sum(n for _, _, n in call)
    ratio = 0.0
    for scale in (1, 16):
        qkv = K9._qkv_rows(T, nh, nkv, scale, gen)
        tiles, row0 = [], 0
        for i, pos0, n in call:
            for j in range(0, n, tile):
                tiles.append([row0 + j, min(tile, n - j), pos0 + j, i])
            row0 += n
        order = torch.randperm(len(tiles), generator=torch.Generator().manual_seed(seed + scale)).tolist()
        tiles_t = torch.tensor([tiles[k] for k in order], dtype=torch.int32, device="cuda")
        out = K9._Out(T, nh * 128, torch.bfloat16, pad=0)
        if impl == "tc":
            ok(L.llmlb_op_prefill_attention_tc(p(qkv), T, p(pages.kp), p(pages.vp), pages.n_pages, p(pages.bt), pages.bt_stride,
                                               p(tiles_t), len(tiles), out.ptr(), nh, nkv, stream_ptr()))
        else:
            ok(L.llmlb_op_prefill_attention(p(qkv), p(pages.kp), p(pages.vp), p(pages.bt), pages.bt_stride, p(tiles_t), len(tiles),
                                            out.ptr(), nh, nkv, stream_ptr()))
        sync()
        assert out.untouched_outside(1) == 0
        row0 = 0
        for i, pos0, n in call:
            for r0 in range(0, n, 32):      # the fp64 reference in row blocks: [nh, rows, 131072] doubles at a time
                r1 = min(n, r0 + 32)
                q = qkv[row0 + r0: row0 + r1, : nh * 128].view(r1 - r0, nh, 128)
                ref, bound = K9.attention_ref(q, K[i], V[i], torch.arange(pos0 + r0, pos0 + r1, device="cuda"), K9.BF16_U)
                got = out.slot(0)[row0 + r0: row0 + r1].view(r1 - r0, nh, 128)
                ratio = max(ratio, K9._attn_check(got, ref, bound, "%s sequence %d rows %d.. scale %d" % (impl, i, pos0 + r0, scale)))
            row0 += n
    K9._report("prefill long " + impl, ratio)


# ---- 3. engine parity with llama3 scaling ----
def _llama31_factors():
    return rope_freq_factors(LLAMA31_8B, THETA).astype(np.float32)


def _oracle_chunked(ref, prompt, chunk=1024):
    out = [ref.forward(prompt[i: i + chunk]).numpy() for i in range(0, len(prompt), chunk)]
    return np.concatenate(out)


def test_engine_parity_across_the_original_context_with_llama3_scaling(built_lib):
    """The tiny 2-layer model, a 9000-token prompt: one-shot prefill logits at every position and 16 teacher-forced decode
    steps against the fp32 oracle; then the same prompt through the request path (chunked prefill, 2048-token steps,
    crossing 8192) and 16 greedy tokens that must each be a (near-)arg-max of the oracle."""
    f = _llama31_factors()
    cfg = dict(TINY, rope_scaling=LLAMA31_8B)
    sd = synth_state_dict(TINY, seed=21)
    prompt = np.random.RandomState(9000).randint(0, TINY["vocab"], 9000).tolist()
    ref = LlamaRef(cfg, sd)
    rl = _oracle_chunked(ref, prompt)
    with ffi.Engine(TINY, max_seqs=2, max_ctx=9216, max_step_tokens=9024, seed=21, rope_freq_factors=f) as eng:
        last, full = eng.debug_prefill_logits(prompt, all_positions=True)
        err = np.abs(full - rl).max(1)
        assert err.max() < LOGIT_TOL, (int(err.argmax()), float(err.max()))
        lg = last
        for _ in range(16):
            t = int(np.argmax(lg))
            lg = eng.debug_decode_logits(t)
            r = ref.forward([t]).numpy()[-1]
            assert np.abs(lg - r).max() < LOGIT_TOL
    # unscaled, the same engine misses the oracle at long positions: the factors are what makes it agree
    plain = LlamaRef(TINY, sd)
    assert np.abs(_oracle_chunked(plain, prompt)[-64:] - rl[-64:]).max() > 3 * LOGIT_TOL
    with ffi.Engine(TINY, max_seqs=2, max_ctx=9216, seed=21, rope_freq_factors=f) as eng:
        toks, _ = eng.generate(prompt, 16, ignore_eos=True)
    ref = LlamaRef(cfg, sd)
    lg = _oracle_chunked(ref, prompt)[-1]
    for t in toks:
        assert lg[t] >= lg.max() - 2 * LOGIT_TOL
        lg = ref.forward([t]).numpy()[-1]


def test_engine_parity_at_120k_context_one_layer(built_lib):
    """A one-layer model at max_ctx 131072: a 120000-token prompt prefilled in one step, last-position logits and 8
    teacher-forced decode steps against the oracle's one-layer tail path (K/V everywhere, queries only where checked)."""
    M = dict(TINY, n_layers=1)
    f = _llama31_factors()
    sd = synth_state_dict(M, seed=33)
    n = 120000
    prompt = np.random.RandomState(120).randint(0, M["vocab"], n).tolist()
    ref = LlamaRef(dict(M, rope_scaling=LLAMA31_8B), sd)
    rl = ref.forward_tail(prompt, 4).numpy()
    with ffi.Engine(M, max_seqs=1, max_ctx=131072, max_step_tokens=n, seed=33, rope_freq_factors=f) as eng:
        last = eng.debug_prefill_logits(prompt)
        assert np.abs(last - rl[-1]).max() < LOGIT_TOL
        lg = last
        for _ in range(8):
            t = int(np.argmax(lg))
            lg = eng.debug_decode_logits(t)
            assert np.abs(lg - ref.forward([t]).numpy()[-1]).max() < LOGIT_TOL


# ---- 4. end to end through the server ----
BIN = os.path.join(os.path.dirname(HERE), "llmlb_b200", "llmlb_b200_server")


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    return port


def _byte_detok(t):
    """The server's text for a token id when it has no tokenizer (gateway.cpp byte_detokenize)."""
    if 3 <= t < 259:
        c = t - 3
        if c < 0x80 and (c >= 0x20 or c in (0x0A, 0x09)):
            return chr(c)
    return "<|%d|>" % t


def _serve_completion(weights, prompt, n_new):
    port = _free_port()
    proc = subprocess.Popen([BIN, "--port", str(port), "--model", "auto", "--model-id", "scaled", "--max-seqs", "2", "--max-ctx", "8192",
                             "--weights", str(weights)], stderr=subprocess.PIPE)
    try:
        deadline = time.time() + 120
        while time.time() < deadline:
            try:
                c = http.client.HTTPConnection("127.0.0.1", port, timeout=2); c.request("GET", "/v1/models"); c.getresponse().read(); c.close()
                break
            except OSError:
                assert proc.poll() is None, proc.stderr.read().decode()
                time.sleep(0.2)
        c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
        c.request("POST", "/v1/completions", json.dumps({"model": "scaled", "prompt_token_ids": prompt, "max_tokens": n_new, "temperature": 0,
                                                         "ignore_eos": True}), {"Content-Type": "application/json"})
        r = c.getresponse()
        body = r.read()
        c.close()
        assert r.status == 200, body
        return json.loads(body)["choices"][0]["text"]
    finally:
        proc.terminate()
        proc.wait(timeout=20)


def test_server_serves_scaled_checkpoints_like_the_engine(built_lib, tmp_path):
    pytest.importorskip("gguf")
    from llmlb_b200 import build
    from rope_scaling_util import native_ckpt, native_open
    build.build_host()
    sd = synth_state_dict(TINY, seed=44)
    prompt = np.random.RandomState(6000).randint(0, TINY["vocab"], 6000).tolist()
    n_new = 16
    g = tmp_path / "llama31.gguf"
    gf = convert_rope_factors(LLAMA31_8B)
    write_llama_gguf(g, TINY, sd, rope_freqs=gf)
    st = write_safetensors_dir(tmp_path / "st", TINY, sd, hf_config(TINY, rope_scaling=LLAMA31_8B))
    _, sf = native_open(native_ckpt(build.build_host()), st)

    def engine_text(factors):
        with ffi.Engine(TINY, max_seqs=2, max_ctx=8192, seed=44, rope_freq_factors=factors) as eng:
            toks, _ = eng.generate(prompt, n_new, ignore_eos=True)
        return "".join(_byte_detok(t) for t in toks)

    plain = engine_text(None)
    for weights, factors in ((g, gf), (st, sf)):
        want = engine_text(factors)
        assert want != plain                                     # the factors change the answer at these positions
        assert _serve_completion(weights, prompt, n_new) == want
