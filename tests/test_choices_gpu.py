"""-m gpu: n choices of one prompt (llmlb_request_submit_choices) on the H100.
- kv_fork (llmlb_op_kv_fork) against torch, byte for byte: rows [0, r) of the source page land in every destination, in K
  and V, for every layer and KV head; rows r..63 of the destinations and every other page keep their poison.  The cases
  span the KV-head counts per rank of LLAMA_TINY (2), Llama-3-8B (8) and Llama-3-70B at tp 2 / 4 / 8 (4, 2, 1).
  tests/test_choices_cpu.py holds every kv_fork launch of the engine's group plans to these cases.
- A greedy group of 4 on LLAMA_TINY: every choice has the same tokens and logprob records, teacher-forced within 2 tol of
  the fp32 oracle's arg-max.
- A seeded temperature / top-k / top-p group of 4 and 8 (LLAMA_TINY and the Llama-3-8B geometry) against n lone requests
  with seeds s + i submitted together at max_step_tokens = L, to the standard of test_continuous_batching_equals_sequential:
  at most one sequence may diverge at a near-tie.  Each lone prefill is one step of the same L rows as the group's one
  prefill, but a lone step computes the lm_head of one row where the group's computes n rows at once, and past 4 rows that
  is another kernel with another summation order: the logprob values differ in their last bits and a near-tie can flip
  (one choice of eight did on an H100), so the tokens are compared.
- With the prefix cache: a group behind a cached prefix (every choice reports the 192 cached tokens, and only the 108 others
  are prefilled), and groups in an over-subscribed pool whose choices are preempted after the fork, follow the oracle.
- The whole server with n = 3 on chat and completions, streamed and not: three choices, each the greedy continuation."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from llmlb_b200 import ffi  # noqa: E402
from oracle.llama_ref import LlamaRef  # noqa: E402
from oracle.synth import synth_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
TINY = ffi.LLAMA_TINY
LOGIT_TOL = 0.03          # tests/test_engine_gpu.py: bf16 engine vs fp32 oracle on LLAMA_TINY

# (KV heads per rank, rows r, destination pages)
KV_FORK_CASES = [(nkv, r, nd) for nkv in (1, 2, 4, 8) for r in (1, 17, 40, 63) for nd in (1, 2, 7, 15)]


@pytest.mark.parametrize("nkv,r,nd", KV_FORK_CASES)
def test_kv_fork_copies_the_rows_and_touches_nothing_else(built_lib, nkv, r, nd):
    import gpu_util as G
    n_layers, n_pages = 3, nd + 5
    g = torch.Generator(device="cpu").manual_seed(nkv * 1000 + r * 20 + nd)
    shape = (n_layers, n_pages, nkv, 64, 128)
    k = torch.randint(-32768, 32767, shape, generator=g, dtype=torch.int16).to(G.dev())
    v = torch.randint(-32768, 32767, shape, generator=g, dtype=torch.int16).to(G.dev())
    src = 2
    dst = [p for p in range(n_pages) if p != src][::-1][:nd]          # unordered, the last page included
    want_k, want_v = k.clone(), v.clone()
    for p in dst:
        want_k[:, p, :, :r] = k[:, src, :, :r]
        want_v[:, p, :, :r] = v[:, src, :, :r]
    d = torch.tensor(dst, dtype=torch.int32, device=G.dev())
    G.ok(ffi.lib().llmlb_op_kv_fork(G.p(k), G.p(v), n_layers, n_pages, nkv, src, G.p(d), nd, r, G.stream_ptr()))
    G.sync()
    assert torch.equal(k, want_k) and torch.equal(v, want_v)


def _drain(e, rids, timeout_s=300):
    """{rid: (tokens, logprob records)} of requests running together, each to LENGTH"""
    outs, pending, deadline = {r: [] for r in rids}, set(rids), time.time() + timeout_s
    while pending and time.time() < deadline:
        for r in list(pending):
            for ev in e.poll_logprobs(r, timeout_ms=5):
                if ev["token_id"] >= 0:
                    outs[r].append(ev)
                if ev["finish_reason"]:
                    assert ev["finish_reason"] == ffi.FINISH_LENGTH, ev
                    pending.discard(r)
    assert not pending
    res = [([x["token_id"] for x in outs[r]], [(x["logprob"], x["top_logprobs"]) for x in outs[r]]) for r in rids]
    for r in rids:
        e.release(r)
    return res


def _tokens(e, rid):
    """one request's tokens, to LENGTH; the request is not released"""
    evs = []
    while not (evs and evs[-1]["finish_reason"]):
        evs += e.poll(rid, timeout_ms=-1)
    assert evs[-1]["finish_reason"] == ffi.FINISH_LENGTH, evs[-1]
    return [x["token_id"] for x in evs if x["token_id"] >= 0]


@pytest.fixture(scope="module")
def sd():
    return synth_state_dict(TINY, seed=0)


def _teacher_forced(sd, prompt, toks):
    ref = LlamaRef(TINY, sd)
    lg = ref.forward(prompt).numpy()[-1]
    for t in toks:
        assert lg[t] >= lg.max() - 2 * LOGIT_TOL, "token %d is not a (near-)arg-max" % t
        lg = ref.forward([t]).numpy()[-1]


def test_a_greedy_group_gives_every_choice_the_same_tokens_and_records(built_lib, sd):
    P = np.random.RandomState(11).randint(0, TINY["vocab"], 150).tolist()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, seed=0) as e:
        t0 = e.health()["tokens_prefill"]
        got = _drain(e, e.submit_choices(P, 24, 4, ignore_eos=True, logprobs=3))
        h = e.health()
        assert h["tokens_prefill"] - t0 == len(P)
        assert h["active_requests"] == 0 and h["free_kv_pages"] == h["total_kv_pages"]
    assert all(g == got[0] for g in got)
    _teacher_forced(sd, P, got[0][0])


SAMPLED = dict(temperature=0.9, top_k=40, top_p=0.95, seed=2 ** 64 - 3)   # the seeds of choices 3.. wrap


@pytest.mark.parametrize("model,n", [("tiny", 4), ("tiny", 8), ("8b", 4), ("8b", 8)])
def test_a_seeded_group_draws_what_lone_requests_with_seeds_s_plus_i_draw(built_lib, model, n):
    cfg = TINY if model == "tiny" else ffi.LLAMA3_8B
    L = 173
    P = np.random.RandomState(n + cfg["vocab"]).randint(0, cfg["vocab"], L).tolist()
    kw = dict(max_seqs=8, max_ctx=1024, max_step_tokens=L, seed=0)
    with ffi.Engine(cfg, **kw) as e:
        group = _drain(e, e.submit_choices(P, 32, n, ignore_eos=True, logprobs=2, **SAMPLED))
    with ffi.Engine(cfg, **kw) as e:
        e.pause(True)
        lone = [e.submit(P, 32, ignore_eos=True, logprobs=2, **dict(SAMPLED, seed=(SAMPLED["seed"] + i) % 2 ** 64)) for i in range(n)]
        e.pause(False)
        lone = _drain(e, lone)
    assert sum(g[0] != w[0] for g, w in zip(group, lone)) <= 1
    assert len({tuple(t) for t, _ in group}) > 1          # the choices do differ


def test_a_group_behind_a_cached_prefix_follows_the_oracle(built_lib, sd):
    P = np.random.RandomState(5).randint(0, TINY["vocab"], 300).tolist()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, seed=0, prefix_cache=True) as e:
        _drain(e, [e.submit(P[:200], 1, ignore_eos=True)])                    # caches 3 pages
        t0 = e.health()["tokens_prefill"]
        rids = e.submit_choices(P, 20, 4, ignore_eos=True)
        got = [_tokens(e, r) for r in rids]
        assert [e.cached_tokens(r) for r in rids] == [192] * 4
        assert e.health()["tokens_prefill"] - t0 == 300 - 192
        for r in rids:
            e.release(r)
        h = e.health()
        assert h["free_kv_pages"] == h["total_kv_pages"]
    for toks in got:
        _teacher_forced(sd, P, toks)


def test_groups_preempted_after_their_fork_follow_the_oracle(built_lib, sd):
    rs = np.random.RandomState(6)
    prompts = [rs.randint(0, TINY["vocab"], 90 + 40 * i).tolist() for i in range(2)]
    for cache in (False, True):
        with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=14, max_step_tokens=256, seed=0, prefix_cache=cache) as e:
            e.pause(True)
            groups = [e.submit_choices(p, 100, 3, ignore_eos=True) for p in prompts]
            e.pause(False)
            got = _drain(e, [r for g in groups for r in g])
            h = e.health()
            assert h["preemptions"] > 0 and h["free_kv_pages"] == h["total_kv_pages"], h
        for i, p in enumerate(prompts):
            for toks, _ in got[3 * i:3 * i + 3]:
                _teacher_forced(sd, p, toks)


def test_the_server_serves_three_choices_streamed_and_not(built_lib):
    import json
    import test_server_gpu as SG
    from llmlb_b200 import build
    build.build_host()
    port = SG._free_port()
    proc = subprocess.Popen([SG.BIN, "--port", str(port), "--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8",
                             "--max-ctx", "512"], stderr=subprocess.PIPE)
    try:
        deadline = time.time() + 120
        while True:
            try:
                if SG.call(port, "GET", "/v1/models")[0] == 200:
                    break
            except OSError:
                assert proc.poll() is None and time.time() < deadline, proc.stderr.read().decode()
                time.sleep(0.2)
        for route, key in (("/v1/chat/completions", "messages"), ("/v1/completions", "prompt")):
            body = {"model": "tiny-llama", "max_tokens": 12, "temperature": 0, "ignore_eos": True, "n": 3,
                    key: [{"role": "user", "content": "say something"}] if key == "messages" else "say something"}
            st, _, data = SG.call(port, "POST", route, body)
            assert st == 200, data
            b = json.loads(data)
            texts = [c["text"] if key == "prompt" else c["message"]["content"] for c in b["choices"]]
            assert [c["index"] for c in b["choices"]] == [0, 1, 2] and all(c["finish_reason"] == "length" for c in b["choices"])
            assert texts[0] == texts[1] == texts[2] and b["usage"]["completion_tokens"] == 36     # greedy: three equal choices
            st, _, data = SG.call(port, "POST", route, dict(body, stream=True, stream_options={"include_usage": True}))
            assert st == 200, data
            evs = [json.loads(l[6:]) for l in data.decode().split("\n") if l.startswith("data: ") and l != "data: [DONE]"]
            streamed = {}
            for ev in evs:
                for c in ev["choices"]:
                    piece = c["text"] if key == "prompt" else c["delta"].get("content", "")
                    streamed[c["index"]] = streamed.get(c["index"], "") + (piece or "")
            assert [streamed[i] for i in range(3)] == texts and evs[-1]["usage"]["completion_tokens"] == 36
    finally:
        proc.terminate()
        proc.wait(timeout=20)
