"""-m gpu: the prefix cache on the H100.  A hit runs the existing suffix prefill over cached context, so these tests check
the kernels at the cache's shapes: a suffix that starts on a page boundary after up to 16 cached pages, long cached context,
and several block tables pointing at the same physical pages.
- A hit computes exactly what a cold engine computes for the same prompt chunked at the hit (max_step_tokens = 64k): greedy
  tokens, logprob records and a seeded temperature / top-k / top-p draw, bit for bit, on LLAMA_TINY and the Llama-3-8B
  geometry.
- Greedy tokens after hits of 64, 128 and 1088 tokens are teacher-forced within 2 tol of the fp32 oracle's arg-max.
- 8 requests sharing a 2000-token prefix decode in one batch and give the tokens of a fresh cache-off engine serving them
  one by one, to the standard of test_continuous_batching_equals_sequential.
- An over-subscribed pool preempts sequences, which hit their own pages when they come back: every token of every sequence
  is teacher-forced within 2 tol of the oracle's arg-max (recomputes run at other step widths, so near-ties may flip and
  sequences diverge from a run without preemption)."""
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from llmlb_b200 import ffi  # noqa: E402
from oracle.llama_ref import LlamaRef  # noqa: E402
from oracle.synth import synth_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
TINY = ffi.LLAMA_TINY
LOGIT_TOL = 0.03          # tests/test_engine_gpu.py: bf16 engine vs fp32 oracle on LLAMA_TINY
SUFFIX = 37


def _run(e, prompt, m, **kw):
    """tokens and logprob records of one request, and its cached_tokens"""
    rid = e.submit(prompt, m, ignore_eos=True, **kw)
    evs = []
    while not (evs and evs[-1]["finish_reason"]):
        evs += e.poll_logprobs(rid, timeout_ms=-1)
    assert evs[-1]["finish_reason"] == ffi.FINISH_LENGTH, evs[-1]
    c = e.cached_tokens(rid)
    e.release(rid)
    evs = [x for x in evs if x["token_id"] >= 0]
    return [x["token_id"] for x in evs], [(x["logprob"], x["top_logprobs"]) for x in evs], c


REQUESTS = (dict(logprobs=5), dict(logprobs=3, temperature=0.8, top_k=50, top_p=0.9, seed=7))


@pytest.mark.parametrize("model,k", [("tiny", 1), ("tiny", 2), ("tiny", 16), ("8b", 1), ("8b", 2), ("8b", 16)])
def test_a_hit_is_bit_identical_to_the_prompt_chunked_at_the_hit(built_lib, model, k):
    cfg = TINY if model == "tiny" else ffi.LLAMA3_8B
    P = np.random.RandomState(k + cfg["vocab"]).randint(0, cfg["vocab"], 64 * k + SUFFIX).tolist()
    kw = dict(max_seqs=4, max_ctx=2048, max_step_tokens=64 * k, seed=0)
    with ffi.Engine(cfg, **kw) as a:
        cold = [_run(a, P, 16, **r) for r in REQUESTS]
    with ffi.Engine(cfg, prefix_cache=True, **kw) as b:
        _run(b, P[:64 * k + 1], 1)
        hit = [_run(b, P, 16, **r) for r in REQUESTS]
        assert b.prefix_cache_stats()["hit_tokens"] == 2 * 64 * k
    for (tc, lc, cc), (th, lh, ch) in zip(cold, hit):
        assert cc == 0 and ch == 64 * k
        assert th == tc
        assert lh == lc                    # logprob values and alternatives, bit for bit


@pytest.fixture(scope="module")
def sd():
    return synth_state_dict(TINY, seed=0)


@pytest.mark.parametrize("cached", [64, 128, 1088])
def test_tokens_after_a_hit_follow_the_oracle(built_lib, sd, cached):
    base = np.random.RandomState(cached).randint(0, TINY["vocab"], cached + 45).tolist()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=2048, seed=0, prefix_cache=True) as e:
        _run(e, base[:cached + 10], 1)                         # caches floor((cached + 10) / 64) = cached / 64 pages
        toks, _, c = _run(e, base, 24, logprobs=0)
    assert c == cached
    _teacher_forced(sd, base, toks)


def _teacher_forced(sd, prompt, toks):
    ref = LlamaRef(TINY, sd)
    lg = ref.forward(prompt).numpy()[-1]
    for t in toks:
        assert lg[t] >= lg.max() - 2 * LOGIT_TOL, "token %d is not a (near-)arg-max" % t
        lg = ref.forward([t]).numpy()[-1]


def _concurrent(e, prompts, m):
    e.pause(True)
    rids = [e.submit(p, m, ignore_eos=True) for p in prompts]
    e.pause(False)
    outs, pending, deadline = {r: [] for r in rids}, set(rids), time.time() + 300
    while pending and time.time() < deadline:
        for r in list(pending):
            for ev in e.poll(r, timeout_ms=5):
                if ev["token_id"] >= 0:
                    outs[r].append(ev["token_id"])
                if ev["finish_reason"]:
                    assert ev["finish_reason"] == ffi.FINISH_LENGTH, ev
                    pending.discard(r)
    assert not pending
    cached = [e.cached_tokens(r) for r in rids]
    assert all(len(outs[r]) == m for r in rids)
    for r in rids:
        e.release(r)
    return [outs[r] for r in rids], cached


def _sequential(prompts, m, **kw):
    with ffi.Engine(TINY, seed=0, **kw) as e:
        return [e.generate(p, m, ignore_eos=True)[0] for p in prompts]


def test_requests_sharing_a_prefix_decode_together_as_each_alone(built_lib):
    rs = np.random.RandomState(3)
    prefix = rs.randint(0, TINY["vocab"], 2000).tolist()
    prompts = [prefix + rs.randint(0, TINY["vocab"], 5 + 7 * i).tolist() for i in range(8)]
    want = _sequential(prompts, 24, max_seqs=8, max_ctx=2200)
    with ffi.Engine(TINY, max_seqs=8, max_ctx=2200, seed=0, prefix_cache=True) as e:
        _run(e, prefix + [1], 1)
        got, cached = _concurrent(e, prompts, 24)
        h = e.health()
        assert h["active_requests"] == 0 and h["free_kv_pages"] == h["total_kv_pages"]
        assert h["steps_decode"] <= 24                         # one batch of eight
    assert cached == [1984] * 8
    assert sum(g != w for g, w in zip(got, want)) <= 1         # a near-tie may flip between step widths


def test_an_oversubscribed_pool_with_the_cache_follows_the_oracle(built_lib, sd):
    rs = np.random.RandomState(4)
    prefix = rs.randint(0, TINY["vocab"], 600).tolist()
    prompts = [prefix + rs.randint(0, TINY["vocab"], 20 + 5 * i).tolist() for i in range(8)]
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=24, max_step_tokens=256, seed=0, prefix_cache=True) as e:
        got, _ = _concurrent(e, prompts, 120)
        h, s = e.health(), e.prefix_cache_stats()
        assert h["preemptions"] > 0 and s["hit_tokens"] > 0, (h, s)
        assert h["active_requests"] == 0 and h["free_kv_pages"] == h["total_kv_pages"]
    for p, toks in zip(prompts, got):
        _teacher_forced(sd, p, toks)
