"""Automatic prefix caching without a GPU, over the fake CUDA runtime (tests/support/fake_cudart.cpp): launch plans with the
cache off and on; which pages a request matches at prompt lengths around page boundaries, on chat turns and after preemption;
eviction before preemption; prompt-logprob requests; the load_tensor refusal; a two-rank plan channel; and random workloads.
The fake runtime samples token 0 every time, so generated tokens are known here.  The GPU tests
(tests/test_prefix_cache_gpu.py) check the values a hit computes.

The scenarios run in a child pytest process that preloads the fake runtime, as in tests/test_engine_host_logic_cpu.py; they
skip themselves elsewhere."""
import contextlib
import json
import os
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_engine_host_logic_cpu as HL  # noqa: E402

INNER = os.environ.get("LLMLB_FAKE_CUDART") == "1"
inner = pytest.mark.skipif(not INNER, reason="runs in the child process that preloads the fake CUDA runtime")
TINY = HL.TINY
SWEEP = os.path.join(HERE, "support", "prefix_cache_plan_sweep.py")


# ---- launch plans ------------------------------------------------------------------------------------------------------
def _sweep(tmp_path, *args):
    log = str(tmp_path / ("_".join(args) + ".log"))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, SWEEP, *args], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "fake cudart:" not in r.stderr, r.stderr[-3000:]
    return open(log).read().splitlines(), json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("graphs", ["graphs", "eager"])
def test_prompts_without_a_shared_prefix_launch_the_same_plan_with_the_cache_on(built_lib, tmp_path, graphs):
    """Prefills 1..2048 wide and decode batches of 1, 3 and 8, every prompt distinct: the cache publishes their pages but
    nothing matches, and the plan is the cache-off plan line for line."""
    off, t_off = _sweep(tmp_path, "unique", "off", graphs)
    on, t_on = _sweep(tmp_path, "unique", "on", graphs)
    assert on == off
    assert t_on == t_off and all(c == 0 for _, c in t_on.values()), t_on


@pytest.mark.parametrize("k", [1, 2, 16])
def test_a_hit_launches_the_second_chunk_of_the_same_prompt_chunked_at_the_hit(built_lib, tmp_path, k):
    """A prompt of 64k + 37 tokens after its first 64k + 1 tokens were served: the hit covers k pages, and the request
    launches exactly the second prefill step that a cache-off engine launches for it with max_step_tokens 64k — the same
    kernels, grids and widths — after the sequence's set-up that precedes its first step, and prefills only the 37 suffix
    tokens."""
    off, t_off = _sweep(tmp_path, "shared", "off", str(k))
    on, t_on = _sweep(tmp_path, "shared", "on", str(k))
    hit = on[on.index("### P") + 1:]
    cold = off[off.index("### P") + 1:]
    assert hit[0] == cold[0] and "slot_init_kernel" in hit[0]
    assert 1 < len(hit) < len(cold) and cold[-(len(hit) - 1):] == hit[1:]
    assert t_off["P"] == [64 * k + 37, 0]
    assert t_on["P"] == [37, 64 * k] and t_on["prefix"] == [64 * k + 1, 0]


# ---- the scenarios below run in a child that preloads the fake runtime ------------------------------------------------
def test_prefix_cache_over_the_fake_cuda_runtime(built_lib):
    if INNER:
        pytest.skip("already inside")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


def _serve(eng, prompt, m=1, **kw):
    """submit, drain to LENGTH, release; returns (prefill tokens it caused, cached_tokens)"""
    t0 = eng.health()["tokens_prefill"]
    rid = eng.submit(prompt, m, ignore_eos=True, **kw)
    evs = HL.drain(eng, rid, 60)
    assert evs[-1]["finish_reason"] == HL.LENGTH, evs[-1]
    c = eng.cached_tokens(rid)
    eng.release(rid)
    HL.settle(eng)
    return eng.health()["tokens_prefill"] - t0, c


def _consistent(eng, total):
    h, s = HL.settle(eng), eng.prefix_cache_stats()
    assert h["free_kv_pages"] == h["total_kv_pages"] == total, h
    assert s["evictable_pages"] == s["cached_pages"] <= total, s    # idle: nobody holds a cached page
    return s


def _family(seed, n):
    return [(seed * 977 + 13 * j) % TINY["vocab"] for j in range(n)]


@inner
def test_scenario_matches_stop_one_token_short_and_cached_tokens_are_exact():
    """Prompt lengths around page boundaries and over several prefill steps, after an identical, a longer (fully cached) and
    a half-length (partially cached) earlier prompt served with one generated token, so that exactly its prompt's full pages
    are cached.  At most floor((n - 1) / 64) pages match, at least one token is prefilled, and cached_tokens is exact."""
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=8192, max_step_tokens=2048, prefix_cache=True) as eng:
        total = eng.health()["total_kv_pages"]
        for fam, n in enumerate((1, 63, 64, 65, 127, 128, 129, 4500)):
            for case, n_e in enumerate((n, n + 100, n // 2)):                       # identical, longer, half
                P = _family(fam * 3 + case, n + 100)
                if n_e:
                    pre, c0 = _serve(eng, P[:n_e])
                    assert c0 == 0 and pre == n_e
                pre, c = _serve(eng, P[:n])
                want = 64 * min((n - 1) // 64, n_e // 64)
                assert c == want and pre == n - want >= 1, (n, case, c, pre)
        s = _consistent(eng, total)
        assert s["hit_tokens"] > 0 and s["lookups"] > 0 and s["published_pages"] >= s["cached_pages"]


@inner
def test_scenario_chat_turn_hits_on_the_previous_reply():
    """Turn 2 = turn 1's prompt + its 100 generated ids + 50 new ids: the hit covers every full page of turn 1's context but
    the one holding its last input position — the generated tokens' pages included."""
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=2048, prefix_cache=True) as eng:
        total = eng.health()["total_kv_pages"]
        hist = _family(5, 150)
        for turn in range(4):
            m = 100
            rid = eng.submit(hist, m, ignore_eos=True)
            evs = HL.drain(eng, rid)
            gen = [e["token_id"] for e in evs if e["token_id"] >= 0]
            c = eng.cached_tokens(rid)
            eng.release(rid)
            if turn:
                assert c == 64 * (prev_end // 64), (turn, c)
                assert c > prev_prompt, (c, prev_prompt)            # reaches into the previous reply
            prev_prompt, prev_end = len(hist), len(hist) + m - 1    # positions that were inputs of launched steps
            hist = hist + gen + _family(50 + turn, 50)
        _consistent(eng, total)


@inner
def test_scenario_evicts_before_preempting_and_preempted_sequences_hit_their_own_pages():
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=14, max_step_tokens=64, prefix_cache=True) as eng:
        # warm: 14 pages of distinct prompts cached and evictable, nothing free
        for i, n in enumerate((256, 256, 256, 128)):
            _serve(eng, _family(100 + i, n))
        s = _consistent(eng, 14)
        assert s["cached_pages"] == 14
        # a load the pool holds without preemption: it runs on evicted pages
        rids = [eng.submit(_family(200 + i, 100), 60, ignore_eos=True) for i in range(4)]
        for r in rids:
            assert HL.drain(eng, r)[-1]["finish_reason"] == HL.LENGTH
            eng.release(r)
        s = _consistent(eng, 14)
        assert eng.health()["preemptions"] == 0 and s["evicted_pages"] > 0, s
        # over-subscribed: 6 sequences of 4..8 pages each on 14 pages; the youngest are preempted, they publish what they
        # computed, and on re-admission they match it (no two prompts share a page, so every hit is a sequence's own)
        lookups0, hits0 = s["lookups"], s["hit_tokens"]
        lens = [100, 350, 120, 200, 130, 300]
        eng.pause(True)
        rids = [eng.submit(_family(300 + i, n), 150, ignore_eos=True) for i, n in enumerate(lens)]
        eng.pause(False)
        for r in rids:
            evs = HL.drain(eng, r, 120)
            assert [e["index"] for e in evs] == list(range(150)) and evs[-1]["finish_reason"] == HL.LENGTH
            assert eng.cached_tokens(r) == 0
            eng.release(r)
        s = _consistent(eng, 14)
        assert eng.health()["preemptions"] > 0
        assert s["lookups"] - lookups0 > len(lens) and s["hit_tokens"] > hits0, s


@inner
def test_scenario_prompt_logprob_requests_never_hit_and_still_get_every_record():
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=1024, max_step_tokens=64, prefix_cache=True) as eng:
        P = _family(7, 300)
        _serve(eng, P)
        lookups = eng.prefix_cache_stats()["lookups"]
        t0 = eng.health()["tokens_prefill"]
        rid = eng.submit(P, 3, ignore_eos=True, logprobs=2, prompt_logprobs=True)
        evs = HL.drain(eng, rid)
        assert evs[-1]["finish_reason"] == HL.LENGTH
        assert len(eng.poll_prompt_logprobs(rid, cap=4096)) == 299
        assert eng.cached_tokens(rid) == 0 and eng.health()["tokens_prefill"] - t0 == 300
        eng.release(rid)
        assert eng.prefix_cache_stats()["lookups"] == lookups
        assert _serve(eng, P)[1] == 256                                       # it published, and a plain request hits


@inner
def test_scenario_load_tensor_is_refused_after_the_first_request_and_debug_hooks_drop_the_cache():
    import numpy as np
    ffi = HL._ffi()
    norm = np.full(TINY["hidden"], 0x3F80, dtype=np.uint16)
    for on in (False, True):
        with ffi.Engine(TINY, max_seqs=2, max_ctx=512, kv_pages=8, prefix_cache=on) as eng:
            eng.load_tensor("model.norm.weight", norm)                        # before any request: always allowed
            rid = eng.submit([1, 2, 3], 1)
            assert eng.cached_tokens(rid) == 0
            HL.drain(eng, rid)
            eng.release(rid)
            with pytest.raises(ffi.LlmlbError) if on else contextlib.nullcontext():
                eng.load_tensor("model.norm.weight", norm)
            if on:
                assert "prefix_cache" in ffi.last_error()
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.cached_tokens(10 ** 9)
            assert ei.value.code == ffi.E_NOT_FOUND
            # fill the 8-page pool with cached pages; the debug hooks need all 8 (pages_per_seq) and drop the cache
            _serve(eng, _family(1, 500))
            assert eng.prefix_cache_stats()["cached_pages"] == (7 if on else 0)
            eng.debug_prefill_logits(_family(2, 100))
            eng.debug_reset()
            assert eng.prefix_cache_stats()["cached_pages"] == 0
            assert _serve(eng, _family(1, 500))[1] == 0
            _consistent(eng, 8)


@inner
def test_scenario_scheduler_invariants_over_random_workloads_with_the_cache_on():
    """The scheduler property test's shape (hypothesis) with the cache on and prompts drawn from a few shared prefixes plus
    distinct tails, some cancelled: every surviving request gets its tokens (an engine that would write into a cached page,
    or give one page two writers, fails its step and ends the request with an error); cached_tokens is a multiple of 64 below
    the prompt; at idle every page is free or evictable and evictable == cached <= total."""
    from hypothesis import HealthCheck, given, settings, strategies as st
    ffi = HL._ffi()
    N = [0]

    @settings(max_examples=60, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
    @given(st.integers(1, 8), st.integers(6, 40), st.sampled_from([64, 128, 500, 2048]), st.sampled_from([0, 1, 3]),
           st.lists(st.tuples(st.integers(0, 3), st.integers(0, 300), st.integers(1, 200), st.integers(1, 80), st.booleans()),
                    min_size=1, max_size=14))
    def run(max_seqs, kv_pages, chunk, lookahead, reqs):
        N[0] += 1
        prompts = [(_family(f, shared) + _family(1000 + i, tail), m, c) for i, (f, shared, tail, m, c) in enumerate(reqs)]
        prompts = [(p, m, c) for p, m, c in prompts if (len(p) + m + 63) // 64 <= kv_pages and len(p) + m <= 512]
        if not prompts:
            return
        with ffi.Engine(TINY, max_seqs=max_seqs, max_ctx=512, kv_pages=kv_pages, max_step_tokens=chunk, lookahead=lookahead,
                        prefix_cache=True) as eng:
            for wave in range(2):                                                   # the second wave finds the first's pages
                eng.pause(True)
                rids = [eng.submit(p, m, ignore_eos=True) for p, m, c in prompts]
                for rid, (p, m, c) in zip(rids, prompts):
                    if c and wave == 0:
                        eng.cancel(rid)
                eng.pause(False)
                for rid, (p, m, c) in zip(rids, prompts):
                    evs = HL.drain(eng, rid, 60)
                    toks = [e for e in evs if e["token_id"] >= 0]
                    if c and wave == 0:
                        assert evs[-1]["finish_reason"] == HL.CANCELLED and not toks
                    else:
                        assert [e["index"] for e in toks] == list(range(m)) and evs[-1]["finish_reason"] == HL.LENGTH, evs[-1]
                    ct = eng.cached_tokens(rid)
                    assert ct % 64 == 0 and ct <= len(p) - 1, (ct, len(p))
                    eng.release(rid)
                _consistent(eng, kv_pages)

    run()
    assert N[0] >= 40, N


def _tp_rank(rank, world, handles, barrier, name, out_q):
    try:
        import random
        os.environ["FAKE_CUDART_STEP_US"] = "100"
        ffi = HL._ffi()
        eng = ffi.Engine(TINY, model_id="tp-pc", device=0, tp_rank=rank, tp_size=world, max_seqs=4, max_ctx=512, kv_pages=12, queue_max=32,
                         queue_timeout_ms=10, request_timeout_ms=40, seed=0, prefix_cache=True)
        handles[rank * 64:(rank + 1) * 64] = list(eng.tp_export())
        barrier.wait(60)
        blob = bytes(handles[:])
        eng.tp_import([blob[r * 64:(r + 1) * 64] for r in range(world)])
        barrier.wait(60)
        if rank == 0:
            eng.tp_plan_channel(name)
        barrier.wait(60)
        if rank != 0:
            eng.tp_plan_channel(name)
        barrier.wait(60)
        res = {}
        if rank == 0:
            rs = random.Random(5)
            live = []
            for _ in range(700):
                op = rs.randrange(10)
                try:
                    if op <= 3:
                        p = _family(rs.randrange(3), rs.choice([0, 64, 130, 200])) + _family(rs.randrange(50), rs.choice([1, 30, 65]))
                        live.append(eng.submit(p, rs.choice([1, 5, 40, 200]), ignore_eos=True, temperature=rs.choice([0.0, 0.8]),
                                               seed=rs.randrange(100)))
                    elif op <= 5 and live:
                        eng.poll(rs.choice(live), timeout_ms=rs.choice([0, 1]))
                    elif op == 6 and live:
                        eng.cancel(rs.choice(live))
                    elif op == 7 and live:
                        eng.release(live.pop(rs.randrange(len(live))))
                    elif op == 8:
                        eng.pause(rs.random() < 0.25)
                    else:
                        time.sleep(rs.choice([0, 0.001, 0.02]))
                except ffi.LlmlbError as e:
                    assert e.code in (ffi.E_QUEUE_FULL, ffi.E_INVALID_ARG, ffi.E_NOT_FOUND), e
            eng.pause(False)
            for r in live:
                eng.release(r)
            HL.settle(eng, 60)
        barrier.wait(180)
        if rank != 0:
            last, t0 = None, time.time()
            while time.time() - t0 < 30:
                cur = eng.health()["kernel_launches"]
                if cur == last:
                    break
                last = cur
                time.sleep(0.3)
        hz = eng.health()
        res["counters"] = {k: hz[k] for k in ("steps_prefill", "steps_decode", "tokens_decode", "tokens_prefill", "kernel_launches", "preemptions")}
        res["pages"] = (hz["free_kv_pages"], hz["total_kv_pages"])
        res["cache"] = eng.prefix_cache_stats()
        out_q.put((rank, res))
        barrier.wait(60)
        eng.close()
    except Exception as e:                                                      # noqa: BLE001
        import traceback
        out_q.put((rank, {"error": repr(e) + traceback.format_exc()[-800:]}))
        try:
            barrier.abort()
        except Exception:                                                       # noqa: BLE001
            pass


@inner
def test_scenario_two_rank_plan_channel_replays_the_cache_decisions():
    """The random walk of the plan-channel test (submits, polls, cancels, releases in flight, pauses, expiries, a small pool
    that forces eviction and preemption) with the cache on and prompts sharing prefixes: the follower, which sees only the
    shared-memory log, must end with the same counters, the same cache statistics and every page free or evictable."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    world = 2
    handles, barrier, q = ctx.Array("B", 64 * world), ctx.Barrier(world), ctx.Queue()
    name = "llmlb_pc_rnd_%d" % os.getpid()
    ps = [ctx.Process(target=_tp_rank, args=(r, world, handles, barrier, name, q)) for r in range(world)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=300) for _ in range(world))
    [p.join(60) for p in ps]
    assert all("error" not in v for v in got.values()), got
    lead, foll = got[0], got[1]
    assert lead["counters"] == foll["counters"], (lead["counters"], foll["counters"])
    assert lead["cache"] == foll["cache"], (lead["cache"], foll["cache"])
    assert lead["pages"] == foll["pages"] == (12, 12)
    assert lead["cache"]["hit_tokens"] > 0 and lead["counters"]["steps_decode"] > 100, lead
    assert all(p.exitcode == 0 for p in ps)
