"""n choices of one prompt (llmlb_request_submit_choices) without a GPU, over the fake CUDA runtime
(tests/support/fake_cudart.cpp), which samples token 0 every time:
- launch plans (tests/support/choices_plan_sweep.py): n = 1 launches line for line what the matching single-request submit
  launches, with the prefix cache off and on; a group of n prefills its prompt once, samples n rows in that step, launches
  one kv_fork (none when the prompt fills its last page) and decodes n wide; every kv_fork launch class (KV heads per rank,
  rows, destinations) is one tests/test_choices_gpu.py launches;
- llmlb_op_kv_fork refuses out-of-range arguments, fuzzed as tests/support/op_fuzz.py fuzzes the other entry points;
- the scheduler: pages taken at admission, pages returned at release, cancels and preemptions before and after the fork,
  argument checks, queue accounting, a two-rank plan channel and random workloads mixing groups with single requests.
The scenarios run in a child pytest process that preloads the fake runtime, as in tests/test_engine_host_logic_cpu.py."""
import json
import os
import random
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
SWEEP = os.path.join(HERE, "support", "choices_plan_sweep.py")


def _sweep(tmp_path, *args):
    log = str(tmp_path / ("_".join(args) + ".log"))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, SWEEP, *args], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "fake cudart:" not in r.stderr, r.stderr[-3000:]
    return open(log).read().splitlines(), json.loads(r.stdout.strip().splitlines()[-1])


def _sections(lines):
    out, cur = {}, None
    for l in lines:
        if l.startswith("### "):
            cur = l[4:]
            out[cur] = []
        elif cur is not None:
            out[cur].append(l.split())
    return out


def _name(p):
    import test_kernel_coverage_cpu as KC
    return KC.short_name(p[0])


@pytest.mark.parametrize("cache", ["off", "on"])
def test_one_choice_launches_what_the_matching_submit_launches(built_lib, tmp_path, cache):
    a, ta = _sweep(tmp_path, "one", "submit", cache)
    b, tb = _sweep(tmp_path, "one", "choices", cache)
    assert b == a and tb == ta
    assert not any("kv_fork" in l for l in b)


@pytest.fixture(scope="module")
def group_plans(built_lib, tmp_path_factory):
    t = tmp_path_factory.mktemp("choices")
    return {c: _sweep(t, "group", c) for c in ("off", "on")}


@pytest.mark.parametrize("cache", ["off", "on"])
def test_a_group_prefills_once_samples_n_rows_forks_once_and_decodes_n_wide(group_plans, cache):
    lines, tot = group_plans[cache]
    for sec, launches in _sections(lines).items():
        L, n = (int(x.split("=")[1]) for x in sec.split())
        assert tot[sec] == [L, 1, 3], (sec, tot[sec])                      # L prefill tokens in one step, 3 decode steps
        names = [_name(p) for p in launches]
        gathers = [p for p in launches if _name(p) == "gather_rows_kernel"]
        assert len(gathers) == 1 and int(gathers[0][1]) == n, sec          # the last row, gathered n times
        samples = [int(p[1]) for p in launches if _name(p) == "sample_kernel"]
        assert samples == [n] * 4, (sec, samples)                          # the prefill step's n rows, then n-wide decodes
        forks = [p for p in launches if _name(p) == "kv_fork_kernel"]
        assert len(forks) == (1 if L % 64 else 0), sec
        if forks:   # after the prefill's forward, the sampler and the copies of the step's ids
            assert names.index("kv_fork_kernel") > names.index("sample_kernel")
            assert forks[0][1:3] == ["16", "2"]                             # 2 x 8 KV heads, 2 layers


def test_every_kv_fork_launch_class_of_the_group_plans_is_gpu_tested(group_plans):
    import test_choices_gpu as CG
    seen = set()
    for lines, _ in group_plans.values():
        for sec, launches in _sections(lines).items():
            L, n = (int(x.split("=")[1]) for x in sec.split())
            for p in launches:
                if _name(p) == "kv_fork_kernel":
                    seen.add((int(p[1]) // 2, L % 64, n - 1))
    assert seen and seen <= set(CG.KV_FORK_CASES), seen - set(CG.KV_FORK_CASES)


def test_kv_fork_refuses_out_of_range_arguments_and_survives_fuzzing(built_lib, tmp_path):
    code = r"""
import ctypes as C, random, sys
sys.path.insert(0, %r)
from llmlb_b200 import ffi
L = ffi.lib()
cu = C.CDLL("libcudart.so.12")
cu.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
def dm(n):
    p = C.c_void_p(); assert cu.cudaMalloc(C.byref(p), n) == 0; return p
BIG = [dm(1 << 32) for _ in range(3)]
E = ffi.E_INVALID_ARG
k, v, d = BIG
assert L.llmlb_op_kv_fork(k, v, 2, 10, 8, 3, d, 4, 17, None) == 0
for args in ((None, v, 2, 10, 8, 3, d, 4, 17), (k, None, 2, 10, 8, 3, d, 4, 17), (k, v, 2, 10, 8, 3, None, 4, 17),
             (k, v, 0, 10, 8, 3, d, 4, 17), (k, v, 65536, 10, 8, 3, d, 4, 17), (k, v, 2, 0, 8, 3, d, 4, 17),
             (k, v, 2, 10, 0, 3, d, 4, 17), (k, v, 2, 10, 257, 3, d, 4, 17), (k, v, 2, 10, 8, 10, d, 4, 17),
             (k, v, 2, 10, 8, -1, d, 4, 17), (k, v, 2, 10, 8, 3, d, 0, 17), (k, v, 2, 10, 8, 3, d, 1025, 17),
             (k, v, 2, 10, 8, 3, d, 4, 0), (k, v, 2, 10, 8, 3, d, 4, 65), (k, v, 80, 1 << 20, 8, 3, d, 4, 17)):
    assert L.llmlb_op_kv_fork(*args, None) == E, args
    assert "llmlb_op_kv_fork" in ffi.last_error()
INTS = [0, 1, 2, 3, 7, 8, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 65535, 65536, 1 << 20, (1 << 31) - 1, (1 << 32) - 1]
rs = random.Random(int(sys.argv[1]))
hist = {}
for _ in range(4000):
    ptr = lambda: rs.choice(BIG) if rs.random() < 0.93 else None
    rc = L.llmlb_op_kv_fork(ptr(), ptr(), rs.choice(INTS), rs.choice(INTS), rs.choice(INTS),
                            rs.choice([-5, -1, 0, 1, 7, 1023, 1 << 20, (1 << 31) - 1]), ptr(), rs.choice(INTS), rs.choice(INTS), None)
    assert rc in (0, E), rc
    hist[rc] = hist.get(rc, 0) + 1
assert len(hist) == 2, hist
print("ok", sorted(hist.items()))
""" % ROOT
    f = tmp_path / "kv_fork_fuzz.py"
    f.write_text(code)
    env = dict(os.environ, LD_PRELOAD=HL.build_fake())
    for seed in (1, 2):
        r = subprocess.run([sys.executable, str(f), str(seed)], env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
        assert "fake cudart:" not in r.stderr, r.stderr[-2000:]


# ---- the scenarios below run in a child that preloads the fake runtime ------------------------------------------------
def test_choices_over_the_fake_cuda_runtime(built_lib):
    if INNER:
        pytest.skip("already inside")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


def _family(seed, n):
    return [(seed * 977 + 13 * j) % TINY["vocab"] for j in range(n)]


def _drain_all(eng, rids, timeout_s=60):
    return [HL.drain(eng, r, timeout_s) for r in rids]


def _idle(eng, total):
    h = HL.settle(eng)
    assert h["free_kv_pages"] == h["total_kv_pages"] == total, h
    return h


def _admission_pages(L, n):
    return (L + 63) // 64 + (n - 1) * (L % 64 != 0)


@inner
@pytest.mark.parametrize("cache", [False, True])
def test_scenario_pages_taken_at_admission_follow_the_formula_and_all_come_back(cache):
    """A group of n over L prompt tokens is admitted into a pool of exactly ceil(L/64) + (n-1) [L mod 64 != 0] pages, and
    not into one page less; one token out needs no further page.  After release every page is free."""
    ffi = HL._ffi()
    for L in (1, 63, 64, 65, 127, 128, 1000):
        for n in (2, 3, 8):
            need = _admission_pages(L, n)
            floor = (L + 1 + 63) // 64                     # the pool a lone request of L + 1 tokens needs at submit
            with ffi.Engine(TINY, max_seqs=8, max_ctx=2048, kv_pages=max(need, floor), prefix_cache=cache) as eng:
                t0 = eng.health()["tokens_prefill"]
                evs = _drain_all(eng, eng.submit_choices(_family(L, L), 1, n, ignore_eos=True))
                assert all(e[-1]["finish_reason"] == HL.LENGTH and e[0]["token_id"] == 0 for e in evs), (L, n)
                assert eng.health()["tokens_prefill"] - t0 == L
                _idle(eng, max(need, floor))
            if need - 1 < floor:
                continue
            with ffi.Engine(TINY, max_seqs=8, max_ctx=2048, kv_pages=need - 1, prefix_cache=cache) as eng:
                rids = eng.submit_choices(_family(L, L), 1, n, ignore_eos=True)
                time.sleep(0.05)
                h = eng.health()
                assert h["queued_requests"] == n and h["active_requests"] == 0 and h["tokens_prefill"] == 0, (L, n, h)
                eng.pause(True)                            # a smaller group would fit: cancel all of them at once
                for r in rids:
                    eng.cancel(r)
                eng.pause(False)
                assert all(e[-1]["finish_reason"] == HL.CANCELLED for e in _drain_all(eng, rids))
                _idle(eng, need - 1)


@inner
def test_scenario_argument_checks_and_queue_accounting():
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=512, queue_max=6) as eng:
        for n in (0, 5):
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.submit_choices([1, 2, 3], 4, n)
            assert ei.value.code == ffi.E_INVALID_ARG and "n must be in [1, max_seqs = 4]" in ffi.last_error()
        for lp in (-2, 21):
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.submit_choices([1, 2, 3], 4, 2, logprobs=lp)
            assert ei.value.code == ffi.E_INVALID_ARG and "top_logprobs" in ffi.last_error()
        eng.pause(True)
        a = eng.submit_choices([1, 2, 3], 4, 4, ignore_eos=True)
        assert a == list(range(a[0], a[0] + 4)) and eng.health()["queued_requests"] == 4
        with pytest.raises(ffi.LlmlbError) as ei:
            eng.submit_choices([1, 2, 3], 4, 3)                    # 4 + 3 > queue_max 6
        assert ei.value.code == ffi.E_QUEUE_FULL
        b = eng.submit_choices([1, 2, 3], 4, 2, ignore_eos=True)
        eng.pause(False)
        for evs in _drain_all(eng, a + b):
            assert [e["index"] for e in evs] == list(range(4)) and evs[-1]["finish_reason"] == HL.LENGTH
        for r in a + b:
            eng.release(r)
        _idle(eng, eng.health()["total_kv_pages"])


@inner
@pytest.mark.parametrize("cache", [False, True])
def test_scenario_cancelling_one_choice_never_ends_another(cache):
    """Cancelled while queued, while its group is still prefilling (the choice that prefills for the group included: the
    next one takes over its pages), and after the fork: the cancelled choice ends CANCELLED, with no token before the fork,
    and every other choice runs to LENGTH with all its tokens."""
    ffi = HL._ffi()
    L, m = 6000, 40
    with ffi.Engine(TINY, max_seqs=8, max_ctx=8192, max_step_tokens=64, prefix_cache=cache) as eng:
        total = eng.health()["total_kv_pages"]
        # queued
        eng.pause(True)
        rids = eng.submit_choices(_family(1, 300), m, 3, ignore_eos=True)
        eng.cancel(rids[0])
        eng.pause(False)
        evs = _drain_all(eng, rids)
        assert evs[0][-1]["finish_reason"] == HL.CANCELLED and all(e["token_id"] < 0 for e in evs[0])
        assert all([e["index"] for e in x] == list(range(m)) and x[-1]["finish_reason"] == HL.LENGTH for x in evs[1:])
        [eng.release(r) for r in rids]
        _idle(eng, total)
        # during the group's prefill (94 steps of 64 tokens): pause there, cancel the prefilling choice and one other
        caught = 0
        for attempt in range(6):
            rids = eng.submit_choices(_family(2 + attempt, L), m, 4, ignore_eos=True)
            while eng.health()["tokens_prefill"] % L == 0 and not eng.poll(rids[0], timeout_ms=0):
                pass
            eng.pause(True)
            pre = eng.health()["tokens_prefill"] % L != 0
            eng.cancel(rids[0])
            eng.cancel(rids[2])
            eng.pause(False)
            evs = _drain_all(eng, rids)
            for i, x in enumerate(evs):
                if i in (0, 2):
                    assert x[-1]["finish_reason"] == HL.CANCELLED
                    if pre:
                        assert all(e["token_id"] < 0 for e in x)
                else:
                    assert [e["index"] for e in x if e["token_id"] >= 0] == list(range(m)) and x[-1]["finish_reason"] == HL.LENGTH
            caught += pre
            [eng.release(r) for r in rids]
            _idle(eng, total)
            if caught:
                break
        assert caught, "never paused inside the group's prefill"
        # after the fork: the first token of every choice is out
        rids = eng.submit_choices(_family(9, 200), 4000, 3, ignore_eos=True)
        while not eng.poll(rids[1], timeout_ms=50):
            pass
        eng.pause(True)
        eng.cancel(rids[1])
        eng.pause(False)
        evs = _drain_all(eng, rids)
        assert evs[1][-1]["finish_reason"] == HL.CANCELLED
        assert all(x[-1]["finish_reason"] == HL.LENGTH for i, x in enumerate(evs) if i != 1)
        [eng.release(r) for r in rids]
        _idle(eng, total)


@inner
@pytest.mark.parametrize("cache", [False, True])
def test_scenario_an_oversubscribed_pool_preempts_choices_and_every_choice_completes(cache):
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=14, max_step_tokens=128, prefix_cache=cache) as eng:
        eng.pause(True)
        groups = [eng.submit_choices(_family(i, 90 + 40 * i), 150, 3, ignore_eos=True) for i in range(2)]
        single = eng.submit(_family(7, 70), 150, ignore_eos=True)
        eng.pause(False)
        for evs in _drain_all(eng, [r for g in groups for r in g] + [single], 120):
            assert [e["index"] for e in evs] == list(range(150)) and evs[-1]["finish_reason"] == HL.LENGTH
        assert eng.health()["preemptions"] > 0
        for r in [r for g in groups for r in g] + [single]:
            eng.release(r)
        _idle(eng, 14)


@inner
def test_scenario_every_choice_delivers_the_prompt_records_and_the_cached_tokens():
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, max_step_tokens=64, prefix_cache=True) as eng:
        P = _family(3, 300)
        _drain_all(eng, [eng.submit(P[:200], 1, ignore_eos=True)])
        rids = eng.submit_choices(P, 5, 3, ignore_eos=True, logprobs=2, prompt_logprobs=True)
        _drain_all(eng, rids)
        recs = [eng.poll_prompt_logprobs(r, cap=4096) for r in rids]
        assert len(recs[0]) == 299 and recs[1] == recs[0] and recs[2] == recs[0]
        assert [eng.cached_tokens(r) for r in rids] == [0, 0, 0]          # prompt records need every prompt row
        t0 = eng.health()["tokens_prefill"]
        rids2 = eng.submit_choices(P, 5, 4, ignore_eos=True)
        _drain_all(eng, rids2)
        assert [eng.cached_tokens(r) for r in rids2] == [256] * 4 and eng.health()["tokens_prefill"] - t0 == 300 - 256
        for r in rids + rids2:
            eng.release(r)
        _idle(eng, eng.health()["total_kv_pages"])


@inner
def test_scenario_scheduler_invariants_over_random_workloads_with_groups():
    """test_scenario_scheduler_invariants_over_random_workloads' shape with groups of 2..max_seqs choices mixed into the
    single requests, shared prompt prefixes, the cache off and on, cancels, and pools small enough to preempt: every
    surviving choice gets its tokens in order and ends LENGTH (an engine that would write into a page another sequence holds
    fails its step and ends the request with an error); a cancelled one ends CANCELLED; at idle every page is free."""
    from hypothesis import HealthCheck, given, settings, strategies as st
    ffi = HL._ffi()
    N = [0]

    @settings(max_examples=50, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
    @given(st.integers(2, 8), st.integers(8, 40), st.sampled_from([64, 128, 500]), st.sampled_from([0, 1, 3]), st.booleans(),
           st.lists(st.tuples(st.integers(0, 2), st.integers(0, 200), st.integers(1, 150), st.integers(1, 60), st.integers(1, 8),
                              st.booleans()), min_size=1, max_size=10))
    def run(max_seqs, kv_pages, chunk, lookahead, cache, reqs):
        N[0] += 1
        work = []
        for i, (f, shared, tail, m, n, c) in enumerate(reqs):
            p = _family(f, shared) + _family(1000 + i, tail)
            n = min(n, max_seqs)
            if (len(p) + m + 63) // 64 > kv_pages or len(p) + m > 512 or _admission_pages(len(p), n) > kv_pages:
                continue
            work.append((p, m, n, c))
        if not work:
            return
        with ffi.Engine(TINY, max_seqs=max_seqs, max_ctx=512, kv_pages=kv_pages, max_step_tokens=chunk, lookahead=lookahead,
                        prefix_cache=cache) as eng:
            eng.pause(True)
            ids = [eng.submit_choices(p, m, n, ignore_eos=True) if n > 1 else [eng.submit(p, m, ignore_eos=True)]
                   for p, m, n, c in work]
            for rids, (p, m, n, c) in zip(ids, work):
                if c:
                    eng.cancel(rids[-1])
            eng.pause(False)
            for rids, (p, m, n, c) in zip(ids, work):
                for j, rid in enumerate(rids):
                    evs = HL.drain(eng, rid, 60)
                    toks = [e for e in evs if e["token_id"] >= 0]
                    if c and j == len(rids) - 1:
                        assert evs[-1]["finish_reason"] == HL.CANCELLED and not toks
                    else:
                        assert [e["index"] for e in toks] == list(range(m)) and evs[-1]["finish_reason"] == HL.LENGTH, evs[-1]
                    eng.release(rid)
            _idle(eng, kv_pages)

    run()
    assert N[0] >= 30, N


def _tp_rank(rank, world, handles, barrier, name, out_q):
    try:
        os.environ["FAKE_CUDART_STEP_US"] = "100"
        ffi = HL._ffi()
        eng = ffi.Engine(TINY, model_id="tp-n", device=0, tp_rank=rank, tp_size=world, max_seqs=6, max_ctx=512, kv_pages=14, queue_max=40,
                         queue_timeout_ms=10, request_timeout_ms=60, seed=0, prefix_cache=True)
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
            rs = random.Random(9)
            live = []
            for _ in range(600):
                op = rs.randrange(10)
                try:
                    if op <= 3:
                        p = _family(rs.randrange(3), rs.choice([0, 64, 130])) + _family(rs.randrange(50), rs.choice([1, 30, 65]))
                        kw = dict(ignore_eos=True, temperature=rs.choice([0.0, 0.8]), seed=rs.randrange(100))
                        n = rs.choice([1, 1, 2, 3, 6])
                        live += eng.submit_choices(p, rs.choice([1, 5, 40, 150]), n, **kw) if n > 1 else [eng.submit(p, 20, **kw)]
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
def test_scenario_two_rank_plan_channel_replays_groups_to_identical_counters():
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    world = 2
    handles, barrier, q = ctx.Array("B", 64 * world), ctx.Barrier(world), ctx.Queue()
    name = "llmlb_n_rnd_%d" % os.getpid()
    ps = [ctx.Process(target=_tp_rank, args=(r, world, handles, barrier, name, q)) for r in range(world)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=300) for _ in range(world))
    [p.join(60) for p in ps]
    assert all("error" not in v for v in got.values()), got
    lead, foll = got[0], got[1]
    assert lead["counters"] == foll["counters"], (lead["counters"], foll["counters"])
    assert lead["cache"] == foll["cache"], (lead["cache"], foll["cache"])
    assert lead["pages"] == foll["pages"] == (14, 14)
    assert lead["counters"]["steps_decode"] > 100, lead
    assert all(p.exitcode == 0 for p in ps)
