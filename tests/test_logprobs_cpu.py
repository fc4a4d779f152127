"""Token logprobs without a GPU: the oracle and its checker (tests/logprob_oracle.py) against a numpy model of
logprob_kernel, with the defects the checker must reject; the engine's launch plan over the fake CUDA runtime
(tests/support/fake_cudart.cpp) with and without logprob requests; the GPU op cases against the vocabularies the engine
samples; the argument checks and event pairing of llmlb_request_submit_logprobs / llmlb_request_poll_logprobs; a
two-process tensor-parallel plan channel that carries logprob requests through cancels and preemptions; and the layout of
llmlb_token_logprobs in C, ctypes and Rust.  The GPU side is tests/test_logprobs_gpu.py.

The scenarios that need the fake runtime run in a child pytest process that preloads it, as in
tests/test_engine_host_logic_cpu.py; they skip themselves elsewhere."""
import ctypes as C
import math
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import logprob_oracle as O  # noqa: E402
import test_engine_host_logic_cpu as HL  # noqa: E402

INNER = os.environ.get("LLMLB_FAKE_CUDART") == "1"
inner = pytest.mark.skipif(not INNER, reason="runs in the child process that preloads the fake CUDA runtime")
TINY = HL.TINY


# ---- oracle and checker ------------------------------------------------------------------------------------------------
def _rows(V, seed):
    rs = np.random.RandomState(seed)
    out = [O.lm_row(V, rs), np.zeros(V, np.float32)]
    z = O.lm_row(V, rs)
    z[rs.choice(V, max(1, V // 10), replace=False)] = -np.inf
    out.append(z)
    return out


@pytest.mark.parametrize("V", O.VOCABS)
def test_checker_accepts_the_kernel_model(V):
    for i, z in enumerate(_rows(V, V)):
        for n in (0, 1, 5, 20, 25):
            for tok in (int(np.argmax(z)), int(np.nonzero(np.isfinite(z))[0][-1])):
                ok, why = O.check(z, n, tok, O.kernel_model(z, n, tok))
                assert ok, (i, n, tok, why)


def test_selection_is_z_descending_ties_by_ascending_id():
    z = np.array([1.0, 3.0, 3.0, -0.0, 0.0, -np.inf, 3.0, 2.0], np.float32)
    assert O.top_ids(z, 20).tolist() == [1, 2, 6, 7, 0, 3, 4, 5]
    assert O.top_ids(z, 2).tolist() == [1, 2] and O.top_ids(z, 0).tolist() == []
    lp, b = O.bound(z)
    assert np.isneginf(lp[5]) and abs(np.exp(lp).sum() - 1) < 1e-12


def test_checker_rejects_expf_at_its_documented_error():
    """__expf (2 + floor(1.173 |d|) ulp) on a row whose mass sits at d = -9: the error of log s exceeds the bound."""
    V = 128256
    rs = np.random.RandomState(1)
    z = (np.float32(-9) + rs.rand(V).astype(np.float32) * np.float32(0.01)).astype(np.float32)
    z[17] = 0
    assert O.check(z, 5, 17, O.kernel_model(z, 5, 17))[0]
    ok, why = O.check(z, 5, 17, O.kernel_model(z, 5, 17, expf_ulps=O.expf_documented_ulps))
    assert not ok and "bound" in why, why


@pytest.mark.parametrize("V", [128256, 32003, 4096, 2048])
def test_checker_rejects_a_dropped_last_warp_span_and_logprobs_after_temperature(V):
    z = O.lm_row(V, np.random.RandomState(V))
    t = int(np.argmax(z))
    assert O.check(z, 5, t, O.kernel_model(z, 5, t))[0]
    assert not O.check(z, 5, t, O.kernel_model(z, 5, t, drop_last_span=True))[0]
    assert not O.check(z, 5, t, O.kernel_model(z, 5, t, temperature=0.7))[0]
    assert not O.check(z, 0, t, O.kernel_model(z, 0, t, temperature=1.3))[0]      # the token's value alone


def test_checker_rejects_ties_by_the_highest_id_and_the_neighbouring_row():
    z = np.zeros(2048, np.float32)
    ok, why = O.check(z, 5, 0, O.kernel_model(z, 5, 0, ties_high=True))
    assert not ok and "ids" in why
    rs = np.random.RandomState(5)
    rows = [O.lm_row(4096, rs) for _ in range(2)]
    t = int(np.argmax(rows[0]))
    assert O.check(rows[0], 5, t, O.kernel_model(rows[0], 5, t))[0]
    assert not O.check(rows[0], 5, t, O.kernel_model(rows[1], 5, t))[0]
    assert not O.check(rows[0], 0, t, O.kernel_model(rows[1], 0, t))[0]


# ---- launch plans over the fake runtime ----------------------------------------------------------------------------------
def _plan(tmp_path, mode, graphs):
    log = str(tmp_path / ("%s_%s.log" % (mode, graphs)))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, os.path.join(HERE, "support", "logprob_plan_sweep.py"), mode, graphs], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "fake cudart:" not in r.stderr, r.stderr[-3000:]          # configuration, shared-memory and capture checks
    return open(log).read().splitlines()


def _kernel(line):
    return re.sub(r"^_ZN5llmlb\d+|^_Z\d+", "", line.split()[0])


@pytest.mark.parametrize("graphs", ["graphs", "eager"])
def test_launch_plan_of_logprobs_adds_only_the_logprob_kernel(built_lib, tmp_path, graphs):
    """The same workload (prefill widths 1..2048, decode batches of 1..64) submitted through llmlb_request_submit, through
    llmlb_request_submit_penalized without penalties and drained with llmlb_request_poll_logprobs, and with every other
    request reporting logprobs: the second plan is identical line for line; the third is the same plan plus one
    logprob_kernel right after each sample_kernel, over the same rows."""
    plain = _plan(tmp_path, "plain", graphs)
    assert plain == _plan(tmp_path, "nolp", graphs)
    mixed = _plan(tmp_path, "mixed", graphs)
    assert [l for l in mixed if l.startswith("###") or not _kernel(l).startswith("logprob_kernel")] == plain
    names = [l if l.startswith("###") else _kernel(l) for l in mixed]
    n_sample = n_lp = 0
    section = ""
    for i, (line, k) in enumerate(zip(mixed, names)):
        if line.startswith("###"):
            section = line
            continue
        p = line.split()
        if k.startswith("logprob_kernel"):
            n_lp += 1
            assert names[i - 1].startswith("sample_kernel")                     # right after the sampler, same rows
            assert mixed[i - 1].split()[1:4] == p[1:4] and p[4:7] == ["1024", "1", "1"] and p[7:12] == ["0", "1", "1", "1", "0"]
        elif k.startswith("sample_kernel") and section:                         # not the warm-up of engine creation
            n_sample += 1
            assert names[i + 1].startswith("logprob_kernel"), (section, i)      # every step of this workload has a logprob row
    assert n_lp == n_sample > 0


def test_gpu_op_cases_launch_every_vocab_the_engine_samples(built_lib, tmp_path):
    """logprob_kernel runs on the rows sample_kernel sampled (the plan test above), so its vocabularies are the sampler's:
    every vocabulary the tp = 1 engine samples at Llama-3-8B, LLAMA_MID and Llama-3-70B shapes must be among those
    tests/test_logprobs_gpu.py launches logprob_kernel with."""
    import test_kernel_coverage_cpu as KC          # both import torch, which the fake-runtime child cannot load
    import test_logprobs_gpu as LG
    cases = ["%d:%d" % (R, V) for R, V in LG.OP_CASES]
    log = str(tmp_path / "logprob_cases.log")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, os.path.join(HERE, "support", "logprob_case_sweep.py")] + cases, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    tested, mark = set(), None
    for line in open(log):
        if line.startswith("###"):
            mark = line.split()
            continue
        if KC.short_name(line.split()[0]) == "logprob_kernel":
            assert line.split()[1] == mark[2]                                    # one CTA per row
            tested.add(int(mark[3]))
    assert tested == set(O.VOCABS), sorted(tested)
    engine = {}
    for model in KC.PLAN_MODELS:
        for c in KC._sample_classes(KC._engine_plan(tmp_path, model, 1, 8)):
            engine.setdefault(c[1], model)
    assert set(engine) >= {128256, 4096}, engine
    assert {128256, 4096, 2048} <= tested
    missing = sorted((V, m) for V, m in engine.items() if V not in tested)
    assert not missing, "the engine samples vocabularies no GPU logprob test runs (vocab, model): %s" % missing


# ---- ABI ---------------------------------------------------------------------------------------------------------------
def test_token_logprobs_layout_in_c_ctypes_and_rust():
    from llmlb_b200 import ffi
    src = r'''#include <stdio.h>
#include <stddef.h>
#include "llmlb_b200.h"
int main(void){printf("%zu %zu %zu %zu %zu %d\n", sizeof(llmlb_token_logprobs), offsetof(llmlb_token_logprobs, n_top),
 offsetof(llmlb_token_logprobs, top_ids), offsetof(llmlb_token_logprobs, top_logprobs), sizeof(llmlb_token_event),
 LLMLB_MAX_TOP_LOGPROBS);return 0;}'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "p.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "p.c"), "-o", os.path.join(d, "p")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "p")], text=True).split()]
    T = ffi.TokenLogprobs
    assert got == [168, 4, 8, 88, C.sizeof(ffi.TokenEvent), 20]
    assert [C.sizeof(T), T.n_top.offset, T.top_ids.offset, T.top_logprobs.offset] == got[:4]
    assert ffi.MAX_TOP_LOGPROBS == 20
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "check_rust_layout.py")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    rs = open(os.path.join(ROOT, "ffi", "llmlb-b200-sys", "src", "lib.rs")).read()
    for name in ("llmlb_token_logprobs", "llmlb_request_submit_logprobs", "llmlb_request_poll_logprobs"):
        assert name in rs


# ---- the scenarios below run in a child that preloads the fake runtime ------------------------------------------------
def test_logprobs_over_the_fake_cuda_runtime(built_lib):
    if INNER:
        pytest.skip("already inside")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


@inner
def test_scenario_submit_logprobs_checks_and_event_pairing():
    ffi = HL._ffi()
    L = ffi.lib()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=512) as eng:
        s = ffi.Sampling(max_tokens=4)
        prompt = (C.c_int32 * 3)(1, 2, 3)
        rid = C.c_uint64()
        for n in (21, 100, 2 ** 32 - 1):
            assert L.llmlb_request_submit_logprobs(eng._h, prompt, 3, C.byref(s), None, n, C.byref(rid)) == ffi.E_INVALID_ARG
            assert "top_logprobs" in ffi.last_error()
        assert L.llmlb_request_submit_logprobs(None, prompt, 3, C.byref(s), None, 5, C.byref(rid)) == ffi.E_INVALID_ARG
        pen = ffi.Penalties(3.0, 0.0, None, None, 0)                             # the penalties are still checked
        assert L.llmlb_request_submit_logprobs(eng._h, prompt, 3, C.byref(s), C.byref(pen), 5, C.byref(rid)) == ffi.E_INVALID_ARG
        assert "frequency_penalty" in ffi.last_error()
        ev, lp, n = (ffi.TokenEvent * 4)(), (ffi.TokenLogprobs * 4)(), C.c_uint32()
        assert L.llmlb_request_poll_logprobs(eng._h, 12345, ev, lp, 4, C.byref(n), 0) == ffi.E_NOT_FOUND
        # both limits are accepted; a request without logprobs polls NaN and no alternatives
        for kw in (dict(logprobs=0), dict(logprobs=20), dict(logprobs=20, logit_bias={3: 1.0}), {}):
            r = eng.submit([1, 2, 3], 6, ignore_eos=True, **kw)
            evs = []
            while not (evs and evs[-1]["finish_reason"]):
                evs += eng.poll_logprobs(r, cap=2, timeout_ms=50)                # small caps: records stay with their events
            assert [e["index"] for e in evs] == list(range(6)) and evs[-1]["finish_reason"] == HL.LENGTH
            if not kw:
                assert all(math.isnan(e["logprob"]) and e["top_logprobs"] == [] for e in evs)
            else:   # the fake runtime computes nothing: the records are the zero-filled device buffer's, not the NaN filler
                assert all(e["logprob"] == 0.0 and e["top_logprobs"] == [] for e in evs), evs
            eng.release(r)
        # llmlb_request_poll drains a logprob request's records with its events; a cancel's end event has none
        r = eng.submit([1, 2, 3], 400, ignore_eos=True, logprobs=3)
        first = eng.poll(r, timeout_ms=-1)
        eng.cancel(r)
        evs = list(first)
        while not (evs and evs[-1]["finish_reason"]):
            evs += eng.poll_logprobs(r, timeout_ms=50)
        assert first and all(e["token_id"] >= 0 for e in first[:-1])
        assert evs[-1]["finish_reason"] in (HL.CANCELLED, HL.LENGTH)
        for e in evs[len(first):]:
            assert math.isnan(e["logprob"]) == (e["token_id"] < 0)
        eng.release(r)
        h = HL.settle(eng)
        assert h["free_kv_pages"] == h["total_kv_pages"]


@inner
def test_scenario_logprob_requests_survive_preemption_with_paired_records():
    """14 pages for 6 sequences of 100 + 250 tokens: the youngest are evicted and recomputed.  Every request gets one record
    per event, with its own number of alternatives."""
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=14) as eng:
        tops = [5, None, 0, 20, None, 1]        # logprob records of the fake runtime: 0.0 (zero-filled), NaN without logprobs
        rids = [eng.submit([(5 * i + j) % TINY["vocab"] for j in range(100)], 250, ignore_eos=True, logprobs=t)
                for i, t in enumerate(tops)]
        outs = {r: [] for r in rids}
        t0 = time.time()
        while any(not (v and v[-1]["finish_reason"]) for v in outs.values()):
            assert time.time() - t0 < 120
            for r in rids:
                if not (outs[r] and outs[r][-1]["finish_reason"]):
                    outs[r] += eng.poll_logprobs(r, timeout_ms=5)
        assert eng.health()["preemptions"] > 0
        for r, t in zip(rids, tops):
            evs = outs[r]
            assert [e["index"] for e in evs] == list(range(250)) and evs[-1]["finish_reason"] == HL.LENGTH
            assert all(math.isnan(e["logprob"]) == (t is None) and e["top_logprobs"] == [] for e in evs)
            eng.release(r)


def _tp_rank(rank, world, handles, barrier, name, out_q):
    try:
        os.environ["FAKE_CUDART_STEP_US"] = "200"
        ffi = HL._ffi()
        eng = ffi.Engine(TINY, model_id="tp-lp", device=0, tp_rank=rank, tp_size=world, max_seqs=8, max_ctx=1024, kv_pages=14, seed=0)
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
            kws = [dict(logprobs=20), {}, dict(logprobs=0, presence_penalty=1.0, logit_bias={3: 5.0}), dict(logprobs=5),
                   dict(frequency_penalty=0.5), dict(logprobs=1)]
            rids = []
            for i, kw in enumerate(kws):
                rids.append(eng.submit([(5 * i + j) % TINY["vocab"] for j in range(100)], 250, ignore_eos=True, **kw))
                if i == 4:
                    eng.cancel(rids[3])
            outs = [HL.drain(eng, r, 120) for r in rids]
            for r in rids:
                eng.release(r)
            res = {"reasons": [o[-1]["finish_reason"] for o in outs]}
            HL.settle(eng, 60)
        barrier.wait(180)
        if rank != 0:                                                           # the follower has drained the log when its counters stop moving
            last, t0 = None, time.time()
            while time.time() - t0 < 20:
                cur = eng.health()["kernel_launches"]
                if cur == last:
                    break
                last = cur
                time.sleep(0.2)
        hz = eng.health()
        res["counters"] = {k: hz[k] for k in ("steps_prefill", "steps_decode", "tokens_decode", "tokens_prefill", "kernel_launches", "preemptions")}
        res["pages"] = (hz["free_kv_pages"], hz["total_kv_pages"], hz["active_requests"], hz["queued_requests"])
        out_q.put((rank, res))
        barrier.wait(60)
        eng.close()
    except Exception as e:                                                      # noqa: BLE001
        out_q.put((rank, {"error": repr(e)}))
        try:
            barrier.abort()
        except Exception:                                                       # noqa: BLE001
            pass


@inner
def test_scenario_two_rank_plan_channel_carries_logprobs_through_preemption():
    """The leader logs logprob, penalised and plain submits, a cancel, and evicts sequences from a small KV pool; the
    follower sees only the shared-memory log.  It must launch exactly what the leader launched — the logprob kernels
    included, which needs top_logprobs from the submit record — and end with the same counters and an empty pool."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    world = 2
    handles = ctx.Array("B", 64 * world)
    barrier = ctx.Barrier(world)
    q = ctx.Queue()
    name = "llmlb_lp_cpu_%d" % os.getpid()
    ps = [ctx.Process(target=_tp_rank, args=(r, world, handles, barrier, name, q)) for r in range(world)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=300) for _ in range(world))
    [p.join(60) for p in ps]
    assert all("error" not in v for v in got.values()), got
    lead, foll = got[0], got[1]
    assert lead["reasons"][3] == HL.CANCELLED and all(r == HL.LENGTH for i, r in enumerate(lead["reasons"]) if i != 3), lead
    assert lead["counters"]["preemptions"] > 0, lead
    assert lead["counters"] == foll["counters"], (lead["counters"], foll["counters"])
    assert lead["pages"] == foll["pages"] and lead["pages"][0] == lead["pages"][1] and lead["pages"][2:] == (0, 0)
    assert all(p.exitcode == 0 for p in ps)
