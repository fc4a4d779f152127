"""Prompt logprobs without a GPU, over the fake CUDA runtime (tests/support/fake_cudart.cpp): the launch plan of prompt-
logprob requests against the same requests without the prompt records; the kernel classes the new launches use against those
the GPU kernel tests run; the argument checks and record counts of llmlb_request_submit_prompt_logprobs /
llmlb_request_poll_prompt_logprobs for prompts of one token, one chunk and several chunks, cancels and a released request;
preemption; and a two-process tensor-parallel plan channel carrying prompt-logprob requests.  The fake runtime computes
nothing, so the records it returns are the zero-filled device buffer's: these tests check which records arrive and when, the
GPU tests (tests/test_prompt_logprobs_gpu.py) their values.

The scenarios that need the fake runtime run in a child pytest process that preloads it, as in
tests/test_engine_host_logic_cpu.py; they skip themselves elsewhere."""
import ctypes as C
import json
import os
import re
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


# ---- launch plans ------------------------------------------------------------------------------------------------------
def _plan_log(tmp_path, mode, graphs, max_seqs, tp=1):
    log = str(tmp_path / ("%s_%s_%d_%d.log" % (mode, graphs, max_seqs, tp)))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, os.path.join(HERE, "support", "prompt_logprob_plan_sweep.py"), mode, graphs, str(max_seqs), str(tp)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "fake cudart:" not in r.stderr, r.stderr[-3000:]
    return log


def _name(line):
    s = re.sub(r"^_ZN5llmlb|^_Z", "", line.split()[0])
    m = re.match(r"\d+", s)
    return s[m.end(): m.end() + int(m.group())] if m else s


GATHERS = ("gather_rows_kernel", "gather_rows_bf16_kernel")
LM_HEAD = ("gemv_ks_kernel", "gemv_kernel", "gemm_tc_kernel", "gemm_tc2_kernel")
STEP_ENDS = ("prefill_finish_kernel", "logprob_kernel", "rmsnorm_parts_kernel", "rmsnorm_parts_cluster_kernel", "tp_reduce_norm_kernel",
             "tp_fold_rows_kernel")


def _split_groups(lines, tp):
    """The plan without its prompt-record groups, and the groups: (index in lines, rows, kernels).  A group is a row gather
    whose rows go to logprob_kernel without passing the sampler; at tp > 1 it starts with the one-block pull barrier before
    the gather (allreduce_add_kernel over no elements), which keeps the group's lm_head from rewriting this rank's logits
    exchange slot while a peer still pulls it."""
    rest, groups, i = [], [], 0
    while i < len(lines):
        l = lines[i]
        if not l.startswith("###") and _name(l) in GATHERS:
            j = i + 1
            while j < len(lines) and not lines[j].startswith("###") and _name(lines[j]) not in ("logprob_kernel", "sample_prepare_kernel"):
                j += 1
            if j < len(lines) and not lines[j].startswith("###") and _name(lines[j]) == "logprob_kernel":
                if tp > 1:
                    assert _name(rest[-1]) == "allreduce_add_kernel" and rest[-1].split()[1:4] == ["1", "1", "1"], rest[-1]
                    rest.pop()
                    i -= 1
                groups.append((i, int(lines[j].split()[1]), [_name(x) for x in lines[i:j + 1]]))
                i = j + 1
                continue
        rest.append(l)
        i += 1
    return rest, groups


def _expected_rows():
    sys.path.insert(0, os.path.join(HERE, "support"))
    import prompt_logprob_plan_sweep as S
    rows = {"prefill T=%d" % T: T - 1 for T in S.PREFILL_WIDTHS}
    rows["chunked T=%d" % S.CHUNKED] = S.CHUNKED - 1
    rows.update({"decode B=%d" % B: sum(8 + i - 1 for i in range(B)) for B in S.DECODE_BATCHES})
    return rows, S


@pytest.mark.parametrize("graphs,max_seqs,tp", [("graphs", 8, 1), ("eager", 8, 1), ("graphs", 64, 1), ("eager", 64, 1), ("eager", 8, 2)])
def test_prompt_records_add_only_their_row_groups(built_lib, tmp_path, graphs, max_seqs, tp):
    """The same logprob workload (prefills 1..2048 wide, a 4500-token prompt over three prefill steps, decode batches of 1, 3
    and 8) with and without prompt logprobs.  Without the prompt groups the plans are identical line for line — prefill and
    decode steps are those of a logprob request.  Each prefill step that computes prompt records ends with groups of at most
    max_seqs rows, all full but the last, each exactly: (at tp > 1) a one-block pull barrier, row gather, lm_head (with its final RMSNorm above 4 rows), the
    logits all-gather at tp > 1, logprob_kernel over the same rows; one record per prompt position but the last."""
    lp = open(_plan_log(tmp_path, "lp", graphs, max_seqs, tp)).read().splitlines()
    pr = open(_plan_log(tmp_path, "prompt", graphs, max_seqs, tp)).read().splitlines()
    rest, groups = _split_groups(pr, tp)
    assert rest == lp
    assert not _split_groups(lp, tp)[1]
    want, _ = _expected_rows()
    rows, section, run = {}, "", []
    marks = [(i, l[4:]) for i, l in enumerate(pr) if l.startswith("###")]
    for gi, (i, R, names) in enumerate(groups):
        section = [m for k, m in marks if k < i][-1]
        if tp > 1:
            names = names[1:]
            i += 1
        mid = names[1:-1]
        if tp > 1:
            assert mid[-1] == "allgather_cols_kernel", names
            mid = mid[:-1]
        assert mid in ([n] for n in LM_HEAD) or (R > 4 and tp == 1 and mid[0] == "rmsnorm_kernel" and len(mid) == 2 and mid[1] in LM_HEAD), names
        assert (mid[-1] in ("gemv_ks_kernel", "gemv_kernel")) == (R <= 4), names
        assert pr[i].split()[1] == str(R)                                                 # the gather: one CTA per row
        prev = _name(pr[groups[gi][0] - 1])
        assert prev in STEP_ENDS, (section, prev)                                        # right after the step's own kernels
        assert 1 <= R <= max_seqs
        rows[section] = rows.get(section, 0) + R
        if prev == "logprob_kernel" and run:
            assert run[-1] == max_seqs, (section, run)                                  # only a step's last group is short
        run = run + [R] if prev == "logprob_kernel" else [R]
    assert rows == {k: v * tp for k, v in want.items() if v}, (rows, want)                # every rank computes them


def test_prompt_groups_launch_only_kernel_classes_the_gpu_tests_run(built_lib, tmp_path):
    """Every lm_head GEMM / GEMV class, final-RMSNorm width and logprob vocabulary the prompt groups launch (Llama-3-8B,
    max_seqs 8 and 64) is among those the GPU kernel tests launch (tests/support/kernel_case_sweep.py)."""
    import logprob_oracle as O
    import test_gemv_sm90_gpu as GV
    import test_kernel_coverage_cpu as KC
    import test_kernels_sm90_gpu as K
    spec = tmp_path / "cases.json"
    spec.write_text(json.dumps({"gemm": [[T, N, Kd, e] for T, N, Kd, epis in K.GEMM_CASES for e in epis],
                                "wave_tail": list(K.WAVE_TAIL_CASE) + [K.wave_tail_rows(*K.WAVE_TAIL_CASE[:2])],
                                "decode_splits": K.DECODE_SPLITS, "max_split": K.GEMM_MAX_SPLIT}))
    tested = set().union(*KC.run_logged(tmp_path, "cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)]).values())
    tested |= KC._gemv_classes(KC._gemv_sweep(tmp_path, "gemv_cases", GV.gemv_params()))
    tested |= KC._kind(KC._step_case_plan(tmp_path))
    used, n_lp = set(), 0
    for max_seqs in (8, 64):
        lines = open(_plan_log(tmp_path, "prompt", "eager", max_seqs)).read().splitlines()
        groups = _split_groups(lines, 1)[1]
        glog = tmp_path / ("groups_%d.log" % max_seqs)
        glog.write_text("".join(l + "\n" for i, _, names in groups for l in lines[i:i + len(names)]))
        used |= set().union(*KC.classes(str(glog)).values())
        for l in open(str(glog)):
            if _name(l) == "logprob_kernel":
                n_lp += 1
    assert n_lp > 0 and any(c[0] == "gemm_tc_kernel" for c in used) and any(c[0] == "gemv_ks" for c in used), sorted(used)
    missing = sorted(used - tested)
    assert not missing, "the prompt groups launch classes no GPU kernel test runs: %s" % missing
    assert 128256 in O.VOCABS


# ---- the scenarios below run in a child that preloads the fake runtime ------------------------------------------------
def test_prompt_logprobs_over_the_fake_cuda_runtime(built_lib):
    if INNER:
        pytest.skip("already inside")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


def _drain(eng, rid, timeout=120):
    """(events, prompt records read right after the first event, prompt records read after the end)"""
    evs, first, t0 = [], None, time.time()
    while not (evs and evs[-1]["finish_reason"]):
        assert time.time() - t0 < timeout
        got = eng.poll_logprobs(rid, timeout_ms=20)
        if got and first is None:
            first = eng.poll_prompt_logprobs(rid, cap=100000)
        evs += got
    return evs, first, eng.poll_prompt_logprobs(rid, cap=100000)


@inner
def test_scenario_submit_and_poll_prompt_logprobs_checks_and_counts():
    ffi = HL._ffi()
    L = ffi.lib()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=1024, max_step_tokens=64) as eng:
        s = ffi.Sampling(max_tokens=3)
        prompt = (C.c_int32 * 3)(1, 2, 3)
        rid = C.c_uint64()
        for n in (21, 2 ** 32 - 1):
            assert L.llmlb_request_submit_prompt_logprobs(eng._h, prompt, 3, C.byref(s), None, n, C.byref(rid)) == ffi.E_INVALID_ARG
            assert "top_logprobs" in ffi.last_error()
        assert L.llmlb_request_submit_prompt_logprobs(None, prompt, 3, C.byref(s), None, 5, C.byref(rid)) == ffi.E_INVALID_ARG
        assert L.llmlb_request_submit_prompt_logprobs(eng._h, prompt, 0, C.byref(s), None, 5, C.byref(rid)) == ffi.E_INVALID_ARG
        pen = ffi.Penalties(0.0, 2.5, None, None, 0)
        assert L.llmlb_request_submit_prompt_logprobs(eng._h, prompt, 3, C.byref(s), C.byref(pen), 5, C.byref(rid)) == ffi.E_INVALID_ARG
        assert "presence_penalty" in ffi.last_error()
        recs, n = (ffi.TokenLogprobs * 4)(), C.c_uint32()
        assert L.llmlb_request_poll_prompt_logprobs(eng._h, 12345, recs, 4, C.byref(n)) == ffi.E_NOT_FOUND
        assert L.llmlb_request_poll_prompt_logprobs(None, 1, recs, 4, C.byref(n)) == ffi.E_INVALID_ARG
        # one token, one chunk, several chunks (max_step_tokens 64), penalised and biased: n - 1 records, all before the first
        # event, none later; the generated tokens keep their own records
        for n_prompt, kw in ((1, dict(logprobs=0)), (2, dict(logprobs=20)), (64, dict(logprobs=3)), (65, dict(logprobs=1)),
                             (300, dict(logprobs=5, frequency_penalty=1.0, logit_bias={7: 100.0}))):
            r = eng.submit([(3 * j) % TINY["vocab"] for j in range(n_prompt)], 5, ignore_eos=True, prompt_logprobs=True, **kw)
            evs, first, after = _drain(eng, r)
            assert [e["index"] for e in evs] == list(range(5))
            assert len(first) == n_prompt - 1 and after == [], (n_prompt, len(first), len(after))
            assert all(x["logprob"] == 0.0 and x["top_logprobs"] == [] for x in first)   # the zero-filled buffer: not the NaN filler
            assert all(e["logprob"] == 0.0 for e in evs)
            eng.release(r)
            assert L.llmlb_request_poll_prompt_logprobs(eng._h, r, recs, 4, C.byref(n)) == ffi.E_NOT_FOUND
        # without the flag: no prompt records
        r = eng.submit(list(range(1, 40)), 3, ignore_eos=True, logprobs=2)
        evs, first, after = _drain(eng, r)
        assert first == [] and after == []
        eng.release(r)
        with pytest.raises(ValueError):
            eng.submit([1, 2], 3, prompt_logprobs=True)
        # a cancel before admission delivers nothing; one during a prefill of several steps a prefix
        eng.pause(True)
        r = eng.submit(list(range(1, 500)), 5, ignore_eos=True, logprobs=1, prompt_logprobs=True)
        eng.cancel(r)
        eng.pause(False)
        evs, first, after = _drain(eng, r)
        assert evs[-1]["finish_reason"] == HL.CANCELLED and (first or []) + after == []
        eng.release(r)
        h = HL.settle(eng)
        assert h["free_kv_pages"] == h["total_kv_pages"]


@inner
def test_scenario_cancel_during_a_chunked_prefill_delivers_a_prefix():
    """A cancel that lands during a prefill of 500 steps: the records of the steps harvested before it, whole 64-row chunks
    from position 0 on, and nothing after.  The fake runtime gives prefill steps no duration (FAKE_CUDART_STEP_US delays
    decode graph launches only), so the cancel, sent once 4 steps have run, races the remaining 496: every attempt must
    deliver such a prefix (or everything, had the prefill won), and one of ten must land inside."""
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=2, max_ctx=32768, max_step_tokens=64) as eng:
        n_prompt, inside = 32000, 0
        for attempt in range(10):
            before = eng.health()["steps_prefill"]
            r = eng.submit([(5 * j) % TINY["vocab"] for j in range(n_prompt)], 5, ignore_eos=True, logprobs=2, prompt_logprobs=True)
            t0 = time.time()
            while eng.health()["steps_prefill"] < before + 4:
                assert time.time() - t0 < 60
            eng.cancel(r)
            evs, first, after = _drain(eng, r)
            got = len(first or []) + len(after)
            if evs[-1]["finish_reason"] == HL.CANCELLED and got < n_prompt - 1:
                assert got % 64 == 0, got
                inside += 1
            else:
                assert got == n_prompt - 1, (evs[-1], got)
            eng.release(r)
            if inside:
                break
        assert inside
        h = HL.settle(eng)
        assert h["free_kv_pages"] == h["total_kv_pages"]


@inner
def test_scenario_prompt_records_survive_preemption_once_each():
    """14 pages for 6 sequences of 100..350-token prompts over 64-token prefill steps, 150 generated tokens each: the youngest
    are evicted and their context (prompt plus generated tokens) is recomputed over several prefill steps.  Every prompt-logprob
    request gets exactly n - 1 prompt records — none twice, none for the generated part of the recomputed context."""
    ffi = HL._ffi()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=1024, kv_pages=14, max_step_tokens=64) as eng:
        lens = [100, 350, 120, 200, 130, 300]
        flags = [True, True, False, True, True, True]
        rids = [eng.submit([(5 * i + j) % TINY["vocab"] for j in range(n)], 150, ignore_eos=True, logprobs=i % 3, prompt_logprobs=f)
                for i, (n, f) in enumerate(zip(lens, flags))]
        outs = {r: ([], []) for r in rids}
        t0 = time.time()
        while any(not (v[0] and v[0][-1]["finish_reason"]) for v in outs.values()):
            assert time.time() - t0 < 120
            for r in rids:
                evs, recs = outs[r]
                if not (evs and evs[-1]["finish_reason"]):
                    got = eng.poll_logprobs(r, timeout_ms=5)
                    recs += eng.poll_prompt_logprobs(r, cap=4096)
                    if got and not evs:                                  # every record is queued before the first event
                        i = rids.index(r)
                        assert len(recs) == (lens[i] - 1 if flags[i] else 0), (i, len(recs))
                    evs += got
        assert eng.health()["preemptions"] > 0
        for r, n, f in zip(rids, lens, flags):
            evs, recs = outs[r]
            recs += eng.poll_prompt_logprobs(r, cap=4096)
            assert [e["index"] for e in evs] == list(range(150)) and evs[-1]["finish_reason"] == HL.LENGTH
            assert len(recs) == (n - 1 if f else 0), (n, f, len(recs))
            eng.release(r)


def _tp_rank(rank, world, handles, barrier, name, out_q):
    try:
        os.environ["FAKE_CUDART_STEP_US"] = "200"
        ffi = HL._ffi()
        eng = ffi.Engine(TINY, model_id="tp-plp", device=0, tp_rank=rank, tp_size=world, max_seqs=8, max_ctx=1024, kv_pages=14,
                         max_step_tokens=64, seed=0)
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
            kws = [dict(logprobs=20, prompt_logprobs=True), {}, dict(logprobs=0, presence_penalty=1.0, logit_bias={3: 5.0}, prompt_logprobs=True),
                   dict(logprobs=5, prompt_logprobs=True), dict(frequency_penalty=0.5), dict(logprobs=1), dict(logprobs=2, prompt_logprobs=True)]
            rids, lens = [], []
            for i, kw in enumerate(kws):
                lens.append(100 + 37 * i)
                rids.append(eng.submit([(5 * i + j) % TINY["vocab"] for j in range(lens[-1])], 200, ignore_eos=True, **kw))
                if i == 4:
                    eng.cancel(rids[3])
            outs = [HL.drain(eng, r, 120) for r in rids]
            res["prompt_records"] = [len(eng.poll_prompt_logprobs(r, cap=4096)) for r in rids]
            res["want_records"] = [n - 1 if kw.get("prompt_logprobs") else 0 for n, kw in zip(lens, kws)]
            for r in rids:
                eng.release(r)
            res["reasons"] = [o[-1]["finish_reason"] for o in outs]
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
def test_scenario_two_rank_plan_channel_carries_prompt_logprobs_through_preemption():
    """The leader logs prompt-logprob, logprob, penalised and plain submits, a cancel, and evicts sequences from a small KV
    pool; the follower sees only the shared-memory log.  It must launch exactly what the leader launched — the prompt groups
    included, which needs the prompt flag of the submit record — and end with the same counters and an empty pool."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    world = 2
    handles = ctx.Array("B", 64 * world)
    barrier = ctx.Barrier(world)
    q = ctx.Queue()
    name = "llmlb_plp_cpu_%d" % os.getpid()
    ps = [ctx.Process(target=_tp_rank, args=(r, world, handles, barrier, name, q)) for r in range(world)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=300) for _ in range(world))
    [p.join(60) for p in ps]
    assert all("error" not in v for v in got.values()), got
    lead, foll = got[0], got[1]
    assert lead["reasons"][3] == HL.CANCELLED and all(r == HL.LENGTH for i, r in enumerate(lead["reasons"]) if i != 3), lead
    assert all(g == w for i, (g, w) in enumerate(zip(lead["prompt_records"], lead["want_records"])) if i != 3), lead
    assert lead["counters"]["preemptions"] > 0, lead
    assert lead["counters"] == foll["counters"], (lead["counters"], foll["counters"])
    assert lead["pages"] == foll["pages"] and lead["pages"][0] == lead["pages"][1] and lead["pages"][2:] == (0, 0)
    assert all(p.exitcode == 0 for p in ps)
