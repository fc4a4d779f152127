"""Frequency / presence penalties and logit bias without a GPU: the oracle against a float64 evaluation of the formula, the
engine's launch plan over the fake CUDA runtime (tests/support/fake_cudart.cpp) with neutral, mixed and no penalties, the
argument checks of llmlb_request_submit_penalized, and a two-process tensor-parallel plan channel that carries
penalised requests through cancels and a preemption.  The GPU side (arithmetic, forcing, teacher-forced generation) is
tests/test_penalties_gpu.py.

The scenarios that need the fake runtime run in a child pytest process that preloads it, as in
tests/test_engine_host_logic_cpu.py; they skip themselves elsewhere."""
import ctypes as C
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_engine_host_logic_cpu as HL  # noqa: E402

INNER = os.environ.get("LLMLB_FAKE_CUDART") == "1"
inner = pytest.mark.skipif(not INNER, reason="runs in the child process that preloads the fake CUDA runtime")
TINY = HL.TINY
PEN_KERNELS = ("penalize_kernel", "penalty_count_kernel", "penalty_reset_kernel")


# ---- oracle ------------------------------------------------------------------------------------------------------------
def test_oracle_penalize_agrees_with_float64_evaluation():
    from penalty_oracle import penalize
    rs = np.random.RandomState(3)
    for vocab, f, p in ((128256, 0.7, 0.0), (1001, 0.0, 1.5), (4099, -0.5, 0.8), (2048, 2.0, -2.0)):
        logits = (rs.randn(vocab) * 4).astype(np.float32)
        counts = rs.randint(0, 3, vocab) * (rs.rand(vocab) < 0.1)
        counts[:3] = (0, 1, 131071)
        ids = rs.choice(vocab, 50, replace=False)
        bias = {int(i): float(np.float32(v)) for i, v in zip(ids, rs.uniform(-100, 100, 50))}
        bias[0], bias[vocab - 1] = 100.0, -100.0
        z = penalize(logits, counts, f, p, bias)
        assert z.dtype == np.float32
        b = np.zeros(vocab)
        for k, v in bias.items():
            b[k] = v
        ref = (logits.astype(np.float64) - (counts * np.float64(np.float32(f)) + (counts > 0) * np.float64(np.float32(p)))) + b
        # three fp32 roundings of values no larger than |logit| + |c * f| + |p| + |bias|
        scale = np.abs(logits) + np.abs(counts * f) + abs(p) + np.abs(b)
        assert np.all(np.abs(z - ref) <= 3 * 2.0 ** -24 * scale + 1e-30)
        assert np.array_equal(penalize(logits, counts, 0.0, 0.0, {}), logits)


# ---- launch plans over the fake runtime ----------------------------------------------------------------------------------
def _plan(tmp_path, mode, graphs):
    log = str(tmp_path / ("%s_%s.log" % (mode, graphs)))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log)
    r = subprocess.run([sys.executable, os.path.join(HERE, "support", "penalty_plan_sweep.py"), mode, graphs], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "fake cudart:" not in r.stderr, r.stderr[-3000:]          # configuration, shared-memory and capture checks
    return open(log).read().splitlines()


def _kernel(line):
    return re.sub(r"^_ZN5llmlb\d+|^_Z\d+", "", line.split()[0])


@pytest.mark.parametrize("graphs", ["graphs", "eager"])
def test_launch_plan_of_penalties_adds_only_the_penalty_kernels(built_lib, tmp_path, graphs):
    """The same workload (prefill widths 1..2048, decode batches of 1..64) submitted without penalties, with neutral ones
    through llmlb_request_submit_penalized, and with every other request penalised: the neutral plan is identical line for
    line; the penalised plan is the same plan plus the three penalty kernels, each where it belongs."""
    plain = _plan(tmp_path, "plain", graphs)
    assert plain == _plan(tmp_path, "neutral", graphs)
    mixed = _plan(tmp_path, "mixed", graphs)
    assert [l for l in mixed if l.startswith("###") or not _kernel(l).startswith(PEN_KERNELS)] == plain
    names = [l if l.startswith("###") else _kernel(l) for l in mixed]
    n_sample = n_pen = n_count = n_reset = 0
    section = ""
    for i, (line, k) in enumerate(zip(mixed, names)):
        if line.startswith("###"):
            section = line
            continue
        p = line.split()
        if k.startswith("penalize_kernel"):
            n_pen += 1
            assert names[i + 1].startswith("sample_kernel")                     # right before the sampler, same rows
            assert mixed[i + 1].split()[1:4] == p[1:4] and p[4:7] == ["1024", "1", "1"] and p[11] == "0"
        elif k.startswith("penalty_count_kernel"):
            n_count += 1
            assert names[i - 1].startswith("step_finish_kernel") and p[11] == "0"
        elif k.startswith("penalty_reset_kernel"):
            n_reset += 1
            assert names[i - 1].startswith("slot_init_kernel") and p[1:7] == ["1", "1", "1", "1024", "1", "1"] and p[11] == "0"
        elif k.startswith("sample_kernel") and section:                         # not the warm-up of engine creation
            n_sample += 1
            assert names[i - 1].startswith("penalize_kernel"), (section, i)     # every batch of this workload has a penalised row
    assert n_pen == n_sample == n_count > 0
    # one reset per penalised admission: the prefill sections' request, and the even-numbered requests of each batch
    decode_widths = range(1, 65) if graphs == "graphs" else (1, 2, 3, 4, 5, 8, 17, 33, 63, 64)
    assert n_reset == 7 + sum((b + 1) // 2 for b in decode_widths)


# ---- the scenarios below run in a child that preloads the fake runtime ------------------------------------------------
def test_penalties_over_the_fake_cuda_runtime(built_lib):
    if INNER:
        pytest.skip("already inside")
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


@inner
def test_scenario_submit_penalized_refuses_what_it_cannot_serve():
    ffi = HL._ffi()
    L = ffi.lib()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=512) as eng:
        def refused(field, **kw):
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.submit([1, 2, 3], 4, **kw)
            assert ei.value.code == ffi.E_INVALID_ARG and field in str(ei.value), str(ei.value)
        for v in (2.001, -2.5, float("nan"), float("inf"), -float("inf")):
            refused("frequency_penalty", frequency_penalty=v)
            refused("presence_penalty", presence_penalty=v)
        for v in (100.5, -101.0, float("nan"), float("inf")):
            refused("logit_bias", logit_bias={3: v})
        refused("logit_bias", logit_bias={-1: 1.0})
        refused("logit_bias", logit_bias={TINY["vocab"]: 1.0})
        refused("logit_bias", logit_bias={i: 1.0 for i in range(1025)})
        # duplicate ids cannot be written as a dict: through the C struct
        s = ffi.Sampling(max_tokens=4)
        prompt = (C.c_int32 * 3)(1, 2, 3)
        rid = C.c_uint64()
        ids, vals = (C.c_int32 * 2)(5, 5), (C.c_float * 2)(1.0, 2.0)
        pen = ffi.Penalties(0.0, 0.0, C.cast(ids, C.POINTER(C.c_int32)), C.cast(vals, C.POINTER(C.c_float)), 2)
        assert L.llmlb_request_submit_penalized(eng._h, prompt, 3, C.byref(s), C.byref(pen), C.byref(rid)) == ffi.E_INVALID_ARG
        assert "duplicate" in ffi.last_error()
        pen = ffi.Penalties(0.0, 0.0, None, None, 3)                           # NULL list with n_bias > 0
        assert L.llmlb_request_submit_penalized(eng._h, prompt, 3, C.byref(s), C.byref(pen), C.byref(rid)) == ffi.E_INVALID_ARG
        assert "logit_bias" in ffi.last_error()
        # the limits themselves are accepted, and so is NULL (no penalties)
        assert L.llmlb_request_submit_penalized(eng._h, prompt, 3, C.byref(s), None, C.byref(rid)) == ffi.OK
        HL.drain(eng, rid.value)
        eng.release(rid.value)
        for kw in (dict(frequency_penalty=2.0, presence_penalty=-2.0), dict(logit_bias={i: (100.0 if i % 2 else -100.0) for i in range(1024)}),
                   dict(logit_bias={0: 1.0, TINY["vocab"] - 1: -1.0})):
            rid2 = eng.submit([1, 2, 3], 4, **kw)
            assert HL.drain(eng, rid2)[-1]["finish_reason"] == HL.LENGTH
            eng.release(rid2)
        h = HL.settle(eng)
        assert h["free_kv_pages"] == h["total_kv_pages"]


def _tp_rank(rank, world, handles, barrier, name, out_q):
    try:
        os.environ["FAKE_CUDART_STEP_US"] = "200"
        ffi = HL._ffi()
        # 14 pages of 64 tokens for 6 sequences of 100 + 250 tokens: the youngest are evicted and recomputed
        eng = ffi.Engine(TINY, model_id="tp-pen", device=0, tp_rank=rank, tp_size=world, max_seqs=8, max_ctx=1024, kv_pages=14, seed=0)
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
            kws = [dict(frequency_penalty=0.5), {}, dict(presence_penalty=1.0, logit_bias={3: 5.0, 9: -5.0}), dict(logit_bias={7: 100.0}),
                   {}, dict(frequency_penalty=-0.5, presence_penalty=0.25)]
            rids = []
            for i, kw in enumerate(kws):
                rids.append(eng.submit([(5 * i + j) % TINY["vocab"] for j in range(100)], 250, ignore_eos=True, **kw))
                if i == 4:
                    eng.cancel(rids[1])
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
def test_scenario_two_rank_plan_channel_carries_penalties_through_preemption():
    """The leader logs penalised and unpenalised submits, a cancel, and evicts sequences from a small KV pool; the follower
    sees only the shared-memory log.  It must launch exactly what the leader launched — the penalty kernels included, which
    needs the penalties from the submit record — and end with the same counters and an empty pool."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    world = 2
    handles = ctx.Array("B", 64 * world)
    barrier = ctx.Barrier(world)
    q = ctx.Queue()
    name = "llmlb_pen_cpu_%d" % os.getpid()
    ps = [ctx.Process(target=_tp_rank, args=(r, world, handles, barrier, name, q)) for r in range(world)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=300) for _ in range(world))
    [p.join(60) for p in ps]
    assert all("error" not in v for v in got.values()), got
    lead, foll = got[0], got[1]
    assert lead["reasons"][1] == HL.CANCELLED and all(r == HL.LENGTH for i, r in enumerate(lead["reasons"]) if i != 1), lead
    assert lead["counters"]["preemptions"] > 0, lead
    assert lead["counters"] == foll["counters"], (lead["counters"], foll["counters"])
    assert lead["pages"] == foll["pages"] and lead["pages"][0] == lead["pages"][1] and lead["pages"][2:] == (0, 0)
    assert all(p.exitcode == 0 for p in ps)
