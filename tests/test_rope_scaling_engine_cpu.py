"""llmlb_engine_set_rope_freq_factors over the fake CUDA runtime (tests/support/fake_cudart.cpp): argument checks,
the rule that the table is fixed once a request or a debug call has run, one table-kernel launch per call, and a launch
list of every prefill and decode step that is the same with and without factors (RoPE scaling adds nothing to the hot
path: the step kernels read the same table, only its contents differ).

Like test_engine_host_logic_cpu.py, the outer test re-runs this file in a child process that preloads the fake runtime."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INNER = os.environ.get("LLMLB_FAKE_CUDART") == "1"
inner = pytest.mark.skipif(not INNER, reason="runs in the child process that preloads the fake CUDA runtime")
TINY = dict(hidden=512, n_layers=2, n_heads=8, n_kv_heads=2, head_dim=128, ffn=1024, vocab=2048, rope_theta=500000.0, rms_eps=1e-5)
LLAMA31 = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}


def test_rope_factor_setter_over_the_fake_cuda_runtime(built_lib, tmp_path):
    if INNER:
        pytest.skip("already inside")
    sys.path.insert(0, HERE)
    from test_engine_host_logic_cpu import build_fake
    log = tmp_path / "launches.log"
    from rope_oracle import rope_freq_factors      # torch cannot be imported in the child: the factors travel in the environment
    factors = json.dumps([float(x) for x in rope_freq_factors(LLAMA31, TINY["rope_theta"])])
    env = dict(os.environ, LD_PRELOAD=build_fake(), LLMLB_FAKE_CUDART="1", FAKE_CUDART_LAUNCH_LOG=str(log), ROPE_TEST_FACTORS=factors)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-p", "no:cacheprovider", "-k", "scenario"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-500:]


def _log_lines():
    with open(os.environ["FAKE_CUDART_LAUNCH_LOG"]) as f:
        return f.read().splitlines()


def _factors():
    return json.loads(os.environ["ROPE_TEST_FACTORS"])


@inner
def test_scenario_setter_checks_its_arguments_and_launches_one_table_kernel():
    from llmlb_b200 import ffi
    good = _factors()
    with ffi.Engine(TINY, max_seqs=4, max_ctx=1024) as eng:
        for bad in (good[:63], good + [1.0], []):
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.set_rope_freq_factors(bad)
            assert ei.value.code == ffi.E_INVALID_ARG and "64" in str(ei.value)
        for v in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
            f = list(good)
            f[17] = v
            with pytest.raises(ffi.LlmlbError) as ei:
                eng.set_rope_freq_factors(f)
            assert ei.value.code == ffi.E_INVALID_ARG and "factor 17" in str(ei.value)
        n0 = len(_log_lines())
        eng.set_rope_freq_factors(good)
        eng.set_rope_freq_factors([1.0] * 64)          # any number of times before the first request
        new = _log_lines()[n0:]
        assert len(new) == 2 and all("rope_table_kernel" in l for l in new), new
        eng.generate(list(range(1, 40)), 3, ignore_eos=True)
        with pytest.raises(ffi.LlmlbError) as ei:
            eng.set_rope_freq_factors(good)
        assert ei.value.code == ffi.E_UNSUPPORTED
    # a debug forward fixes the table too
    with ffi.Engine(TINY, max_seqs=4, max_ctx=1024) as eng:
        eng.debug_prefill_logits(list(range(1, 20)))
        with pytest.raises(ffi.LlmlbError) as ei:
            eng.set_rope_freq_factors(good)
        assert ei.value.code == ffi.E_UNSUPPORTED
    # and the constructor argument sets them before anything else runs
    with ffi.Engine(TINY, max_seqs=4, max_ctx=1024, rope_freq_factors=good) as eng:
        eng.generate([1, 2, 3], 2, ignore_eos=True)
    with pytest.raises(ffi.LlmlbError):
        ffi.Engine(TINY, max_seqs=4, max_ctx=1024, rope_freq_factors=[0.0] * 64)


@inner
def test_scenario_step_launch_list_is_the_same_with_and_without_factors():
    """Chunked prefill (a 2600-token prompt over 1024-token steps), batched prefill and decode, with and without CUDA
    graphs: every kernel launch after engine creation is identical, name, grid, block and shared memory."""
    from llmlb_b200 import ffi

    def steps(factors, graphs):
        with ffi.Engine(TINY, max_seqs=4, max_ctx=4096, max_step_tokens=1024, use_cuda_graphs=graphs) as eng:
            if factors:
                eng.set_rope_freq_factors(factors)
            n0 = len(_log_lines())
            eng.generate([i % 2000 + 1 for i in range(2600)], 5, ignore_eos=True)
            eng.pause(True)                                  # one queue, so that both runs batch the same way
            rids = [eng.submit(list(range(3, 3 + n)), 6, ignore_eos=True) for n in (17, 130, 64)]
            eng.pause(False)
            for rid in rids:
                while not any(e["finish_reason"] for e in eng.poll(rid, timeout_ms=50)):
                    pass
                eng.release(rid)
            return _log_lines()[n0:]

    for graphs in (False, True):
        plain, scaled = steps(None, graphs), steps(_factors(), graphs)
        assert len(plain) > 20
        assert not any("rope_table_kernel" in l for l in plain)
        assert plain == scaled
