"""-m gpu: prompt logprobs from the served prefill (llmlb_request_submit_prompt_logprobs).  Every record against the
engine's own logits of the same prompt (llmlb_debug_prefill_logits: the same forward pass, so the checker's derived bound
of tests/logprob_oracle.py applies) on LLAMA_TINY and the Llama-3-8B geometry; against the fp64 oracle over prompts of
several prefill steps and several max_seqs groups, in steps shared with other requests whose tokens and records must not
move; greedy scoring (lm-eval's is_greedy) bit for bit; and lm-eval's request shape through the HTTP shim on the engine."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from llmlb_b200 import ffi  # noqa: E402
import logprob_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
TINY = ffi.LLAMA_TINY
LP_TOL = 0.06          # engine vs oracle log_softmax on this geometry (tests/test_logprobs_gpu.py)


def _served(e, prompt, n, max_tokens=2, **kw):
    """(generated events, prompt records) of one request, the records read right after its first event."""
    rid = e.submit(prompt, max_tokens, ignore_eos=True, logprobs=n, prompt_logprobs=True, **kw)
    evs, recs = [], None
    while not (evs and evs[-1]["finish_reason"]):
        got = e.poll_logprobs(rid, timeout_ms=-1)
        if got and recs is None:
            recs = e.poll_prompt_logprobs(rid, cap=1 << 16)
        evs += got
    assert e.poll_prompt_logprobs(rid) == []
    e.release(rid)
    return [x for x in evs if x["token_id"] >= 0], recs


def _rec(r):
    return dict(logprob=r["logprob"], n_top=len(r["top_logprobs"]), ids=[t for t, _ in r["top_logprobs"]],
                vals=[v for _, v in r["top_logprobs"]])


@pytest.mark.parametrize("model,n_prompt", [("tiny", 65), ("8b", 33)])
def test_records_pass_the_checker_against_the_engines_own_logits(built_lib, model, n_prompt):
    """One prefill step; n_prompt - 1 is a multiple of max_seqs = 8, so the served groups and the debug hook's groups hold
    the same rows and take the same lm_head path."""
    cfg = TINY if model == "tiny" else ffi.LLAMA3_8B
    V = cfg["vocab"]
    prompt = np.random.RandomState(V + n_prompt).randint(0, V, n_prompt).tolist()
    with ffi.Engine(cfg, max_seqs=8, max_ctx=256, seed=0) as e:
        for n in (0, 5, 20):
            _, recs = _served(e, prompt, n)
            assert len(recs) == n_prompt - 1
            e.debug_reset()
            _, raw = e.debug_prefill_logits(prompt, all_positions=True)
            e.debug_reset()
            for i, r in enumerate(recs):
                ok, why = O.check(raw[i], n, prompt[i + 1], _rec(r))
                assert ok, (model, n, i, why)


def _lsm(row):
    return O.log_softmax64(np.asarray(row, np.float32))


def _check_oracle(recs, prompt, ref_rows, n):
    for i, r in enumerate(recs):
        ref = _lsm(ref_rows[i])
        t = prompt[i + 1]
        assert abs(r["logprob"] - ref[t]) <= LP_TOL, (i, r["logprob"], ref[t])
        assert len(r["top_logprobs"]) == n
        kth = np.sort(ref)[::-1][n - 1] if n else None
        for j, (tid, v) in enumerate(r["top_logprobs"]):
            assert abs(v - ref[tid]) <= LP_TOL and ref[tid] >= kth - LP_TOL, (i, j, tid, v, ref[tid])
            if tid == t:
                assert np.float32(v).view(np.uint32) == np.float32(r["logprob"]).view(np.uint32)


def _batch(e, reqs):
    """reqs: (prompt, max_tokens, kw) submitted together; per request (events, prompt records or None)."""
    e.pause(True)
    rids = [e.submit(p, m, ignore_eos=True, **kw) for p, m, kw in reqs]
    e.pause(False)
    outs = []
    for r, (_, _, kw) in zip(rids, reqs):
        evs, recs = [], None
        while not (evs and evs[-1]["finish_reason"]):
            got = e.poll_logprobs(r, timeout_ms=-1) if kw.get("logprobs") is not None else e.poll(r, timeout_ms=-1)
            if got and recs is None and kw.get("prompt_logprobs"):
                recs = e.poll_prompt_logprobs(r, cap=1 << 16)
            evs += got
        e.release(r)
        key = [(x["token_id"], np.float32(x.get("logprob", np.nan)).tobytes(),
                [(t, np.float32(v).tobytes()) for t, v in x.get("top_logprobs", [])]) for x in evs if x["token_id"] >= 0]
        outs.append((key, recs))
    return outs


@pytest.mark.parametrize("max_seqs", [4, 8])
def test_chunked_prompt_in_a_shared_step_matches_the_oracle_and_moves_no_neighbour(built_lib, max_seqs):
    """A 150-token prompt over three 64-token prefill steps, scored beside a sampled neighbour and a logprob neighbour that
    share those steps: its records against the fp64 oracle's logits of every position; its own generated tokens and records,
    and the neighbours', bit-identical to the same batch without prompt logprobs."""
    from oracle.llama_ref import LlamaRef
    from oracle.synth import synth_state_dict
    rs = np.random.RandomState(21)
    prompt = rs.randint(0, TINY["vocab"], 150).tolist()
    nb = [rs.randint(0, TINY["vocab"], 40 + 17 * i).tolist() for i in range(2)]
    with ffi.Engine(TINY, max_seqs=max_seqs, max_ctx=512, max_step_tokens=64, seed=0) as e:
        def run(flag):
            kw = dict(logprobs=4, **(dict(prompt_logprobs=True) if flag else {}))
            return _batch(e, [(nb[0], 12, dict(temperature=0.9, top_p=0.95, seed=5)), (prompt, 12, kw), (nb[1], 12, dict(logprobs=3))])
        with_p, without = run(True), run(False)
    assert [k for k, _ in with_p] == [k for k, _ in without]
    recs = with_p[1][1]
    assert len(recs) == len(prompt) - 1
    ref = LlamaRef(TINY, synth_state_dict(TINY, 0)).forward(prompt).numpy()
    _check_oracle(recs, prompt, ref, 4)


def test_greedy_continuations_are_their_rows_top_entry_bit_for_bit(built_lib):
    """lm-eval's is_greedy: score a seed followed by its own greedy continuation.  Each continuation token is its row's
    arg-max, so its record must list it first with the very same value; the served prompt records also match the logprob
    records the generation reported for the same tokens, within the logits' tolerance."""
    rs = np.random.RandomState(4)
    seed = rs.randint(0, TINY["vocab"], 30).tolist()
    with ffi.Engine(TINY, max_seqs=8, max_ctx=512, seed=0) as e:
        toks, evs = e.generate(seed, 24, ignore_eos=True, logprobs=5)
        evs = [x for x in evs if x["token_id"] >= 0]
        _, recs = _served(e, seed + toks, 5, max_tokens=1)
    cont = recs[len(seed) - 1:]
    assert len(cont) == len(toks)
    greedy = 0
    for t, r, g in zip(toks, cont, evs):
        tid, v = r["top_logprobs"][0]
        if tid == t:
            greedy += 1
            assert np.float32(v).view(np.uint32) == np.float32(r["logprob"]).view(np.uint32)
        else:   # a tie with a lower id
            assert np.float32(v) == np.float32(r["logprob"]), (t, r["top_logprobs"][:2])
        assert abs(r["logprob"] - g["logprob"]) <= LP_TOL
    assert greedy >= len(toks) - 2


def test_lm_eval_request_shape_through_the_server(built_lib):
    import test_server_gpu as S
    from llmlb_b200 import build
    build.build_host()
    port = S._free_port()
    proc = subprocess.Popen([S.BIN, "--port", str(port), "--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8",
                             "--max-ctx", "512"], stderr=subprocess.PIPE)
    try:
        deadline = time.time() + 120
        while time.time() < deadline:
            try:
                S.call(port, "GET", "/v1/models")
                break
            except OSError:
                assert proc.poll() is None, proc.stderr.read().decode()
                time.sleep(0.2)
        ids = np.random.RandomState(2).randint(3, 2000, 41).tolist()
        body = {"model": "tiny-llama", "prompt": [ids], "echo": True, "logprobs": 1, "max_tokens": 1, "temperature": 0}
        st, _, d = S.call(port, "POST", "/v1/completions", body)
        assert st == 200, d
        lp = json.loads(d)["choices"][0]["logprobs"]
        assert len(lp["tokens"]) == len(lp["token_logprobs"]) == len(lp["top_logprobs"]) == len(ids) + 1
        assert lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None
        for v, top in zip(lp["token_logprobs"][1:], lp["top_logprobs"][1:]):
            assert v <= 0 and len(top) == 1 and max(top.values()) >= v
        assert lp["text_offset"] == sorted(lp["text_offset"])
    finally:
        proc.terminate()
        proc.wait(timeout=20)
