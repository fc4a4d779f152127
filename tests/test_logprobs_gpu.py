"""-m gpu: token logprobs on the device.  llmlb_op_logprobs against the float64 definition of tests/logprob_oracle.py at
every vocabulary the engine samples (and 32003 and 7), on LM-like rows, all-equal rows, -inf entries, logits around
+-1e30, a dominant token and skipped rows, inside NaN guard bands; then the engine on LLAMA_TINY and the Llama-3-8B
geometry: greedy tokens are the top entry, values teacher-forced against the oracle and against the engine's own prefill
logits, a +100 bias and the penalties, neighbours without logprobs untouched, preemption, graphs against eager."""
import math

import numpy as np
import pytest
import torch

from llmlb_b200 import ffi
import logprob_oracle as O
from penalty_oracle import penalize

pytestmark = pytest.mark.gpu
TINY = ffi.LLAMA_TINY
LOGIT_TOL = 0.03       # engine vs oracle logits on this geometry (tests/test_engine_gpu.py)
LP_TOL = 2 * LOGIT_TOL  # a log_softmax moves by at most twice the largest logit error
GUARD = 64             # NaN words before and after every buffer the kernel writes
VOCABS = O.VOCABS
lm_row = O.lm_row
N_ROWS = 9
OP_CASES = [(N_ROWS, V) for V in VOCABS]
REC_WORDS = 42         # sizeof(llmlb_token_logprobs) / 4
NAN_BITS = 0x7FC00000


def _rows(V, n, rs):
    """(logits [N_ROWS, V], top_n [N_ROWS], tokens [N_ROWS]); rows 5 and 8 are skipped."""
    rows = [lm_row(V, rs), np.zeros(V, np.float32)]
    z = lm_row(V, rs)
    z[rs.choice(V, max(1, V // 10), replace=False)] = -np.inf
    z[int(np.argmax(z))] = 3.0                              # the maximum stays finite
    rows.append(z)
    big = np.where(rs.rand(V) < 0.5, np.float32(1e30), np.float32(-1e30)).astype(np.float32)
    big *= (1 + rs.rand(V).astype(np.float32) * np.float32(1e-3))
    rows.append(big.astype(np.float32))
    z = lm_row(V, rs)
    z[V // 3] += np.float32(100)                            # what a +100 logit bias does
    rows.append(z)
    rows.append(lm_row(V, rs))
    z = lm_row(V, rs)                                       # ties straddling the n-th place
    top = O.top_ids(z, 3)
    z[rs.choice(V, min(V, 6), replace=False)] = z[top[-1]]
    rows.append(z)
    z = np.full(V, -7.5, np.float32)
    z[rs.choice(V, min(V, 3), replace=False)] = -7.25
    rows.append(z)
    rows.append(lm_row(V, rs))
    top_n = np.full(N_ROWS, n, np.int32)
    top_n[[5, 8]] = -1
    tokens = np.array([int(np.argmax(r)) if i % 2 == 0 else int(rs.choice(np.nonzero(np.isfinite(r))[0]))
                       for i, r in enumerate(rows)], np.int32)
    return np.stack(rows), top_n, tokens


def _records(words):
    """int32 [R, 42] -> list of {logprob, n_top, ids, vals}"""
    out = []
    for w in words:
        out.append(dict(logprob=w[0:1].view(np.float32)[0], n_top=int(w[1]), ids=w[2:22].copy(), vals=w[22:42].view(np.float32).copy()))
    return out


def run_op(logits, top_n, tokens):
    R, V = logits.shape
    d_lg = torch.full((GUARD + R * V + GUARD,), float("nan"), device="cuda")
    d_lg[GUARD:GUARD + R * V] = torch.from_numpy(logits.ravel()).cuda()
    d_top, d_tok = torch.from_numpy(top_n).cuda(), torch.from_numpy(tokens).cuda()
    d_rec = torch.full((GUARD + R * REC_WORDS + GUARD,), NAN_BITS, dtype=torch.int32, device="cuda")
    before = (d_lg.clone(), d_top.clone(), d_tok.clone())
    rc = ffi.lib().llmlb_op_logprobs(d_lg.data_ptr() + GUARD * 4, R, V, d_tok.data_ptr(), d_top.data_ptr(), d_rec.data_ptr() + GUARD * 4, None)
    assert rc == 0, ffi.last_error()
    torch.cuda.synchronize()
    assert torch.equal(before[0].view(torch.int32), d_lg.view(torch.int32)) and torch.equal(before[1], d_top) and torch.equal(before[2], d_tok)
    w = d_rec.cpu().numpy()
    assert (w[:GUARD] == NAN_BITS).all() and (w[-GUARD:] == NAN_BITS).all()
    return w[GUARD:GUARD + R * REC_WORDS].reshape(R, REC_WORDS)


# ---- the kernel -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 5, 20])
@pytest.mark.parametrize("V", VOCABS)
def test_op_logprobs_against_float64(built_lib, V, n):
    logits, top_n, tokens = _rows(V, n, np.random.RandomState(V + n))
    words = run_op(logits, top_n, tokens)
    for r, rec in enumerate(_records(words)):
        if top_n[r] < 0:
            assert (words[r] == NAN_BITS).all(), "a skipped row's record was written"
            continue
        ok, why = O.check(logits[r], n, int(tokens[r]), rec)
        assert ok, (r, why)
        k = rec["n_top"]
        assert (rec["ids"][k:] == -1).all() and (rec["vals"][k:] == 0).all()
        assert not np.isnan(rec["vals"][:k]).any() and not np.isnan(rec["logprob"])
        assert (rec["vals"][:k] <= 0).all() and rec["logprob"] <= 0
    recs = _records(words)
    if n:   # all-equal row: the lowest ids, each log(1/V)
        assert recs[1]["ids"][:recs[1]["n_top"]].tolist() == list(range(min(n, V)))
    dom = recs[4]                                            # the dominant token: at the top, logprob <= 0 and about 0
    if n:
        assert dom["ids"][0] == V // 3 and -1e-3 <= dom["vals"][0] <= 0
    if V > 20:
        assert recs[2]["n_top"] == n
    else:
        assert recs[0]["n_top"] == min(n, V)


def test_op_logprobs_n_above_20_is_capped_and_small_vocab_lists_everything(built_lib):
    rs = np.random.RandomState(3)
    for V, n, want in ((7, 25, 7), (7, 7, 7), (4096, 25, 20), (3, 20, 3)):
        z = lm_row(V, rs)
        words = run_op(z[None, :], np.array([n], np.int32), np.array([int(np.argmax(z))], np.int32))
        rec = _records(words)[0]
        assert rec["n_top"] == want
        assert O.check(z, n, int(np.argmax(z)), rec)[0]


def test_op_logprobs_is_deterministic_and_rows_are_independent(built_lib):
    rs = np.random.RandomState(11)
    logits, top_n, tokens = _rows(128256, 20, rs)
    a = run_op(logits, top_n, tokens)
    b = run_op(logits, top_n, tokens)
    assert np.array_equal(a, b)
    for r in (0, 3, 7):
        one = run_op(logits[r:r + 1].copy(), top_n[r:r + 1].copy(), tokens[r:r + 1].copy())
        assert np.array_equal(one[0], a[r])


def test_op_logprobs_refuses_bad_arguments(built_lib):
    L = ffi.lib()
    t = torch.zeros(64, device="cuda")
    p = t.data_ptr()
    assert L.llmlb_op_logprobs(None, 1, 8, p, p, p, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_logprobs(p, 1, 0, p, p, p, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_logprobs(p, 1, 8, None, p, p, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_logprobs(p, 1, 8, p, None, p, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_logprobs(p, 1, 8, p, p, None, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_logprobs(p, 0, 8, p, p, p, None) == ffi.OK


# ---- the engine -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng(built_lib):
    e = ffi.Engine(TINY, max_seqs=8, max_ctx=1024, seed=0)
    yield e
    e.close()


def _lsm(row):
    return O.log_softmax64(np.asarray(row, np.float32))


def _check_against_rows(toks, evs, rows, n):
    """Each event's record against log_softmax of its logits row (rows[i] produced toks[i]) within LP_TOL: the token's
    value, the listed values, and the listed ids being within LP_TOL of the row's n best."""
    assert len(evs) == len(toks) == len(rows)
    for i, (t, e, row) in enumerate(zip(toks, evs, rows)):
        ref = _lsm(row)
        assert e["token_id"] == t and abs(e["logprob"] - ref[t]) <= LP_TOL, (i, e["logprob"], ref[t])
        top = e["top_logprobs"]
        assert len(top) == n
        kth = np.sort(ref)[::-1][n - 1] if n else None
        for j, (tid, v) in enumerate(top):
            assert abs(v - ref[tid]) <= LP_TOL, (i, j, tid, v, ref[tid])
            assert ref[tid] >= kth - LP_TOL
            if j:
                assert v <= top[j - 1][1]
            if tid == t:
                assert np.float32(v).view(np.uint32) == np.float32(e["logprob"]).view(np.uint32)


def _greedy_is_top(toks, evs):
    for t, e in zip(toks, evs):
        tid, v = e["top_logprobs"][0]
        assert tid == t or np.float32(e["logprob"]) == np.float32(v), (t, e["top_logprobs"][:3])


def test_greedy_tokens_are_the_top_entry_and_match_the_oracle_tiny(eng):
    from oracle.llama_ref import LlamaRef
    from oracle.synth import synth_state_dict
    prompt = np.random.RandomState(0).randint(0, TINY["vocab"], 70).tolist()
    toks, evs = eng.generate(prompt, 16, ignore_eos=True, logprobs=5)
    evs = [e for e in evs if e["token_id"] >= 0]
    _greedy_is_top(toks, evs)
    ref = LlamaRef(TINY, synth_state_dict(TINY, 0))
    rows = [ref.forward(prompt).numpy()[-1]]
    for t in toks[:-1]:
        rows.append(ref.forward([t]).numpy()[-1])
    _check_against_rows(toks, evs, rows, 5)


@pytest.mark.parametrize("model", ["tiny", "8b"])
def test_teacher_forced_logprobs_bias_and_penalties(built_lib, model):
    """Records against log_softmax of the engine's own logits (a prefill, then teacher-forced batch-1 decode steps) after
    penalize() (tests/penalty_oracle.py) with the counts of the tokens generated so far: plain, with penalties and a bias,
    and a +100 bias whose token gets about 0."""
    cfg = TINY if model == "tiny" else ffi.LLAMA3_8B
    V = cfg["vocab"]
    with ffi.Engine(cfg, max_seqs=4, max_ctx=256, seed=0) as e:
        prompt = np.random.RandomState(V).randint(0, V, 40).tolist()
        for f, p, bias, n in ((0.0, 0.0, {}, 20), (0.7, 0.4, {3: 2.5, V - 1: -1.0}, 5), (0.0, 0.0, {V // 2: 100.0}, 1)):
            kw = dict(frequency_penalty=f, presence_penalty=p, logit_bias=bias) if (f or p or bias) else {}
            toks, evs = e.generate(prompt, 12, ignore_eos=True, logprobs=n, **kw)
            evs = [x for x in evs if x["token_id"] >= 0]
            _greedy_is_top(toks, evs)
            e.debug_reset()                      # the prefill and batch-1 decode paths the generation took
            raw = [e.debug_prefill_logits(prompt)] + [e.debug_decode_logits(t) for t in toks[:-1]]
            e.debug_reset()
            counts = np.zeros(V, np.int64)
            rows = []
            for i, t in enumerate(toks):
                rows.append(penalize(raw[i], counts, f, p, bias))
                counts[t] += 1
            _check_against_rows(toks, evs, rows, n)
            if bias.get(V // 2) == 100.0:
                assert toks == [V // 2] * 12
                assert all(-1e-4 <= x["logprob"] <= 0 and x["top_logprobs"][0][0] == V // 2 for x in evs), evs[:2]


def _batch(e, reqs, lp=False):
    e.pause(True)
    rids = [e.submit(p, n, ignore_eos=True, **kw) for p, n, kw in reqs]
    e.pause(False)
    outs = []
    for r, (_, _, kw) in zip(rids, reqs):
        evs = []
        while True:
            ev = e.poll_logprobs(r, timeout_ms=-1) if lp else e.poll(r, timeout_ms=-1)
            evs += [x for x in ev if x["token_id"] >= 0]
            if ev and ev[-1]["finish_reason"]:
                break
        e.release(r)
        outs.append(evs)
    return outs


def test_neighbours_without_logprobs_are_bit_identical(eng):
    rs = np.random.RandomState(5)
    a, b = (rs.randint(0, TINY["vocab"], 30 + 9 * i).tolist() for i in range(2))
    samp = dict(temperature=0.9, top_p=0.95, seed=77)
    for w in (2, 3, 6):   # GEMV (<= 4 rows) and tensor-core batches
        plain = _batch(eng, [(a, 24, {})] + [(b, 24, samp)] * (w - 1))
        mixed = _batch(eng, [(a, 24, dict(logprobs=20))] + [(b, 24, samp)] * (w - 1), lp=True)
        assert [x["token_id"] for x in mixed[0]] == [x["token_id"] for x in plain[0]]
        assert [[x["token_id"] for x in o] for o in mixed[1:]] == [[x["token_id"] for x in o] for o in plain[1:]], w
        assert all(math.isnan(x["logprob"]) and x["top_logprobs"] == [] for o in mixed[1:] for x in o)
        assert all(len(x["top_logprobs"]) == 20 for x in mixed[0])


def test_records_survive_preemption(built_lib):
    """Four logprob sequences share a pool of 9 pages: some are evicted and recomputed, and the first token after a
    re-admission takes its record from the prefill step.  Every record must still match its teacher-forced row."""
    rs = np.random.RandomState(9)
    prompts = [rs.randint(0, TINY["vocab"], 90).tolist() for _ in range(4)]
    with ffi.Engine(TINY, max_seqs=4, max_ctx=512, kv_pages=9, seed=0) as e:
        outs = _batch(e, [(q, 120, dict(logprobs=3)) for q in prompts], lp=True)
        assert e.health()["preemptions"] > 0, "the pool was sized to force evictions"
        for q, evs in zip(prompts, outs):
            toks = [x["token_id"] for x in evs]
            assert len(toks) == 120
            _greedy_is_top(toks, evs)
            e.debug_reset()
            _, raw = e.debug_prefill_logits(q + toks[:-1], all_positions=True)
            e.debug_reset()
            _check_against_rows(toks, evs, [raw[len(q) - 1 + i] for i in range(len(toks))], 3)


def test_graphs_and_eager_give_the_same_records(built_lib):
    rs = np.random.RandomState(13)
    reqs = [(rs.randint(0, TINY["vocab"], 20 + 5 * i).tolist(), 30,
             dict(logprobs=(i * 7) % 21, temperature=0.8, seed=i, **(dict(presence_penalty=0.4) if i % 3 == 0 else {})) if i % 2 == 0 else {})
            for i in range(6)]
    got = []
    for graphs in (True, False):
        with ffi.Engine(TINY, max_seqs=8, max_ctx=512, seed=0, use_cuda_graphs=graphs) as e:
            got.append([[(x["token_id"], np.float32(x["logprob"]).tobytes(), [(t, np.float32(v).tobytes()) for t, v in x["top_logprobs"]])
                         for x in o] for o in _batch(e, reqs, lp=True)])
    assert got[0] == got[1]
