"""-m gpu: frequency / presence penalties and logit bias on the device.  llmlb_op_penalize against the float32 restatement
of tests/penalty_oracle.py bit for bit; forcing and banning tokens with a bias on LLAMA_TINY and the Llama-3-8B geometry;
teacher-forced penalised generation (each token the arg-max, or the sampler's draw, of the penalised raw logits);
isolation of unpenalised neighbours and of a slot's next occupant; penalties across a preemption; graphs against eager."""
import numpy as np
import pytest
import torch

from llmlb_b200 import ffi
from oracle.sampling_ref import sample
from penalty_oracle import penalize

pytestmark = pytest.mark.gpu
TINY = ffi.LLAMA_TINY
LOGIT_TOL = 0.03       # engine vs oracle logits on this geometry (tests/test_engine_gpu.py); decode vs prefill path: less
LOGIT_TOL_EMULATED = 0.012   # the same with only the accumulation order differing
GUARD = 64             # NaN floats before and after every buffer the kernel writes


def _ptr(t):
    return t.data_ptr()


# ---- the kernel -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vocab,stride_pad", [(128256, 0), (128256, 3), (1001, 0), (7, 1)])
def test_op_penalize_is_bit_exact(built_lib, vocab, stride_pad):
    """Rows 1 and 4 are not penalised (their counts are not zero) and must come back bit-unchanged; the others mix positive
    and negative penalties, counts up to 131071 and biases of +-100 on ids 0 and vocab - 1.  stride_pad != 0 makes the
    count rows unaligned (the scalar path)."""
    rs = np.random.RandomState(vocab + stride_pad)
    n_rows, stride, bias_stride = 6, vocab + stride_pad, 16
    logits = (rs.randn(n_rows, vocab) * 5).astype(np.float32)
    counts = (rs.randint(0, 4, (n_rows, stride)) * (rs.rand(n_rows, stride) < 0.2)).astype(np.int32)
    counts[:, 0] = 131071
    counts[:, min(2, vocab - 1)] = 65536
    freq = np.array([0.7, 0.0, -0.5, 2.0, 0.0, 0.0], np.float32)
    pres = np.array([0.0, 0.0, 0.8, -2.0, 0.0, 1.5], np.float32)
    n_bias = np.array([2, 0, 0, 5, 0, 3], np.uint32)
    bias_ids = np.zeros((n_rows, bias_stride), np.int32)
    bias_vals = np.full((n_rows, bias_stride), np.nan, np.float32)       # entries past n_bias must never be read
    biases = []
    for r in range(n_rows):
        ids = [0, vocab - 1] + [int(x) for x in rs.choice(np.arange(1, vocab - 1), min(int(n_bias[r]), vocab - 2), replace=False)]
        ids = ids[:n_bias[r]]
        vals = [100.0, -100.0] + list(rs.uniform(-100, 100, 8).astype(np.float32))
        vals = [float(np.float32(v)) for v in vals[:n_bias[r]]]
        bias_ids[r, :len(ids)], bias_vals[r, :len(vals)] = ids, vals
        biases.append(dict(zip(ids, vals)))
    nan = float("nan")
    d_logits = torch.full((GUARD + n_rows * vocab + GUARD,), nan, device="cuda")
    d_logits[GUARD:GUARD + n_rows * vocab] = torch.from_numpy(logits.ravel()).cuda()
    ins = [torch.from_numpy(a.ravel().copy()).cuda() for a in (counts, freq, pres, bias_ids, bias_vals)]
    d_nb = torch.from_numpy(n_bias.astype(np.int32)).cuda()
    before = [t.clone() for t in ins] + [d_nb.clone()]
    rc = ffi.lib().llmlb_op_penalize(_ptr(d_logits) + GUARD * 4, n_rows, vocab, _ptr(ins[0]), stride, _ptr(ins[1]), _ptr(ins[2]),
                                     _ptr(ins[3]), _ptr(ins[4]), _ptr(d_nb), bias_stride, None)
    assert rc == 0, ffi.last_error()
    torch.cuda.synchronize()
    out = d_logits.cpu().numpy()
    assert np.isnan(out[:GUARD]).all() and np.isnan(out[-GUARD:]).all()
    got = out[GUARD:GUARD + n_rows * vocab].reshape(n_rows, vocab)
    for r in range(n_rows):
        want = penalize(logits[r], counts[r, :vocab], freq[r], pres[r], biases[r])
        assert np.array_equal(got[r].view(np.int32), want.view(np.int32)), (r, np.flatnonzero(got[r] != want)[:8])
    assert np.array_equal(got[1].view(np.int32), logits[1].view(np.int32)) and np.array_equal(got[4].view(np.int32), logits[4].view(np.int32))
    for a, b in zip(before, ins + [d_nb]):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)


def test_op_penalize_refuses_bad_arguments(built_lib):
    L = ffi.lib()
    t = torch.zeros(64, device="cuda")
    assert L.llmlb_op_penalize(None, 1, 8, _ptr(t), 8, _ptr(t), _ptr(t), None, None, _ptr(t), 0, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_penalize(_ptr(t), 1, 8, _ptr(t), 7, _ptr(t), _ptr(t), None, None, _ptr(t), 0, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_penalize(_ptr(t), 1, 8, _ptr(t), 8, _ptr(t), _ptr(t), None, None, _ptr(t), 4, None) == ffi.E_INVALID_ARG
    assert L.llmlb_op_penalize(_ptr(t), 1, 8, _ptr(t), 8, _ptr(t), _ptr(t), _ptr(t), _ptr(t), _ptr(t), 1025, None) == ffi.E_INVALID_ARG


# ---- the engine -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng(built_lib):
    e = ffi.Engine(TINY, max_seqs=8, max_ctx=1024, seed=0)
    yield e
    e.close()


def _forcing(e, vocab):
    rs = np.random.RandomState(vocab)
    prompt = rs.randint(0, vocab, 40).tolist()
    for t in (1234 % vocab, vocab - 1, 0):
        toks, _ = e.generate(prompt, 12, ignore_eos=True, logit_bias={t: 100.0})
        assert toks == [t] * 12, (t, toks)
    e.debug_reset()
    raw = e.debug_prefill_logits(prompt)
    e.debug_reset()
    first = e.generate(prompt, 1, ignore_eos=True)[0][0]
    assert raw[first] >= raw.max() - 2 * LOGIT_TOL
    banned = e.generate(prompt, 1, ignore_eos=True, logit_bias={first: -100.0})[0][0]
    runner_up = raw.copy()
    runner_up[first] = -np.inf
    assert banned != first and runner_up[banned] >= runner_up.max() - 2 * LOGIT_TOL, (banned, first)


def test_bias_forces_and_bans_tokens_tiny(eng):
    _forcing(eng, TINY["vocab"])


def test_bias_forces_and_bans_tokens_8b(built_lib):
    with ffi.Engine(ffi.LLAMA3_8B, max_seqs=4, max_ctx=256, seed=0) as e:
        _forcing(e, ffi.LLAMA3_8B["vocab"])


CASES = [(0.7, 0.0, {}), (0.0, 1.5, {}), (-0.5, 0.8, {}), (0.7, 0.0, {3: 2.5, 100: -1.0})]


def _teacher_forced(e, prompt, toks, f, p, bias, sampled=None):
    """toks[i] must be the arg-max (or the draw) of penalize(raw logits after prompt + toks[:i], counts of toks[:i]).
    Returns the number of steps where the penalties changed the arg-max of the raw logits."""
    e.debug_reset()
    _, rows = e.debug_prefill_logits(prompt + toks[:-1], all_positions=True)
    e.debug_reset()
    counts = np.zeros(TINY["vocab"], np.int64)
    changed = checked = 0
    for i, t in enumerate(toks):
        raw = rows[len(prompt) - 1 + i]
        z = penalize(raw, counts, f, p, bias)
        changed += int(np.argmax(z) != np.argmax(raw))
        if sampled is None:
            assert z[t] >= z.max() - 2 * LOGIT_TOL, (i, t, int(np.argmax(z)))
        else:
            # the engine sampled decode-path logits, these are prefill-path ones: a step is decided only when the draw is the
            # same under perturbations of that size (CDF edges, and the top-k / top-p sets changing at a near-tie)
            temp, top_k, top_p, seed = sampled
            want = sample(z, temp, top_k, top_p, seed, i)[0]
            rs = np.random.RandomState(i)
            if all(sample(z + np.float32(LOGIT_TOL_EMULATED) * rs.uniform(-1, 1, z.size).astype(np.float32), temp, top_k, top_p, seed, i)[0] == want
                   for _ in range(8)):
                assert t == want, (i, t, want)
                checked += 1
        counts[t] += 1
    if sampled is not None:
        assert checked >= len(toks) // 3, checked
    return changed


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("mode", ["greedy", "sampled"])
def test_teacher_forced_penalised_generation(eng, case, mode):
    f, p, bias = CASES[case]
    prompt = np.random.RandomState(50 + case).randint(0, TINY["vocab"], 40).tolist()
    sampled = None if mode == "greedy" else (1.0, 8, 0.9, 1000 + case)
    kw = dict(temperature=0.0) if mode == "greedy" else dict(temperature=1.0, top_k=8, top_p=0.9, seed=1000 + case)
    toks, _ = eng.generate(prompt, 32, ignore_eos=True, frequency_penalty=f, presence_penalty=p, logit_bias=bias, **kw)
    assert len(toks) == 32
    changed = _teacher_forced(eng, prompt, toks, f, p, bias, sampled)
    if mode == "greedy" and f > 0:
        assert changed > 0, "the penalty never acted: the check would not see it missing"


def _batch(e, reqs):
    e.pause(True)
    rids = [e.submit(p, n, ignore_eos=True, **kw) for p, n, kw in reqs]
    e.pause(False)
    outs = []
    for r in rids:
        toks = []
        while True:
            ev = e.poll(r, timeout_ms=-1)
            toks += [x["token_id"] for x in ev if x["token_id"] >= 0]
            if ev and ev[-1]["finish_reason"]:
                break
        e.release(r)
        outs.append(toks)
    return outs


def test_unpenalised_neighbours_and_next_occupants_are_unaffected(eng, built_lib):
    rs = np.random.RandomState(5)
    a, b, c = (rs.randint(0, TINY["vocab"], 30 + 9 * i).tolist() for i in range(3))
    pen = dict(frequency_penalty=2.0, presence_penalty=2.0, logit_bias={7: 50.0})
    samp = dict(temperature=0.9, top_p=0.95, seed=77)
    for w in (2, 3, 6):   # GEMV (<= 4 rows) and tensor-core batches
        plain = _batch(eng, [(a, 24, {})] + [(b, 24, samp)] * (w - 1))
        mixed = _batch(eng, [(a, 24, pen)] + [(b, 24, samp)] * (w - 1))
        assert mixed[0] != plain[0]
        assert mixed[1:] == plain[1:], w
    with ffi.Engine(TINY, max_seqs=1, max_ctx=512, seed=0) as e:    # one slot: every request takes it after the previous one
        before = e.generate(c, 24, ignore_eos=True)[0]
        e.generate(a, 40, ignore_eos=True, **pen)
        assert e.generate(c, 24, ignore_eos=True)[0] == before
        assert e.generate(c, 24, ignore_eos=True, **samp)[0] == e.generate(c, 24, ignore_eos=True, **samp)[0]


def test_penalties_survive_preemption(built_lib):
    """Four penalised sequences share a pool of 9 pages: some are evicted and recomputed.  The counts rebuilt at
    re-admission must give the same teacher-forced tokens as if nothing had happened."""
    rs = np.random.RandomState(9)
    prompts = [rs.randint(0, TINY["vocab"], 90).tolist() for _ in range(4)]
    f, p = 0.7, 0.3
    with ffi.Engine(TINY, max_seqs=4, max_ctx=512, kv_pages=9, seed=0) as e:
        outs = _batch(e, [(q, 120, dict(frequency_penalty=f, presence_penalty=p)) for q in prompts])
        assert e.health()["preemptions"] > 0, "the pool was sized to force evictions"
        for q, toks in zip(prompts, outs):
            assert len(toks) == 120
            _teacher_forced(e, q, toks, f, p, {})


def test_graphs_and_eager_give_the_same_tokens(built_lib):
    rs = np.random.RandomState(13)
    reqs = [(rs.randint(0, TINY["vocab"], 20 + 5 * i).tolist(), 30,
             dict(frequency_penalty=0.5 * (i % 3), presence_penalty=0.4, logit_bias={i: 3.0}, temperature=0.8, seed=i) if i % 2 else {})
            for i in range(6)]
    got = []
    for graphs in (True, False):
        with ffi.Engine(TINY, max_seqs=8, max_ctx=512, seed=0, use_cuda_graphs=graphs) as e:
            got.append(_batch(e, reqs))
    assert got[0] == got[1]
