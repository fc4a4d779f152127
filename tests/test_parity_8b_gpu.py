"""The SURVEY.md §8d parity set at FULL Llama-3-8B geometry: 8 prompts x 512 tokens x 32 greedy steps
against the CPU oracle that rounds activations to bf16 where the kernels do
(oracle/llama_ref.py, emulate_bf16=True, C/OpenMP bf16 linears).  Three legs over the same prompts:

  batch 1      parity hooks (llmlb_debug_prefill_logits / llmlb_debug_decode_logits): per-step logits
               -> max-abs and mean-abs error, top-1 agreement, first divergence.  512-token prompt =
               the BASELINE shape: CTA-pair tcgen05 GEMMs, 8 q-tiles of prefill attention, 10 KV pages.
  8 streams    all prompts submitted at once through submit/poll (packed prefill, CUDA-graph decode)
  64 streams   every prompt 8 times: gemm_tc<64,*> + decode_attention_mma_kernel at full geometry

The concurrent legs reuse the oracle logits of the first leg: while a stream's tokens equal the
batch-1 tokens the oracle's logits for the next step are known, and at the first difference the
stream's token must be a near-arg-max of those logits (the near-tie rule).
LLMLB_PARITY_PROMPTS (default 8) shortens the run for ad-hoc GPU sessions; each prompt costs the
oracle about half a minute of host time."""
import os

import numpy as np
import pytest

from llmlb_b200 import ffi

pytestmark = pytest.mark.gpu

N_PROMPTS = int(os.environ.get("LLMLB_PARITY_PROMPTS", "8"))
PROMPT, STEPS = 512, 32
# Logit standard deviation here is about 1.28 — the synthetic N(0, 0.02^2) weights give
# very flat distributions (the top two of 128256 logits are typically ~0.1 apart), so arg-max flips at
# near-ties are the common case and TOKEN IDENTITY is not the criterion: every token the engine picks
# must be within NEAR_TIE of the oracle's arg-max logit.  Bounds = measured + margin.
MAX_ABS_TOL = 0.30
MEAN_ABS_TOL = 0.04
NEAR_TIE = 0.30


@pytest.fixture(scope="module")
def legs(built_lib):
    import torch
    from oracle import synth_native
    from oracle.llama_ref import LlamaRef
    cfg = ffi.LLAMA3_8B
    rs = [np.random.RandomState(4000 + i) for i in range(N_PROMPTS)]
    prompts = [r.randint(0, cfg["vocab"], PROMPT).tolist() for r in rs]
    eng = ffi.Engine(cfg, max_seqs=64, max_ctx=1024, seed=0)
    # leg 1: batch 1, logits of every step
    gpu_logits, gpu_tokens = [], []
    for p in prompts:
        lg = eng.debug_prefill_logits(p)
        steps, toks = [], []
        for s in range(STEPS):
            steps.append(lg.copy())
            t = int(np.argmax(lg))
            toks.append(t)
            if s + 1 < STEPS:
                lg = eng.debug_decode_logits(t)
        eng.debug_reset()
        gpu_logits.append(np.stack(steps)); gpu_tokens.append(toks)

    def concurrent(plist):
        eng.pause(True)        # all requests queued before the first scheduling decision: packed prefill waves
        rids = [eng.submit(p, STEPS, ignore_eos=True) for p in plist]
        eng.pause(False)
        outs = []
        for r in rids:
            toks = []
            while True:
                ev = eng.poll(r, timeout_ms=-1)
                toks += [e["token_id"] for e in ev if e["token_id"] >= 0]
                if ev and ev[-1]["finish_reason"]:
                    break
            eng.release(r)
            outs.append(toks)
        return outs
    c8 = concurrent(prompts)
    reps = max(1, 64 // N_PROMPTS)
    c64 = concurrent([p for p in prompts for _ in range(reps)])
    eng.close()
    # the oracle, teacher-forced with the batch-1 tokens
    cores = synth_native.effective_cpus()
    torch.set_num_threads(cores)
    synth_native.set_threads(cores)
    sd = synth_native.synth_state_dict_bits(cfg, seed=0)
    ref = LlamaRef(cfg, sd, emulate_bf16=True)
    ref_logits = []
    for p, toks in zip(prompts, gpu_tokens):
        ref.reset()
        lg = ref.forward(p)[-1].numpy()
        steps = []
        for s in range(STEPS):
            steps.append(lg.copy())
            if s + 1 < STEPS:
                lg = ref.forward([toks[s]])[-1].numpy()
        ref_logits.append(np.stack(steps))
    return dict(prompts=prompts, gpu_logits=gpu_logits, gpu_tokens=gpu_tokens, ref_logits=ref_logits, c8=c8, c64=c64, reps=reps)


def test_batch1_logits_512_prompt_32_steps(legs):
    max_abs, mean_abs, agree, first_div = [], [], 0, []
    for g, r, toks in zip(legs["gpu_logits"], legs["ref_logits"], legs["gpu_tokens"]):
        d = np.abs(g - r)
        max_abs.append(float(d.max())); mean_abs.append(float(d.mean()))
        top = r.argmax(axis=1)
        eq = [int(a == b) for a, b in zip(toks, top)]
        agree += sum(eq)
        first_div.append(eq.index(0) if 0 in eq else None)
        # where the arg-max differs the engine's token must be a near-tie under the oracle
        for s, (t, o) in enumerate(zip(toks, top)):
            if t != o:
                assert r[s, o] - r[s, t] <= NEAR_TIE, (s, float(r[s, o] - r[s, t]))
    total = len(legs["gpu_tokens"]) * STEPS
    print("\n8B parity, batch 1, %d prompts x %d-token prompt x %d steps vs bf16-emulating oracle: max|dlogit| %.4f (per prompt %s), "
          "mean|dlogit| %.5f, top-1 agreement %d/%d, first divergence per prompt %s, logit std %.3f"
          % (len(max_abs), PROMPT, STEPS, max(max_abs), ["%.3f" % m for m in max_abs], float(np.mean(mean_abs)), agree, total,
             first_div, float(legs["ref_logits"][0].std())))
    assert max(max_abs) <= MAX_ABS_TOL
    assert float(np.mean(mean_abs)) <= MEAN_ABS_TOL
    assert agree >= int(0.75 * total)


def _check_streams(legs, outs, reps):
    n_equal = 0
    for i, toks in enumerate(outs):
        base, r = legs["gpu_tokens"][i // reps], legs["ref_logits"][i // reps]
        assert len(toks) == STEPS
        for s in range(STEPS):
            if toks[s] != base[s]:
                # same context up to here, so the oracle's logits of this step apply: near-tie rule
                assert r[s].max() - r[s, toks[s]] <= NEAR_TIE, (i, s, float(r[s].max() - r[s, toks[s]]))
                break
        else:
            n_equal += 1
    return n_equal


def test_8_concurrent_streams_match(legs):
    n_equal = _check_streams(legs, legs["c8"], 1)
    print("\n8B parity, %d concurrent streams: %d/%d token-identical to batch 1, the rest diverge at an oracle near-tie" % (len(legs["c8"]), n_equal, len(legs["c8"])))
    assert n_equal >= 0   # reported, not required: see the note on near-ties at the top


def test_64_concurrent_streams_match(legs):
    n_equal = _check_streams(legs, legs["c64"], legs["reps"])
    print("\n8B parity, %d concurrent streams: %d/%d token-identical to batch 1, the rest diverge at an oracle near-tie" % (len(legs["c64"]), n_equal, len(legs["c64"])))
    assert n_equal >= 0
