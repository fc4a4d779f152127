"""Without a GPU: the GPU kernel tests (tests/test_kernels_sm90_gpu.py) cover what the engine launches, and their checkers
would notice the mistakes they are meant to catch.

  * coverage: the GEMM cases, the wave-tail pair and the decode splits of the GPU tests are run through the product library
    over the fake CUDA runtime (tests/support/kernel_case_sweep.py), and so is the engine at Llama-3-8B, tp = 1, over every
    prefill width 1..2048 and decode batch 1..128 (tests/support/launch_plan_sweep.py), once as configured by default and
    once with the wave tail on.  Every projection class the engine launches with epilogues 0..4 — kernel, token tile BN,
    epilogue, K-split or not — and every decode-attention cluster size must be among those the GPU tests launch.  A
    dispatch change that sends the engine down an untested path fails here.
  * teeth: the probe comparison and the attention bound, applied with torch on the CPU to outputs that are wrong in the ways
    a kernel goes wrong (swapped 8-row groups, a dropped k16 step, swapped token halves, a causal mask off by one, a dropped
    64-token page, a running sum l that is not rescaled), must reject every one of them.
"""
import collections
import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_engine_host_logic_cpu as HL  # noqa: E402
import test_kernels_sm90_gpu as K  # noqa: E402

GEMM_RE = re.compile(r"(gemm_tc2?_kernel)ILi(\d+)ELi(\d+)E")


def classes(log):
    """{context: set of launch classes}: ("gemm_tc_kernel" | "gemm_tc2_kernel", BN, EPI, K-split) for the projections,
    ("decode", cluster size) for decode attention (1 = the unsplit tensor-core kernel), ("prefill", kernel)."""
    out, ctx = collections.defaultdict(set), "init"
    for line in open(log):
        if line.startswith("###"):
            ctx = line[4:].strip()
            continue
        p = line.split()
        m = GEMM_RE.search(p[0])
        if m:
            assert len(p) == 13, line            # the fake runtime appends split_k to projection launches
            out[ctx].add((m.group(1), int(m.group(2)), int(m.group(3)), int(p[12]) > 1))
        elif "decode_attention_mma_kernel" in p[0]:
            out[ctx].add(("decode", 1))
        elif "decode_attention_kernel" in p[0]:
            out[ctx].add(("decode", int(p[8])))
        elif "prefill_attention_kernel_tc" in p[0]:
            out[ctx].add(("prefill", "tc"))
        elif "prefill_attention_kernel" in p[0]:
            out[ctx].add(("prefill", "mma"))
    return out


def run_logged(tmp_path, name, argv, extra_env=None):
    log = str(tmp_path / (name + ".log"))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log, **(extra_env or {}))
    r = subprocess.run([sys.executable] + argv, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return classes(log)


def test_case_table_spans_the_dispatch_boundaries():
    Ts = {c[0] for c in K.GEMM_CASES}
    assert Ts >= {5, 16, 17, 24, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 512, 640}
    assert {c[2] % 64 for c in K.GEMM_CASES} >= {0, 8, 56}
    res = {c[1] % 256 for c in K.GEMM_CASES}
    assert 0 in res and 128 in res and {8, 120} <= {r % 128 for r in res}
    assert all(K.probe_rounds(T, Kd) * T >= (Kd + 15) // 16 for T, _, Kd, _ in K.GEMM_CASES)


def test_gpu_cases_launch_every_class_the_engine_launches(built_lib, tmp_path):
    cases = {"gemm": [[T, N, Kd, e] for T, N, Kd, epis in K.GEMM_CASES for e in epis],
             "wave_tail": list(K.WAVE_TAIL_CASE) + [K.wave_tail_rows(*K.WAVE_TAIL_CASE[:2])],
             "decode_splits": K.DECODE_SPLITS, "max_split": K.GEMM_MAX_SPLIT}
    spec = tmp_path / "cases.json"
    spec.write_text(json.dumps(cases))
    per_ctx = run_logged(tmp_path, "cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)])
    tested = set().union(*per_ctx.values())
    # the wave-tail pair ran both of its kernels: CTA pairs over the whole waves, 128-row K-split tiles over the rest
    tail = per_ctx["wave tail 2"]
    assert ("gemm_tc2_kernel", 256, 2, False) in tail and ("gemm_tc_kernel", 256, 2, True) in tail, tail
    engine = set()
    for extra in ({}, {"LLMLB_WAVE_TAIL": "1"}):
        plan = run_logged(tmp_path, "engine%d" % len(extra), [os.path.join(HERE, "support", "launch_plan_sweep.py"), "8b", "1"], extra)
        engine |= set().union(*plan.values())
    engine_gemm = {c for c in engine if c[0].startswith("gemm") and c[2] <= 4}
    engine_attn = {c for c in engine if c[0] in ("decode", "prefill")}
    assert len(engine_gemm) >= 20 and {("decode", s) for s in (1, 2, 4, 8, 16)} <= engine_attn, sorted(engine)
    missing = sorted((engine_gemm | engine_attn) - tested)
    assert not missing, "the engine launches classes no GPU kernel test runs: %s" % missing


# ------------------------------------------------------------------------------------------------------------ teeth --
def _probe_setup(T=16, N=256, Kd=200):
    gen = torch.Generator().manual_seed(3)
    w = K.probe_weights(N, Kd, gen, "cpu")
    return w, [K.probe_x_and_ref(w, T, Kd, r) for r in range(K.probe_rounds(T, Kd))]


def _gemm(x, w):
    return (x.double() @ w.double().t()).float()


def test_probe_accepts_the_exact_product():
    w, rounds = _probe_setup()
    for x, ref in rounds:
        assert K.bits_equal(_gemm(x, w), ref) == 0
        assert K.bits_equal(_gemm(x, w).to(torch.bfloat16), ref.to(torch.bfloat16)) == 0


def test_probe_rejects_swapped_8_row_groups():
    w, rounds = _probe_setup()
    for g0, g1 in ((0, 1), (1, 2), (6, 7), (8, 9), (15, 31)):
        bad = 0
        for x, ref in rounds:
            out = _gemm(x, w)
            a, b = out[:, 8 * g0: 8 * g0 + 8].clone(), out[:, 8 * g1: 8 * g1 + 8].clone()
            out[:, 8 * g0: 8 * g0 + 8], out[:, 8 * g1: 8 * g1 + 8] = b, a
            bad += K.bits_equal(out, ref)
        assert bad > 0, (g0, g1)


def test_probe_rejects_every_dropped_k16_step():
    Kd = 200                                  # 12 full steps and a tail step of 8 columns
    w, rounds = _probe_setup(Kd=Kd)
    for s in range((Kd + 15) // 16):
        bad = 0
        for x, ref in rounds:
            xd = x.clone()
            xd[:, 16 * s: 16 * s + 16] = 0
            bad += K.bits_equal(_gemm(xd, w), ref)
        assert bad > 0, "dropping k16 step %d goes unnoticed" % s


def test_probe_rejects_swapped_token_halves_and_a_shifted_k_slab():
    w, rounds = _probe_setup()
    assert sum(K.bits_equal(_gemm(torch.cat([x[8:], x[:8]]), w), ref) for x, ref in rounds) > 0
    # the second 64-wide slab read from the first one's address (a wrong slab offset)
    assert sum(K.bits_equal(_gemm(torch.cat([x[:, :64], x[:, :64], x[:, 128:]], 1), w), ref) for x, ref in rounds) > 0


def _attn_case(scale=4.0, nh=2, nkv=1, ctx=100, n=100):
    gen = torch.Generator().manual_seed(7)
    S = ctx + n
    q = (torch.randn(n, nh, 128, generator=gen) * scale).to(torch.bfloat16)
    k = torch.randn(S, nkv, 128, generator=gen).to(torch.bfloat16)
    v = torch.randn(S, nkv, 128, generator=gen).to(torch.bfloat16)
    pad = -S % 64                             # the rest of the last page holds what an earlier sequence left there
    sgn = torch.randint(0, 2, (pad, nkv, 128), generator=gen) * 2 - 1
    k_pages = torch.cat([k, (sgn * K.POISON_K).to(torch.bfloat16)])
    v_pages = torch.cat([v, (sgn * K.POISON_V).to(torch.bfloat16)])
    return q, k, v, k_pages, v_pages, torch.arange(ctx, S)


def _online(q, k_pages, v_pages, q_pos, visible, rescale_l=True):
    """Flash attention over 64-token blocks of the pages in fp64, bf16 output; visible(s, pos) -> keys that take part."""
    g = q.shape[1] // k_pages.shape[1]
    qd = q.double()
    kd, vd = k_pages.double().repeat_interleave(g, 1), v_pages.double().repeat_interleave(g, 1)
    n, nh = q.shape[:2]
    m = torch.full((nh, n, 1), float("-inf"), dtype=torch.float64)
    l = torch.zeros(nh, n, 1, dtype=torch.float64)
    o = torch.zeros(nh, n, 128, dtype=torch.float64)
    for j in range(0, kd.shape[0], 64):
        s = torch.arange(j, j + 64)
        sc = torch.einsum("thd,shd->hts", qd, kd[j:j + 64]) / math.sqrt(128)
        sc = sc.masked_fill(~visible(s[None, :], q_pos[:, None])[None], float("-inf"))
        m_new = torch.maximum(m, sc.amax(-1, keepdim=True))
        mu = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
        corr, pj = torch.exp(m - mu), torch.exp(sc - mu)
        l = (l * corr if rescale_l else l) + pj.sum(-1, keepdim=True)
        o = o * corr + torch.einsum("hts,shd->htd", pj, vd[j:j + 64])
        m = m_new
    return (o / l).permute(1, 0, 2).to(torch.bfloat16)


def _over_bound(got, q, k, v, q_pos):
    ref, bound = K.attention_ref(q, k, v, q_pos, K.BF16_U)
    return int(((got.double() - ref).abs() > bound).sum())


def test_attention_bound_accepts_a_correct_kernel():
    for scale in K.ATTN_SCALES:
        q, k, v, kp, vp, pos = _attn_case(scale)
        assert _over_bound(_online(q, kp, vp, pos, lambda s, p: s <= p), q, k, v, pos) == 0, scale


@pytest.mark.parametrize("scale", K.ATTN_SCALES)
def test_attention_bound_rejects_an_off_by_one_causal_mask(scale):
    q, k, v, kp, vp, pos = _attn_case(scale)
    assert _over_bound(_online(q, kp, vp, pos, lambda s, p: s <= p + 1), q, k, v, pos) > 0
    assert _over_bound(_online(q, kp, vp, pos, lambda s, p: s < p), q, k, v, pos) > 0


@pytest.mark.parametrize("scale", K.ATTN_SCALES)
def test_attention_bound_rejects_a_dropped_page(scale):
    q, k, v, kp, vp, pos = _attn_case(scale)
    for page in range(4):
        lo = 64 * page
        got = _online(q, kp, vp, pos, lambda s, p, lo=lo: (s <= p) & ((s < lo) | (s >= lo + 64)))
        assert _over_bound(got, q, k, v, pos) > 0, page


@pytest.mark.parametrize("scale", K.ATTN_SCALES)
def test_attention_bound_rejects_an_unrescaled_running_sum(scale):
    q, k, v, kp, vp, pos = _attn_case(scale)
    assert _over_bound(_online(q, kp, vp, pos, lambda s, p: s <= p, rescale_l=False), q, k, v, pos) > 0
