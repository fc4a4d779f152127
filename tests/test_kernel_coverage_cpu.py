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
  * decode GEMVs (tests/test_gemv_sm90_gpu.py): the GEMV cases launch every GEMV class — K-split kernel (B, epilogue, NORM,
    CW, TW) or row-owner kernel (B, epilogue, NORM) — that the tp = 1 engine launches at Llama-3-8B, LLAMA_MID and
    Llama-3-70B shapes (prefill widths and decode batches 1..4: wider steps use the GEMMs); every K-split launch for
    K = 256 j, j = 1..400, and 1..4 tokens has at most 15 teams, so its named barriers 1 + team stay within PTX's 0..15;
    and the GEMV probe and bounds reject outputs wrong in the ways these kernels go wrong.
  * wide-step kernels (tests/test_step_kernels_sm90_gpu.py): the cases launch every class of the residual fold (kernel,
    n_parts, gain, H), RoPE (n_heads, n_kv, tensor-parallel shards included), final RMSNorm (H) and embedding (H) that the
    tp = 1 engine launches at Llama-3-8B, LLAMA_MID and Llama-3-70B shapes; every kernel in those launch plans is either
    launched by a GPU kernel test case or listed with the test that covers it; and the fold, norm and RoPE checkers reject
    a dropped or reordered part, a gain a quarter off, a missing DSMEM exchange, another token's RMS scale, wrong RoPE
    pairs, positions or sin sign, and K in the neighbouring page slot.
  * decode attention (tests/test_decode_attention_sm90_gpu.py): DECODE_CASES is decode_splits' classes at their smallest and
    largest batch, and launches every (cluster size, n_heads, n_kv) class the engine's plans launch — tp = 1 at Llama-3-8B,
    LLAMA_TINY, LLAMA_MID and Llama-3-70B shapes, the 8B and 70B shards at tp 2, 4 and 8, decode batches 1..128 — at the
    smallest and the largest batch the engine launches it at; the decode layer chain of tests/test_gemv_sm90_gpu.py makes
    exactly the engine's launches of a decode step's first two layers at B = 1..4 (kernel, grid, block, cluster, shared
    memory, PDL); and the decode checkers reject a kernel that rotates with the identity table, at position L, with the sin
    sign flipped or interleaved pairs, attends over the stale page row instead of the new token, appends k to the next
    slot or the neighbouring kv head, reads another head group's kv head, or attends with the previous layer's qkv rows.
  * sampler (tests/test_sampling_sm90_gpu.py): its vocabularies cover every vocabulary the engine samples at 8B, MID and
    70B; and its draw checker, applied to a numpy model of the kernel's fp32 orders, rejects the old fallback to the last
    kept index on draws inside the gap between the warp totals and the row scans, a run not carried across rows, a strict
    top-k threshold, top-p one token short, u from step + 1, and top_p = 0 taken as "off".
"""
import collections
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_decode_attention_sm90_gpu as DA  # noqa: E402
import test_engine_host_logic_cpu as HL  # noqa: E402
import test_gemv_sm90_gpu as GV  # noqa: E402
import test_kernels_sm90_gpu as K  # noqa: E402
import test_sampling_sm90_gpu as SS  # noqa: E402
import test_step_kernels_sm90_gpu as SK  # noqa: E402

GEMM_RE = re.compile(r"(gemm_tc2?_kernel)ILi(\d+)ELi(\d+)E")
GEMV_KS_RE = re.compile(r"14gemv_ks_kernelILi(\d+)ELi(\d+)ELb([01])ELi(\d+)ELi(\d+)E")
GEMV_RE = re.compile(r"11gemv_kernelILi(\d+)ELi(\d+)ELb([01])E")


def short_name(mangled):
    """The kernel's own name out of its mangled name: _ZN5llmlb14gemm_tc_kernelILi... -> gemm_tc_kernel."""
    s = re.sub(r"^_ZN5llmlb|^_Z", "", mangled)
    m = re.match(r"\d+", s)
    return s[m.end(): m.end() + int(m.group())] if m else mangled


FOLD_KERNELS = ("rmsnorm_parts_kernel", "rmsnorm_parts_cluster_kernel")


def classes(log):
    """{context: set of launch classes}: ("gemm_tc_kernel" | "gemm_tc2_kernel", BN, EPI, K-split) for the projections,
    ("decode", cluster size, n_heads, n_kv) for decode attention (cluster size 1 = the unsplit tensor-core kernel),
    ("prefill", kernel),
    ("gemv_ks", B, EPI, NORM, CW, TW) for the K-split GEMV, ("gemv", B, EPI, NORM) for the row-owner GEMV,
    ("fold", kernel, n_parts, gain, H) for the residual fold, ("rope", n_heads, n_kv), ("rmsnorm_kernel", H) and
    ("embed_kernel", H) and ("sample", vocab)."""
    out, ctx = collections.defaultdict(set), "init"
    for line in open(log):
        if line.startswith("###"):
            ctx = line[4:].strip()
            continue
        p = line.split()
        name = short_name(p[0])
        if name in FOLD_KERNELS:
            assert len(p) == 15, line            # n_parts, gain given, hidden appended
            out[ctx].add(("fold", name, int(p[12]), p[13] == "1", int(p[14])))
            continue
        if name == "rope_append_kernel":
            assert len(p) == 14, line            # n_heads, n_kv appended
            out[ctx].add(("rope", int(p[12]), int(p[13])))
            continue
        if name == "sample_kernel":
            assert len(p) == 13, line            # vocab appended
            out[ctx].add(("sample", int(p[12])))
            continue
        if name in ("rmsnorm_kernel", "embed_kernel"):
            assert len(p) == 13, line            # hidden appended
            out[ctx].add((name, int(p[12])))
            continue
        m = GEMM_RE.search(p[0])
        if m:
            assert len(p) == 13, line            # the fake runtime appends split_k to projection launches
            out[ctx].add((m.group(1), int(m.group(2)), int(m.group(3)), int(p[12]) > 1))
            continue
        m = GEMV_KS_RE.search(p[0])
        if m:
            assert len(p) == 13 and m.group(5) == "0", line     # TW appended; no tensor-parallel variant at tp = 1
            out[ctx].add(("gemv_ks", int(m.group(1)), int(m.group(2)), m.group(3) == "1", int(m.group(4)), int(p[12])))
            continue
        m = GEMV_RE.search(p[0])
        if m:
            out[ctx].add(("gemv", int(m.group(1)), int(m.group(2)), m.group(3) == "1"))
        elif "decode_attention_mma_kernel" in p[0]:
            assert len(p) == 15, line            # n_heads, n_kv, sequences appended
            out[ctx].add(("decode", 1, int(p[12]), int(p[13])))
        elif "decode_attention_kernel" in p[0]:
            assert len(p) == 15, line
            out[ctx].add(("decode", int(p[8]), int(p[12]), int(p[13])))
        elif "prefill_attention_kernel_tc" in p[0]:
            out[ctx].add(("prefill", "tc"))
        elif "prefill_attention_kernel" in p[0]:
            out[ctx].add(("prefill", "mma"))
    return out


def launched_kernels(tmp_path, name):
    """The kernel names of every launch in the log run_logged(tmp_path, name, ...) wrote."""
    return {short_name(l.split()[0]) for l in open(str(tmp_path / (name + ".log"))) if not l.startswith("###")}


def run_logged(tmp_path, name, argv, extra_env=None, parse=classes):
    log = str(tmp_path / (name + ".log"))
    env = dict(os.environ, LD_PRELOAD=HL.build_fake(), FAKE_CUDART_LAUNCH_LOG=log, **(extra_env or {}))
    r = subprocess.run([sys.executable] + argv, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return parse(log)


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
    assert len(engine_gemm) >= 20 and {("decode", s, 32, 8) for s in (1, 2, 4, 8, 16)} <= engine_attn, sorted(engine)
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


# ------------------------------------------------------------------------------------------------------ decode GEMVs --
EPIS = (K.EPI_STORE_BF16, K.EPI_RESID_F32, K.EPI_SILU_MUL, K.EPI_STORE_F32)
KS_INSTANCES = ((1, 1), (1, 2), (1, 4), (2, 1), (2, 2), (3, 1), (4, 1))    # (B, CW) of gemv_ks_try's dispatch


def _gemv_sweep(tmp_path, name, rows):
    """The classes of llmlb_op_gemv launches over the fake runtime, per case: rows of (n_out, K, tokens, epi, norm)."""
    spec = tmp_path / (name + ".json")
    spec.write_text(json.dumps({"gemv": [[N, Kd, B, e, int(n), GV.n_cols(N, e) + GV.PAD] for N, Kd, B, e, n in rows]}))
    return run_logged(tmp_path, name, [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)])


def _gemv_classes(per_ctx):
    return {c for cs in per_ctx.values() for c in cs if c[0] in ("gemv_ks", "gemv")}


def test_gpu_gemv_cases_launch_every_gemv_class_the_engine_launches(built_lib, tmp_path):
    per_case = _gemv_sweep(tmp_path, "gemv_cases", GV.gemv_params())
    tested = _gemv_classes(per_case)
    engine = {}
    for model in ("8b", "mid", "70b"):
        plan = run_logged(tmp_path, "engine_" + model, [os.path.join(HERE, "support", "launch_plan_sweep.py"), model, "1", "4"])
        for c in _gemv_classes(plan):
            engine.setdefault(c, model)
    assert len(engine) >= 40 and {c[0] for c in engine} == {"gemv_ks", "gemv"}, sorted(engine)
    missing = sorted((c, model) for c, model in engine.items() if c not in tested)
    assert not missing, "the engine launches GEMV classes no GPU GEMV test runs (class, model): %s" % missing
    # what the case table promises besides: every K-split instantiation with every epilogue, with and without NORM; the
    # team shapes TW 16, 14, 8, 7, 3, 2 (CW 1), 14 and 16 (CW 2), 14 (CW 4); every row-owner instantiation
    ks = {c for c in tested if c[0] == "gemv_ks"}
    missing = sorted({(B, cw, e, n) for B, cw in KS_INSTANCES for e in EPIS for n in (False, True)} - {(c[1], c[4], c[2], c[3]) for c in ks})
    assert not missing, "no GPU GEMV case launches the K-split instantiations (B, CW, EPI, NORM) %s" % missing
    missing = sorted({(1, 16), (1, 14), (1, 8), (1, 7), (1, 3), (1, 2), (2, 14), (2, 16), (4, 14)} - {(c[4], c[5]) for c in ks})
    assert not missing, "no GPU GEMV case launches the K-split team shapes (CW, TW) %s" % missing
    missing = sorted({("gemv", B, e, n) for B in (1, 2, 3, 4) for e in EPIS for n in (False, True)} - tested)
    assert not missing, "no GPU GEMV case launches the row-owner instantiations %s" % missing
    assert per_case["gemv 8454 28672 4 1 0"] == {("gemv", 1, K.EPI_RESID_F32, False)}      # one row-owner pass per token
    assert per_case["gemv 264 256 1 3 0"] == {("gemv", 1, K.EPI_STORE_F32, False)}          # K = 256: no one-warp teams


def test_every_k_split_gemv_launch_keeps_its_team_barriers_in_range(built_lib, tmp_path):
    """gemv_ks_kernel synchronises team t with named barrier 1 + t and runs 16 // TW teams; PTX has barriers 0..15."""
    per_case = _gemv_sweep(tmp_path, "gemv_barriers", [(8, 256 * j, B, K.EPI_STORE_F32, False)
                                                       for j in range(1, 401) for B in (1, 2, 3, 4)])
    n_ks = 0
    for ctx, cs in per_case.items():
        for c in cs:
            if c[0] == "gemv_ks":
                n_ks += 1
                assert 16 // c[5] <= 15, "%s: TW %d makes %d teams, barrier ids up to %d" % (ctx, c[5], 16 // c[5], 16 // c[5])
    assert n_ks >= 60, n_ks                     # K = 512 .. 16384 where ks_pick finds a team shape


# GEMV teeth: a model GEMV on the CPU, right or wrong in one of the ways these kernels go wrong, checked by the GPU test's
# probe and bounds.  Case: K = 2048 (8 chunks of 256: a K-split team of 8 warps), 264 rows, 2 tokens.
TN, TK, TB = 264, 2048, 2


def _model(w, x, epi, prev=None, gain=None, eps=0.0, gain_shift=0, rs_from=None, gate_up=None, resid=None):
    """epi(W . y) in fp64 with the kernels' rounding points: y = x (bf16), or y = bf16(x rs g) with NORM."""
    y = x.double()
    if gain is not None:
        rs = (y.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
        if rs_from is not None:
            rs = rs[rs_from]
        y = (y * rs * gain.double().roll(-gain_shift)).to(torch.bfloat16).double()
    acc = (y @ w.double().t()).float()
    if epi == K.EPI_SILU_MUL:
        g, u = acc[:, 0::2].double(), acc[:, 1::2].double()
        if gate_up:
            g, u = gate_up(g, u)
        return (g / (1 + (-g).exp()) * u).to(torch.bfloat16)
    if epi == K.EPI_RESID_F32:
        return resid(prev, acc) if resid else prev + acc
    return acc.to(torch.bfloat16) if epi == K.EPI_STORE_BF16 else acc


def _probe_rejects(epi=K.EPI_STORE_F32, norm=False, mutate_x=None, **knobs):
    """Mismatches the GEMV probe finds over all rounds of the teeth case."""
    w = K.probe_weights(TN, TK, torch.Generator().manual_seed(5), "cpu")
    plan = GV.probe_plan(TB, TK, norm, 11)
    e, gain, eps = GV.probe_norm_setup(TK, plan[0][0].shape[1], 11, "cpu") if norm else (None, None, 0.0)
    prev = K.probe_weights(TB, GV.n_cols(TN, epi), torch.Generator().manual_seed(6), "cpu").float()
    bad = 0
    for cols, signs in plan:
        x, acc = GV.probe_x_and_ref(w, cols, signs, e)
        out = _model(w, mutate_x(x.clone()) if mutate_x else x, epi, prev, gain, eps, **knobs)
        bad += GV.probe_mismatches(out, acc, epi, prev)
    return bad


def _random_rejects(epi=K.EPI_STORE_F32, norm=False, B=TB, **knobs):
    """Elements over the GEMV random-data bound."""
    w = GV.random_w(TN, TK, 3, "cpu")
    x, gain = GV.random_x(B, TK, norm, 4, "cpu")
    prev = torch.randn(B, TN, generator=torch.Generator().manual_seed(7))
    out = _model(w, x, epi, prev, gain if norm else None, GV.RANDOM_EPS, **knobs)
    ref, bound, _ = GV.random_ref(w, x, epi, prev, gain if norm else None, GV.RANDOM_EPS)
    return GV.over_bound(out, ref, bound)[0]


def test_gemv_case_table_probe_covers_every_8_group_of_every_token():
    for _, Kd, toks, _, norms in GV.GEMV_CASES:
        for B in toks:
            for norm in norms:
                plan = GV.probe_plan(B, Kd, norm, 1)
                for t in range(B):
                    hit = torch.cat([cols[t] for cols, _ in plan])
                    assert set((hit // 8).tolist()) == set(range(Kd // 8)), (Kd, B, norm, t)
                    assert len(set((hit % 8).tolist())) == min(8, len(hit)), (Kd, B, norm, t)
                assert all(len(set((cols[t] // 8).tolist())) == cols.shape[1] for cols, _ in plan for t in range(B))


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("epi", EPIS)
def test_gemv_probe_and_bound_accept_a_correct_gemv(epi, norm):
    assert _probe_rejects(epi, norm) == 0
    assert _random_rejects(epi, norm) == 0
    assert _random_rejects(epi, norm, B=4) == 0


@pytest.mark.parametrize("norm", [False, True])
def test_gemv_probe_rejects_a_dropped_or_neighbouring_256_chunk(norm):
    for j in range(TK // 256):
        lo, hi = 256 * j, 256 * j + 256

        def drop(x):
            x[:, lo:hi] = 0
            return x

        def neighbour(x):                   # the warp reads W and x at the next warp's offset: chunk j + 1 twice, j never
            x[:, lo:hi], x[:, hi % TK:hi % TK + 256] = 0, 2 * x[:, hi % TK:hi % TK + 256]
            return x
        assert _probe_rejects(norm=norm, mutate_x=drop) > 0, j
        assert _probe_rejects(norm=norm, mutate_x=neighbour) > 0, j


@pytest.mark.parametrize("norm", [False, True])
def test_gemv_probe_rejects_a_shifted_8_group(norm):
    for g in (0, 1, 31, 32, 33, 100, 255):
        def shift(x, g=g):                  # the lane's activations come from the next 8-group (its weights do not)
            nxt = (g + 1) % (TK // 8)
            x[:, 8 * g:8 * g + 8] = x[:, 8 * nxt:8 * nxt + 8].clone()
            return x
        assert _probe_rejects(norm=norm, mutate_x=shift) > 0, g


RN = 266       # 133 row pairs over gemv_ks's 132 CTAs: CTA ranges of one and of two pairs


def _ks_rows(b, grid, n_pairs, n_out):
    """gemv_ks_kernel's rows of CTA b: whole row pairs, in contiguous near-equal ranges."""
    return (b * n_pairs // grid) * 2, min(n_out, ((b + 1) * n_pairs // grid) * 2)


def _ranged_output(acc, epi, prev, rows_of):
    """What the CTAs of a gemv_ks launch write when CTA b takes rows rows_of(b, grid, n_pairs, n_out): each CTA applies the
    epilogue to its own rows (SiLU to the pairs (r, r + 1) counted from its first row while r + 1 is in range; the
    residual add accumulates, so a row two CTAs take gets it twice); rows no CTA takes keep the NaN sentinel."""
    n_out = acc.shape[1]
    n_pairs = (n_out + 1) // 2
    grid = min(n_pairs, 132)                             # ks_launch
    if epi == K.EPI_RESID_F32:
        out = prev.clone()
    else:
        out = torch.full((acc.shape[0], GV.n_cols(n_out, epi)), float("nan"),
                         dtype=torch.float32 if epi == K.EPI_STORE_F32 else torch.bfloat16)
    for b in range(grid):
        lo, hi = rows_of(b, grid, n_pairs, n_out)
        if epi == K.EPI_SILU_MUL:
            r = torch.arange(lo, max(lo, hi - 1), 2)
            g, u = acc[:, r].double(), acc[:, r + 1].double()
            out[:, r >> 1] = (g / (1 + (-g).exp()) * u).to(torch.bfloat16)
        elif epi == K.EPI_RESID_F32:
            out[:, lo:hi] += acc[:, lo:hi]
        else:
            out[:, lo:hi] = acc[:, lo:hi].to(out.dtype)
    return out


def _range_rejects(epi, rows_of):
    w = K.probe_weights(RN, 512, torch.Generator().manual_seed(8), "cpu")
    prev = K.probe_weights(TB, RN, torch.Generator().manual_seed(9), "cpu").float()
    bad = 0
    for cols, signs in GV.probe_plan(TB, 512, False, 12):
        _, acc = GV.probe_x_and_ref(w, cols, signs)
        bad += GV.probe_mismatches(_ranged_output(acc, epi, prev, rows_of), acc, epi, prev)
    return bad


def test_gemv_ks_cta_ranges_are_uneven_at_266_rows():
    lens = {hi - lo for lo, hi in (_ks_rows(b, 132, RN // 2, RN) for b in range(132))}
    assert lens == {2, 4}


@pytest.mark.parametrize("epi", EPIS)
def test_gemv_probe_rejects_cta_row_ranges_that_lose_or_duplicate_a_row_pair(epi):
    assert _range_rejects(epi, _ks_rows) == 0
    # each range one pair short: the pair at every CTA boundary is lost
    assert _range_rejects(epi, lambda *a: (_ks_rows(*a)[0], _ks_rows(*a)[1] - 2)) > 0
    # each range one pair long: the pair at every boundary is computed by two CTAs, the same value twice, which only the
    # residual add turns into a wrong result
    long = _range_rejects(epi, lambda *a: (_ks_rows(*a)[0], min(a[3], _ks_rows(*a)[1] + 2)))
    assert (long > 0) == (epi == K.EPI_RESID_F32)
    # ranges cut at rows rather than pairs: harmless for rowwise epilogues, but a (gate, up) pair straddles two CTAs
    rows = _range_rejects(epi, lambda b, grid, n_pairs, n_out: (b * n_out // grid, (b + 1) * n_out // grid))
    assert (rows > 0) == (epi == K.EPI_SILU_MUL)


@pytest.mark.parametrize("norm", [False, True])
def test_gemv_probe_rejects_swapped_gate_and_up_or_the_next_pairs_up(norm):
    assert _probe_rejects(K.EPI_SILU_MUL, norm, gate_up=lambda g, u: (u, g)) > 0
    assert _probe_rejects(K.EPI_SILU_MUL, norm, gate_up=lambda g, u: (g, u.roll(-1, 1))) > 0


@pytest.mark.parametrize("norm", [False, True])
def test_gemv_probe_and_bound_reject_a_residual_added_twice(norm):
    for resid in (lambda p, a: p + a + a, lambda p, a: p + p + a):
        assert _probe_rejects(K.EPI_RESID_F32, norm, resid=resid) > 0
        assert _random_rejects(K.EPI_RESID_F32, norm, resid=resid) > 0


@pytest.mark.parametrize("epi", EPIS)
def test_gemv_bound_rejects_another_tokens_rms_scale(epi):
    assert _random_rejects(epi, True, rs_from=[1, 0]) > 0
    assert _random_rejects(epi, True, B=4, rs_from=[0, 1, 2, 1]) > 0


@pytest.mark.parametrize("epi", EPIS)
def test_gemv_probe_rejects_a_gain_shifted_by_8(epi):
    assert _probe_rejects(epi, True, gain_shift=8) > 0
    assert _probe_rejects(epi, True, gain_shift=-8) > 0


# ---------------------------------------------------------------------------- wide-step kernels: fold, norm, RoPE, embed --
# Kernels of the tp = 1 launch plans that none of the case sweeps launches, with the tests that run them on the GPU.  A
# kernel that appears in the plans and is neither launched by a GPU kernel test case nor listed here fails
# test_every_kernel_of_the_launch_plans_is_gpu_tested_or_classified.
COVERED_ELSEWHERE = {
    "rope_table_kernel": "test_rope_scaling_gpu.py (the scaled table against fp64 up to position 131071)",
    "slot_init_kernel": "the engine tests (test_engine_gpu.py, test_parity_8b_gpu.py): step bookkeeping",
    "prefill_finish_kernel": "the engine tests: step bookkeeping",
    "step_finish_kernel": "the engine tests: step bookkeeping",
    "sample_prepare_kernel": "the engine tests: step bookkeeping",
    "decode_prepare_kernel": "the engine tests: step bookkeeping",
    "iota_kernel": "the engine tests: step bookkeeping",
    "fill_bf16_kernel": "the engine tests: weight set-up",
    "synth_strided_kernel": "the engine tests: synthetic weights (test_engine_gpu.py checks them against the oracle generator)",
    "gather_rows_kernel": "the engine tests: the rows that need logits",
}
STEP_KINDS = ("fold", "rope", "rmsnorm_kernel", "embed_kernel")
PLAN_MODELS = ("8b", "mid", "70b")


def _step_case_plan(tmp_path):
    spec = tmp_path / "step_cases.json"
    spec.write_text(json.dumps({
        "fold": [[T, H, n, int(g), T * H + (SK.STRIDE_PAD if pad else 0)] for T, H, n, g, pad in SK.FOLD_CASES],
        "rmsnorm": [list(c) for c in SK.RMSNORM_CASES],
        "rope": [[T, nh, nkv] for nh, nkv in SK.ROPE_HEADS for T in SK.ROPE_TOKENS],
        "embed": [[T, H, SK.EMBED_VOCAB] for T, H in SK.EMBED_CASES]}))
    return run_logged(tmp_path, "step_cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)])


def _sample_case_plan(tmp_path):
    spec = tmp_path / "sample_cases.json"
    spec.write_text(json.dumps({"sample": [[3, V] for V in SS.VOCABS]}))
    return run_logged(tmp_path, "sample_cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)])


def _engine_plan(tmp_path, model, tp, max_width=None, parse=classes):
    argv = [os.path.join(HERE, "support", "launch_plan_sweep.py"), model, str(tp)] + ([str(max_width)] if max_width else [])
    return run_logged(tmp_path, "engine_%s_tp%d" % (model, tp), argv, parse=parse)


def rope_shapes(log):
    """{("rope", n_heads, n_kv)} of the rope_append_kernel launches in a log (of any tensor-parallel degree)."""
    return {("rope", int(p[12]), int(p[13])) for p in (l.split() for l in open(log) if not l.startswith("###"))
            if short_name(p[0]) == "rope_append_kernel"}


def _kind(per_ctx, kinds=STEP_KINDS):
    return {c for cs in per_ctx.values() for c in cs if c[0] in kinds}


def test_step_case_tables_span_the_dispatch_boundaries():
    Ts = {c[0] for c in SK.FOLD_CASES}
    assert {T for T in Ts if T <= SK.CLUSTER_MAX_TOKENS} and {T for T in Ts if T > SK.CLUSTER_MAX_TOKENS}
    assert {255, 256, 257} <= Ts and {c[2] for c in SK.FOLD_CASES} == {0, 1, 2, 4, 8}
    assert {(c[3], c[4]) for c in SK.FOLD_CASES if c[2] >= 2} == {(g, p) for g in (False, True) for p in (False, True)}
    assert SK.STRIDE_PAD % 4 == 0 and all(SK.STRIDE_PAD % H for H in SK.HIDDENS)
    assert max(max(SK.rope_layout(T)[0]) for T in SK.ROPE_TOKENS) == SK.ROPE_MAX_POS - 1
    slots = {p % 64 for T in SK.ROPE_TOKENS for p in SK.rope_layout(T)[0]}
    assert {0, 63} <= slots
    assert any(-1 in SK.rope_pages(*SK.rope_layout(T), 1)[0] for T in SK.ROPE_TOKENS)


def test_gpu_step_kernel_cases_launch_every_class_the_engine_launches(built_lib, tmp_path):
    """Every (kernel, n_parts, gain, H) of the residual fold, (n_heads, n_kv) of RoPE and H of the final RMSNorm and the
    embedding that the tp = 1 engine launches at Llama-3-8B, LLAMA_MID and Llama-3-70B shapes over prefill widths 1..2048
    (so the one-CTA-per-row fold above 256 rows is seen) must be among the classes the GPU step-kernel cases launch; and
    so must the RoPE head shapes of the tensor-parallel shards of 8B and 70B at tp 2, 4 and 8."""
    tested = _kind(_step_case_plan(tmp_path))
    engine = {}
    for model in PLAN_MODELS:
        for c in _kind(_engine_plan(tmp_path, model, 1)):
            engine.setdefault(c, model)
    folds = {c for c in engine if c[0] == "fold"}
    assert {c[1] for c in folds} == set(FOLD_KERNELS) and {c[4] for c in folds} == {2048, 4096, 8192}, sorted(folds)
    assert ("fold", "rmsnorm_parts_cluster_kernel", 4, False, 4096) in folds                 # the last fold of 8B: no gain
    assert ("fold", "rmsnorm_parts_cluster_kernel", 8, True, 2048) in folds                  # LLAMA_MID: 8 parts
    missing = sorted((c, model) for c, model in engine.items() if c not in tested)
    assert not missing, "the engine launches step-kernel classes no GPU test runs (class, model): %s" % missing
    shards = set()
    for model in ("8b", "70b"):
        for tp in (2, 4, 8):
            shards |= _engine_plan(tmp_path, model, tp, 8, parse=rope_shapes)
    assert shards == {("rope", 32 // t, 8 // t) for t in (2, 4, 8)} | {("rope", 64 // t, 8 // t) for t in (2, 4, 8)}, sorted(shards)
    missing = sorted(shards - tested)
    assert not missing, "the tensor-parallel engine launches RoPE head shapes no GPU test runs: %s" % missing


def test_every_kernel_of_the_launch_plans_is_gpu_tested_or_classified(built_lib, tmp_path):
    """Every kernel the tp = 1 engine launches (8B, LLAMA_MID, 70B) is launched by a GPU kernel test case (GEMMs,
    attention, GEMVs, step kernels, sampler) or is listed in COVERED_ELSEWHERE with the test that covers it.  A kernel added to
    the engine fails here until someone classifies it."""
    cases = {"gemm": [[T, N, Kd, e] for T, N, Kd, epis in K.GEMM_CASES for e in epis],
             "wave_tail": list(K.WAVE_TAIL_CASE) + [K.wave_tail_rows(*K.WAVE_TAIL_CASE[:2])],
             "decode_splits": K.DECODE_SPLITS, "max_split": K.GEMM_MAX_SPLIT}
    spec = tmp_path / "cases.json"
    spec.write_text(json.dumps(cases))
    run_logged(tmp_path, "cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)])
    _gemv_sweep(tmp_path, "gemv_cases", GV.gemv_params())
    _step_case_plan(tmp_path)
    _sample_case_plan(tmp_path)
    tested = set().union(*(launched_kernels(tmp_path, n) for n in ("cases", "gemv_cases", "step_cases", "sample_cases")))
    engine = set()
    for model in PLAN_MODELS:
        _engine_plan(tmp_path, model, 1)
        engine |= launched_kernels(tmp_path, "engine_%s_tp1" % model)
    assert len(engine) >= 20 and "?" not in engine, sorted(engine)
    unclassified = sorted(engine - tested - set(COVERED_ELSEWHERE))
    assert not unclassified, "kernels the engine launches that no GPU kernel test case runs and nobody classified: %s" % unclassified
    stale = sorted(set(COVERED_ELSEWHERE) - engine)
    assert not stale, "COVERED_ELSEWHERE names kernels the engine no longer launches: %s" % stale
    assert not set(COVERED_ELSEWHERE) & tested, sorted(set(COVERED_ELSEWHERE) & tested)


# teeth: the fold, norm and RoPE checkers applied on the CPU to outputs that are wrong in the ways these kernels go wrong
FT, FH = 17, 2048          # a cluster-kernel step: each CTA owns a quarter (512 columns) of the row


def _fold_case(n_parts=4):
    return SK.fold_inputs(FT, FH, n_parts, 5, "cpu")


def _norm_model(xf, gain, eps, gain_shift=0, quarter_ss=False, rs_from=None):
    """y = bf16(x r g) in fp32 per token, as the kernels compute it, or wrong in one way."""
    ss = (xf * xf).sum(-1, keepdim=True)
    r = torch.rsqrt(ss / FH + torch.tensor(eps, dtype=torch.float32))
    if quarter_ss:          # each CTA normalises its quarter by its own partial sum: no DSMEM exchange
        q = FH // 4
        r = torch.cat([torch.rsqrt((xf[:, i * q:(i + 1) * q] ** 2).sum(-1, keepdim=True) / FH + eps).expand(-1, q) for i in range(4)], 1)
    if rs_from is not None:
        r = r[rs_from]
    return (xf * r * gain.float().roll(-gain_shift)).to(torch.bfloat16)


def _norm_rejects(**knobs):
    x, parts, g = _fold_case()
    xf = SK.fold_ref(x, parts)
    return SK.check_norm(_norm_model(xf, g, SK.EPS, **knobs), xf, g, SK.EPS, FH, True)[0]


def test_fold_and_norm_checkers_accept_a_correct_kernel():
    x, parts, g = _fold_case()
    assert K.bits_equal(SK.fold_ref(x, parts), SK.fold_ref(x.clone(), [p.clone() for p in parts])) == 0
    assert _norm_rejects() == 0
    for cluster in (False, True):
        for H in SK.HIDDENS:
            assert 2.0 ** -21 < SK.norm_rel_bound(H, cluster) < 2.0 ** -18


def test_fold_checker_rejects_a_dropped_last_part_and_the_reverse_order():
    x, parts, g = _fold_case()
    want = SK.fold_ref(x, parts)
    assert K.bits_equal(SK.fold_ref(x, parts[:-1]), want) > 0
    assert K.bits_equal(SK.fold_ref(x, parts[::-1]), want) > 0


def test_norm_checker_rejects_a_gain_one_quarter_off_a_missing_exchange_and_another_tokens_scale():
    assert _norm_rejects(gain_shift=FH // 4) > 0
    assert _norm_rejects(gain_shift=-FH // 4) > 0
    assert _norm_rejects(quarter_ss=True) > 0
    assert _norm_rejects(rs_from=[(t + 1) % FT for t in range(FT)]) > 0


_TABLE = {}


def _rope_table():
    """The Llama 3.1 table, fp64 angles rounded to fp32 (what rope_table_kernel computes)."""
    if not _TABLE:
        from rope_oracle import rope_freq_factors
        from rope_scaling_util import LLAMA31_8B, THETA
        f = torch.tensor(rope_freq_factors(LLAMA31_8B, THETA), dtype=torch.float32).double()
        inv = torch.pow(torch.tensor(THETA, dtype=torch.float32).double(), -torch.arange(0, 128, 2).double() / 128) / f
        ang = torch.arange(SK.ROPE_MAX_POS).double()[:, None] * inv[None]
        _TABLE[0] = torch.stack([ang.cos(), ang.sin()], -1).float()
    return _TABLE[0]


RT, RNH, RNKV = 65, 8, 2


def _rope_case():
    pos_l, seq = SK.rope_layout(RT)
    page_l, n_pages = SK.rope_pages(pos_l, seq, 3)
    gen = torch.Generator().manual_seed(4)
    qkv = (torch.randn(RT, (RNH + 2 * RNKV) * 128, generator=gen) * 4).to(torch.bfloat16)
    pool = torch.full((n_pages, RNKV, 64, 128), float("nan"), dtype=torch.bfloat16)
    return qkv, torch.tensor(pos_l, dtype=torch.int32), torch.tensor(page_l, dtype=torch.int32), pool


def _rope_model(qkv, pos, page, pool, pair_stride=64, pos_shift=0, sin_sign=1.0, slot_shift=0):
    """rope_append in fp32 on the CPU, right or wrong in one way: returns (qkv out, K pool, V pool)."""
    tab = _rope_table()
    nr = RNH + RNKV
    x = qkv[:, : nr * 128].reshape(RT, nr, 128).float()
    cs = tab[(pos.long() + pos_shift).clamp(min=0)]
    c, s = cs[:, None, :, 0], sin_sign * cs[:, None, :, 1]
    if pair_stride == 64:
        a, b = x[..., :64], x[..., 64:]
    else:                                   # pairs (2i, 2i + 1)
        a, b = x[..., 0::2], x[..., 1::2]
    ra, rb = a * c - b * s, b * c + a * s
    rot = torch.cat([ra, rb], -1) if pair_stride == 64 else torch.stack([ra, rb], -1).flatten(-2)
    out = qkv.clone()
    out[:, : nr * 128] = rot.reshape(RT, nr * 128).to(torch.bfloat16)
    kp, vp = SK.rope_pool_expected(pool, pool, qkv, out, pos + slot_shift, page, RNH, RNKV)
    return out, kp, vp


def _rope_rejects(**knobs):
    qkv, pos, page, pool = _rope_case()
    out, kp, vp = _rope_model(qkv, pos, page, pool, **knobs)
    n_bad, _ = SK.rope_check(qkv, out, pos, _rope_table(), RNH, RNKV)
    kw, vw = SK.rope_pool_expected(pool, pool, qkv, out, pos, page, RNH, RNKV)
    return n_bad + K.bits_equal(kp, kw) + K.bits_equal(vp, vw)


def test_rope_checker_accepts_a_correct_kernel():
    assert _rope_rejects() == 0


def test_rope_checker_rejects_wrong_pairs_positions_sin_sign_and_slot():
    assert _rope_rejects(pair_stride=1) > 0
    assert _rope_rejects(pos_shift=-1) > 0
    assert _rope_rejects(sin_sign=-1.0) > 0
    assert _rope_rejects(slot_shift=1) > 0


# ---------------------------------------------------------------------------------------------------- decode attention --
DECODE_PLANS = [("tiny", 1), ("mid", 1), ("8b", 1), ("70b", 1)] + [(m, tp) for m in ("8b", "70b") for tp in (2, 4, 8)]
DECODE_KERNELS = ("decode_attention_kernel", "decode_attention_mma_kernel")


def decode_launches(log):
    """{(cluster size, n_heads, n_kv, sequences)} of the decode attention launches in a log (1 = the tensor-core kernel)."""
    out = set()
    for p in (l.split() for l in open(log) if not l.startswith("###")):
        name = short_name(p[0])
        if name in DECODE_KERNELS:
            assert len(p) == 15, p
            out.add((int(p[8]) if name == DECODE_KERNELS[0] else 1, int(p[12]), int(p[13]), int(p[14])))
    return out


def launch_lines(log):
    """{context: [fields of each launch]}, in launch order."""
    out, ctx = collections.defaultdict(list), "init"
    for line in open(log):
        if line.startswith("###"):
            ctx = line[4:].strip()
        else:
            out[ctx].append(line.split())
    return out


def test_decode_cases_are_every_decode_splits_class_at_its_smallest_and_largest_batch():
    assert DA.DECODE_CASES == DA.derived_cases()
    assert len({(DA.cluster_size(sp), nh, nkv) for sp, nh, nkv, _ in DA.DECODE_CASES}) == 39
    # the cluster kernel on narrow shards at wide batches, the tensor-core kernel up to 128 sequences
    assert (3, 4, 1, 95) in DA.DECODE_CASES and (1, 4, 1, 96) in DA.DECODE_CASES and (1, 64, 8, 128) in DA.DECODE_CASES
    for B in (1, 4, 9, 128):
        lens = DA.launch_lens(B)
        flat = [n for launch in lens for n in launch]
        assert all(len(launch) == B for launch in lens) and set(flat) == set(DA.LENS) | {DA.LONG} and flat.count(DA.LONG) == 1


def test_gpu_decode_cases_launch_every_decode_class_of_the_engine_at_its_smallest_and_largest_batch(built_lib, tmp_path):
    """Every (cluster size, n_heads, n_kv) decode class the engine's plans launch (tp = 1 at TINY, MID, 8B and 70B shapes;
    8B and 70B at tp 2, 4 and 8; decode batches 1..128), at the smallest and at the largest batch it is launched at, is
    launched by a case of tests/test_decode_attention_sm90_gpu.py."""
    spec = tmp_path / "decode_cases.json"
    spec.write_text(json.dumps({"decode": [list(c) for c in DA.DECODE_CASES]}))
    tested = run_logged(tmp_path, "decode_cases", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)], parse=decode_launches)
    assert tested == {(DA.cluster_size(sp), nh, nkv, B) for sp, nh, nkv, B in DA.DECODE_CASES}
    engine = {}
    for model, tp in DECODE_PLANS:
        for c, nh, nkv, nb in _engine_plan(tmp_path, model, tp, DA.MAX_BATCH, parse=decode_launches):
            engine.setdefault((c, nh, nkv), set()).add(nb)
    assert {k[1:] for k in engine} == set(DA.HEADS_TP1 + DA.HEADS_SHARDS), sorted(engine)
    assert {k[0] for k in engine} == {1, 2, 4, 8, 16} and max(max(b) for b in engine.values()) == DA.MAX_BATCH
    missing = sorted(k + (nb,) for k, batches in engine.items() for nb in (min(batches), max(batches)) if k + (nb,) not in tested)
    assert not missing, "the engine launches decode attention (cluster, n_heads, n_kv, batch) no GPU case runs: %s" % missing


def test_decode_layer_chain_launches_what_the_engine_launches(built_lib, tmp_path):
    """The decode layer chain of tests/test_gemv_sm90_gpu.py, layers 0 and 1 at B = 1..4, against the first two layers of
    the engine's decode step at Llama-3-8B, tp = 1: the same kernels with the same grid, block, dynamic shared memory,
    cluster, PDL flag and logged arguments, in the same order."""
    spec = tmp_path / "chain.json"
    spec.write_text(json.dumps({"chain": list(GV.CHAIN_BATCHES)}))
    chain = run_logged(tmp_path, "chain", [os.path.join(HERE, "support", "kernel_case_sweep.py"), str(spec)], parse=launch_lines)
    plan = _engine_plan(tmp_path, "8b", 1, 4, parse=launch_lines)
    assert (GV.CHAIN_H, GV.CHAIN_QKV, GV.CHAIN_FFN) == (4096, 6144, 14336) and (GV.CHAIN_HEADS, GV.CHAIN_KV) == (32, 8)
    for B in GV.CHAIN_BATCHES:
        ours = chain["chain B=%d" % B]
        steps = plan["decode B=%d" % B]
        i = next(j for j, p in enumerate(steps) if short_name(p[0]) in DECODE_KERNELS and int(p[14]) == B)
        engine = steps[i - 1: i + 9]
        assert len(ours) == 10 and [short_name(p[0]) for p in engine[:2]] == ["gemv_ks_kernel", short_name(ours[1][0])], engine
        assert short_name(engine[6][0]) in DECODE_KERNELS and (engine[1][11], engine[6][11]) == ("0", "1")   # layer 1: PDL
        assert ours == engine, "B = %d: the chain launches\n%s\nthe engine\n%s" % (B, "\n".join(map(" ".join, ours)), "\n".join(map(" ".join, engine)))


# teeth: the decode checkers of the GPU test applied on the CPU to a model of the kernels, right or wrong in one way
DNH, DNKV, DLENS = 16, 2, (1, 33, 64, 65, 300)      # GQA group 8: two head groups of 4 share a kv head


def _rotate(qkv, pos, table, nh, nkv, pos_shift=0, sin_sign=1.0, interleaved=False):
    """rope_append's rotation of the q and k heads of the bf16 rows at pos in fp32, or wrong in one way: a rotated copy."""
    B, nr = qkv.shape[0], nh + nkv
    x = qkv[:, : nr * 128].reshape(B, nr, 128).float()
    cs = table[pos.long() + pos_shift]
    c, s = cs[:, None, :, 0], sin_sign * cs[:, None, :, 1]
    a, b = (x[..., 0::2], x[..., 1::2]) if interleaved else (x[..., :64], x[..., 64:])
    ra, rb = (a * c - b * s).to(torch.bfloat16), (b * c + a * s).to(torch.bfloat16)
    rot = torch.stack([ra, rb], -1).flatten(-2) if interleaved else torch.cat([ra, rb], -1)
    out = qkv.clone()
    out[:, : nr * 128] = rot.reshape(B, nr * 128)
    return out


def _decode_case():
    """A CPU pool with random context for DLENS and the qkv rows of this step and of the previous layer."""
    pool = DA.Pool(DNKV, DLENS, 21, device="cpu")
    gen = torch.Generator().manual_seed(22)
    ctx_k = [torch.randn(n - 1, DNKV, 128, generator=gen).to(torch.bfloat16) for n in DLENS]
    ctx_v = [torch.randn(n - 1, DNKV, 128, generator=gen).to(torch.bfloat16) for n in DLENS]
    for i, n in enumerate(DLENS):
        pool.write(i, 0, ctx_k[i], ctx_v[i])
    qkv, prev = DA.qkv_rows(len(DLENS), DNH, DNKV, gen), DA.qkv_rows(len(DLENS), DNH, DNKV, gen, row0=1)
    return pool, ctx_k, ctx_v, qkv, prev, torch.tensor(DLENS, dtype=torch.int32)


def _decode_model(pool, qkv, seq_lens, table, stale_new=False, slot_shift=0, kv_shift=0, group4=False, **rot):
    """A decode launch in fp64 on the CPU: (out, K pool, V pool).  Right, or wrong in one way: the rotation (_rotate's
    knobs), the new token read from the stale page row, k appended slot_shift slots on or kv_shift kv heads over, q head h
    reading kv head (h // 4) % n_kv (the head group's index instead of its kv head)."""
    nh, nkv, g = DNH, DNKV, DNH // DNKV
    r = _rotate(qkv, seq_lens - 1, table, nh, nkv, **rot)
    kp, vp = pool.kp.clone(), pool.vp.clone()
    outs = []
    for b, L in enumerate(seq_lens.tolist()):
        pos, row = L - 1, pool.bt[int(pool.rows[b])].long()
        kn, vn = r[b, nh * 128:(nh + nkv) * 128].view(nkv, 128), qkv[b, (nh + nkv) * 128:].view(nkv, 128)
        p_at = pos + slot_shift
        kp[row[p_at // 64], (torch.arange(nkv) + kv_shift) % nkv, p_at % 64] = kn
        vp[row[pos // 64], :, pos % 64] = vn
        t = torch.arange(L)
        k, v = pool.kp[row[t // 64], :, t % 64].clone(), pool.vp[row[t // 64], :, t % 64].clone()
        if not stale_new:
            k[pos], v[pos] = kn, vn
        kv_of = (torch.arange(nh) // 4) % nkv if group4 else torch.arange(nh) // g
        q = r[b, : nh * 128].view(nh, 128).double()
        sc = torch.einsum("hd,shd->hs", q, k.double()[:, kv_of]) / 128 ** 0.5
        outs.append(torch.einsum("hs,shd->hd", torch.softmax(sc, -1), v.double()[:, kv_of]).to(torch.bfloat16).flatten())
    return torch.stack(outs), kp, vp


def _decode_rejects(prev_rows=False, table=None, **knobs):
    """(output elements over the bound, K pool words wrong, V pool words wrong) of the model, by the GPU test's checker."""
    pool, ctx_k, ctx_v, qkv, prev, seq_lens = _decode_case()
    real = _rope_table()
    out, kp, vp = _decode_model(pool, prev if prev_rows else qkv, seq_lens, real if table is None else table, **knobs)
    rot = _rotate(qkv, seq_lens - 1, real, DNH, DNKV)            # what rope_append computes for this step's rows
    return DA.decode_rejects(out, kp, vp, pool.kp, pool.vp, pool.bt, pool.rows, seq_lens, qkv, rot, ctx_k, ctx_v, DNH, DNKV, 0.0)[:3]


def test_decode_checkers_accept_a_correct_kernel():
    assert _decode_rejects() == (0, 0, 0)


def test_decode_checkers_reject_a_wrong_rotation():
    identity = torch.zeros_like(_rope_table())
    identity[..., 0] = 1
    for knobs in (dict(table=identity), dict(pos_shift=1), dict(sin_sign=-1.0), dict(interleaved=True)):
        n_out, n_k, _ = _decode_rejects(**knobs)
        assert n_out > 0 and n_k > 0, knobs


def test_decode_checkers_reject_the_stale_page_row_a_misplaced_append_another_head_groups_kv_and_the_previous_rows():
    assert _decode_rejects(stale_new=True)[0] > 0
    assert _decode_rejects(slot_shift=1)[1] > 0
    assert _decode_rejects(kv_shift=1)[1] > 0
    assert _decode_rejects(group4=True)[0] > 0
    n_out, n_k, n_v = _decode_rejects(prev_rows=True)
    assert n_out > 0 and n_k > 0 and n_v > 0


# ------------------------------------------------------------------------------------------------------------- sampler --
def _sample_classes(per_ctx):
    return {c for cs in per_ctx.values() for c in cs if c[0] == "sample"}


def test_gpu_sampler_cases_launch_every_vocab_the_engine_launches(built_lib, tmp_path):
    """Every vocabulary the tp = 1 engine samples at Llama-3-8B, LLAMA_MID and Llama-3-70B shapes is among the
    vocabularies tests/test_sampling_sm90_gpu.py launches sample_kernel with."""
    tested = _sample_classes(_sample_case_plan(tmp_path))
    assert tested == {("sample", V) for V in SS.VOCABS}, sorted(tested)
    assert any(V % 32 for V in SS.VOCABS)
    engine = {}
    for model in PLAN_MODELS:
        for c in _sample_classes(_engine_plan(tmp_path, model, 1, 8)):
            engine.setdefault(c, model)
    assert {c[1] for c in engine} >= {128256, 4096}, sorted(engine)
    missing = sorted((c, model) for c, model in engine.items() if c not in tested)
    assert not missing, "the engine samples vocabularies no GPU sampling test runs (class, model): %s" % missing


# teeth: the draw checker of the GPU test applied on the CPU to a numpy model of the kernel — fp32 e (np.exp standing in
# for __expf), top-k / top-p thresholds over 2^-40 fixed-point masses, and FP32Draw's orders — right, or wrong in one way.
def _model_sample(logits, T, k, p, step, fallback="span", carry=True, strict_k=False, p_short=False, p_zero_off=False,
                  step_shift=0):
    if not T > 0:
        return int(np.argmax(logits))
    e = SS.kernel_e(logits, T)
    keep = np.ones(e.size, bool)
    if 0 < k < e.size:
        kth = np.sort(e)[::-1][k - 1]
        keep = e > kth if strict_k else e >= kth
    if p < 1.0 and not (p_zero_off and p <= 0):
        q = np.floor(np.where(keep, e, 0).astype(np.float64) * 2.0 ** 40)
        vals = np.unique(e[keep])[::-1]                                      # descending
        cum = np.cumsum([q[keep & (e == v)].sum() for v in vals]) if vals.size < 64 else \
            np.cumsum(np.bincount(np.searchsorted(-vals, -e[keep]), weights=q[keep], minlength=vals.size))
        i = int(np.searchsorted(cum, np.floor(p * cum[-1]), side="left"))
        i = min(i, vals.size - 1)
        if p_short and i > 0:
            i -= 1
        keep &= e >= vals[i]
    ek = np.where(keep, e, np.float32(0))
    d = SS.FP32Draw(ek, carry=carry)
    last_kept = int(np.nonzero(keep)[0][-1])
    fb = (lambda w: d.last_positive(w) if w is not None else 0) if fallback == "span" else (lambda w: last_kept)
    return d.draw(SS.u_of(step + step_shift), fb)


def _model_rejects(cases, **knobs):
    """Draws of the model the checker rejects, over cases [(logits, T, k, p, steps)]."""
    bad = 0
    for row, T, k, p, steps in cases:
        ref = SS.Ref(row, T, k, p)
        for s in steps:
            bad += not ref.check(_model_sample(row, T, k, p, int(s), **knobs), SS.u_of(s))[0]
    return bad


def _teeth_cases():
    rs = np.random.RandomState(12)
    out = []
    for V in (SS.VOCAB_LLAMA3, SS.VOCAB_ODD):
        lm, tied = SS.make_row("lm", V, 3), SS.make_row("tiedk", V, 4)
        out += [(lm, 1.0, 0, 1.0, rs.randint(0, SS.N_STEPS, 24)), (lm, 0.7, 0, 0.0, rs.randint(0, SS.N_STEPS, 8)),
                (tied, 1.0, SS.TIED_K, 1.0, rs.randint(0, SS.N_STEPS, 48)), (tied, 1.0, 0, 0.9, rs.randint(0, SS.N_STEPS, 48))]
    return out


def _gap_cases():
    out = []
    for V, where in SS.GAP_CASES:
        row = SS.crafted_gap_row(V, 16 if where == "mid" else (V - 1) // SS.span_of(V))
        out.append((row, 1.0, 0, 1.0, SS.gap_steps(SS.kernel_e(row, 1.0), per_warp=16)))
    return out


def test_sampler_checker_accepts_a_correct_kernel_model():
    cases = _teeth_cases() + _gap_cases()
    for V in (SS.VOCAB_TINY, SS.VOCAB_ODD):
        rs = np.random.RandomState(V)
        for kind, seed, T, k, p in SS.case_list(V)[::3]:
            row = SS.make_row(kind, V, seed)
            cases.append((row, T, k, p, np.concatenate([SS.Ref(row, T, k, p).directed_steps(rs, 2), rs.randint(0, SS.N_STEPS, 2)])))
    assert _model_rejects(cases) == 0


def test_sampler_checker_rejects_the_fallback_to_the_last_kept_index_on_gap_draws():
    """The kernel's old fallback: a target in the gap between the crossing warp's total and its row scans crossed no lane,
    and the draw became the last index with key >= floor_key — vocab - 1 whenever no top-k / top-p was set."""
    cases = _gap_cases()
    assert all(len(c[4]) >= 4 for c in cases)
    for row, T, k, p, steps in cases:
        assert all(_model_sample(row, T, k, p, int(s), fallback="last_kept") == row.size - 1 for s in steps)
        assert _model_rejects([(row, T, k, p, steps)], fallback="last_kept") == len(steps)


def test_sampler_checker_rejects_a_dropped_run_carry_a_strict_top_k_a_short_top_p_a_shifted_counter_and_top_p_0_off():
    cases = _teeth_cases()
    lm_t1 = [c for c in cases if c[1] == 1.0 and c[2] == 0 and c[3] == 1.0]
    assert _model_rejects(lm_t1, carry=False) > 0
    assert _model_rejects([c for c in cases if c[2] == SS.TIED_K], strict_k=True) > 0
    assert _model_rejects([c for c in cases if c[3] == 0.9], p_short=True) > 0
    assert _model_rejects(lm_t1, step_shift=1) > 0
    assert _model_rejects([c for c in cases if c[3] == 0.0], p_zero_off=True) > 0
