"""-m gpu: decode attention — the cluster kernel (decode_attention_kernel, a cluster of 2..16 CTAs per sequence and head
group) and the tensor-core kernel (decode_attention_mma_kernel, wide batches) in attention.cu — with the Llama 3.1 RoPE
table, at every (kernel / cluster size, n_heads, n_kv) class the engine launches, each at the smallest and the largest
batch the engine launches it at.

Both kernels rotate the new token's q and k themselves, append k and v to the pages and attend, in one launch.  They promise
to use exactly the rotation rope_append_kernel (the prefill path) computes, so the reference is anchored in two steps:
  * rope_append (llmlb_op_rope_append, no page written) rotates a copy of the same qkv rows at positions L - 1, and that
    copy is checked against the fp64 rotation by the GPU table (rope_check, as for prefill);
  * the decode output must meet attention_ref (tests/test_kernels_sm90_gpu.py) on (rotated q, context K ++ rotated k,
    context V ++ v) with today's bound — P rounded to bf16 for the tensor-core kernel only.
After each launch every word of the K and V pools must equal the pool before it with only each sequence's new slot
replaced: K by rope_append's rotated k for that row, bit for bit (the prefix cache publishes pages of generated tokens, and
later requests attend over them as if prefill had written them), V by the input v.  qkv, seq_lens, bt_rows and the block
table must come back unchanged and the output must stay inside its NaN guard band.

The pool is poisoned (every slot a sequence has not written holds K ~ +-30, V ~ +-1e3, the new token's slot included until
the kernel writes it) and permuted; block-table rows are slot ids, not 0..B-1, and every table entry past a sequence's pages
points at a spare poisoned page.  Context lengths (including the new token) 1, 2, 31..33 and 63..65 (the tensor-core
kernel's 32-token chunks and the 64-token pages), 4097 and 131071; a second step on the same pool at L + 1 attends over the
k the first one appended, opens a new page for the 64-token sequence and puts the long sequence's new token at position
131071, the last of the table.

DECODE_CASES is plain data: tests/test_kernel_coverage_cpu.py runs it through the library over the fake CUDA runtime and
checks that it launches every decode class of the engine's launch plans (tp = 1 at Llama-3-8B, LLAMA_TINY, LLAMA_MID and
Llama-3-70B shapes; the 8B and 70B shards at tp 2, 4 and 8) at the smallest and the largest batch the engine uses it at.
"""
import pytest

from test_kernels_sm90_gpu import BF16_U, POISON_K, POISON_V, _Out, _poison, _report, attention_ref, bits_equal
from test_step_kernels_sm90_gpu import ROPE_MAX_POS, rope_check, rope_pool_expected, rope_table  # noqa: F401 (fixture)

# ---------------------------------------------------------------------------------------------------------------- cases --
SM_COUNT = 132
HEADS_TP1 = [(8, 2), (16, 4), (32, 8), (64, 8)]                 # LLAMA_TINY, LLAMA_MID, Llama-3-8B, Llama-3-70B
HEADS_SHARDS = [(16, 4), (8, 2), (4, 1), (32, 4), (16, 2), (8, 1)]   # 8B at tp 2 / 4 / 8, 70B at tp 2 / 4 / 8
MAX_BATCH = 128


def decode_splits(nb, n_heads):
    """The engine's KV split for a decode step of nb sequences (engine.cu, decode_splits): 1 = the tensor-core kernel when
    the step has more than 4 sequences and at least 96 (sequence, head group) pairs, else enough splits to give the 132
    SMs two CTAs each, at most 16."""
    ctas = nb * (n_heads // 4)
    if nb > 4 and ctas >= 96:
        return 1
    return max(1, min(16, -(-2 * SM_COUNT // ctas)))


def cluster_size(splits):
    """decode_attention_launch rounds the split down to a cluster size; 1 = the tensor-core kernel."""
    return max(c for c in (1, 2, 4, 8, 16) if c <= splits)


# (splits, n_heads, n_kv, batch): every (cluster size, n_heads, n_kv) class at the smallest and the largest batch of 1..128
# the engine launches it at, with the split the engine passes there (decode_splits; a CPU test derives this table from it)
DECODE_CASES = [
    (16, 8, 2, 1), (16, 8, 2, 8), (15, 8, 2, 9), (8, 8, 2, 18), (7, 8, 2, 19), (4, 8, 2, 43), (3, 8, 2, 44), (3, 8, 2, 47),
    (1, 8, 2, 48), (1, 8, 2, 128),
    (16, 16, 4, 1), (16, 16, 4, 4), (14, 16, 4, 5), (8, 16, 4, 9), (7, 16, 4, 10), (4, 16, 4, 21), (3, 16, 4, 22),
    (3, 16, 4, 23), (1, 16, 4, 24), (1, 16, 4, 128),
    (16, 32, 8, 1), (16, 32, 8, 2), (11, 32, 8, 3), (9, 32, 8, 4), (7, 32, 8, 5), (4, 32, 8, 10), (3, 32, 8, 11),
    (1, 32, 8, 12), (1, 32, 8, 128),
    (16, 64, 8, 1), (9, 64, 8, 2), (6, 64, 8, 3), (4, 64, 8, 5), (1, 64, 8, 6), (1, 64, 8, 128),
    (16, 4, 1, 1), (16, 4, 1, 17), (15, 4, 1, 18), (8, 4, 1, 37), (7, 4, 1, 38), (4, 4, 1, 87), (3, 4, 1, 88), (3, 4, 1, 95),
    (1, 4, 1, 96), (1, 4, 1, 128),
    (16, 32, 4, 1), (16, 32, 4, 2), (11, 32, 4, 3), (9, 32, 4, 4), (7, 32, 4, 5), (4, 32, 4, 10), (3, 32, 4, 11),
    (1, 32, 4, 12), (1, 32, 4, 128),
    (16, 16, 2, 1), (16, 16, 2, 4), (14, 16, 2, 5), (8, 16, 2, 9), (7, 16, 2, 10), (4, 16, 2, 21), (3, 16, 2, 22),
    (3, 16, 2, 23), (1, 16, 2, 24), (1, 16, 2, 128),
    (16, 8, 1, 1), (16, 8, 1, 8), (15, 8, 1, 9), (8, 8, 1, 18), (7, 8, 1, 19), (4, 8, 1, 43), (3, 8, 1, 44), (3, 8, 1, 47),
    (1, 8, 1, 48), (1, 8, 1, 128),
]


def derived_cases(heads=HEADS_TP1 + HEADS_SHARDS, max_batch=MAX_BATCH):
    """DECODE_CASES as decode_splits gives them: per head shape and class, the first and the last batch of 1..max_batch."""
    out = []
    for nh, nkv in dict.fromkeys(heads):
        seen = {}
        for nb in range(1, max_batch + 1):
            sp = decode_splits(nb, nh)
            seen.setdefault(cluster_size(sp), []).append((sp, nb))
        for c in sorted(seen, reverse=True):
            for sp, nb in dict.fromkeys([seen[c][0], seen[c][-1]]):
                out.append((sp, nh, nkv, nb))
    return out


LENS = (1, 2, 31, 32, 33, 63, 64, 65, 4097)   # tokens including the new one, first step
LONG = ROPE_MAX_POS - 1                        # new token at position 131070, at the second step 131071: the table's last row
SCALES = (1, 4, 16)                            # q x scale per row: scores from nearly flat to nearly one-hot


def launch_lens(B):
    """The sequence lengths of the launches of a B-wide case: every length of LENS and LONG once, the rest of each launch
    filled with LENS again; as many launches as that takes."""
    base = list(LENS) + [LONG]
    n = -(-len(base) // B) * B
    flat = base + [LENS[i % len(LENS)] for i in range(n - len(base))]
    return [flat[j * B:(j + 1) * B] for j in range(n // B)]


# --------------------------------------------------------------------------------------------------- reference math --
def new_slots(bt, rows, seq_lens):
    """(positions L - 1, pages) of the new tokens of a launch."""
    pos = (seq_lens - 1).long()
    return pos, bt[rows.long(), pos // 64].long()


def pools_expected(kp0, vp0, bt, rows, seq_lens, qkv, rot, nh, nkv):
    """The K and V pools after a decode launch: the pools before it with each sequence's new slot holding the rotated k as
    rope_append left it in `rot` and the input v."""
    pos, page = new_slots(bt, rows, seq_lens)
    return rope_pool_expected(kp0, vp0, qkv, rot, pos, page, nh, nkv)


def attention_errors(out, qkv, rot, ctx_k, ctx_v, seq_lens, nh, nkv, p_round):
    """(elements of out [B, nh * 128] over attention_ref's bound, NaN included; largest err / bound).  Sequence b attends
    with rot's q over ctx_k[b] ++ rot's k and ctx_v[b] ++ qkv's v; one kv head (and its q heads) per reference call when the
    context is long, so that fp64 copies of a 131071-token context stay small."""
    import torch
    g = nh // nkv
    bad, ratios = [], []
    for b, L in enumerate(seq_lens.tolist()):
        q = rot[b, : nh * 128].view(1, nh, 128)
        k = torch.cat([ctx_k[b], rot[b, nh * 128:(nh + nkv) * 128].view(1, nkv, 128)])
        v = torch.cat([ctx_v[b], qkv[b, (nh + nkv) * 128:].view(1, nkv, 128)])
        assert k.shape[0] == L
        step = max(1, min(nkv, (1 << 20) // (L * g)))
        for h0 in range(0, nkv, step):
            h1 = min(nkv, h0 + step)
            ref, bound = attention_ref(q[:, h0 * g:h1 * g], k[:, h0:h1], v[:, h0:h1], torch.tensor([L - 1], device=q.device), p_round)
            err = (out[b].view(1, nh, 128)[:, h0 * g:h1 * g].double() - ref).abs()
            bad.append((~(err <= bound)).sum())
            ratios.append((err / bound).max())
    return int(torch.stack(bad).sum()), float(torch.stack(ratios).max())


def decode_rejects(out, kp, vp, kp0, vp0, bt, rows, seq_lens, qkv, rot, ctx_k, ctx_v, nh, nkv, p_round):
    """Everything the GPU test holds a decode launch to, given rope_append's rotation `rot` of its qkv rows: (output
    elements over the bound, K pool words and V pool words other than expected, largest err / bound)."""
    kw, vw = pools_expected(kp0, vp0, bt, rows, seq_lens, qkv, rot, nh, nkv)
    n_out, ratio = attention_errors(out, qkv, rot, ctx_k, ctx_v, seq_lens, nh, nkv, p_round)
    return n_out, bits_equal(kp, kw), bits_equal(vp, vw), ratio


# ------------------------------------------------------------------------------------------------------- GPU tests --
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(built_lib):
    from llmlb_b200 import ffi
    return ffi.lib()


class Pool:
    """Paged K/V pools [n_pages][nkv][64][128] full of poison.  Sequence i owns shuffled pages for positions [0, horizon_i);
    its block-table row is rows[i], a slot id among n_seqs + 3 rows; every other table entry points at a spare page."""

    def __init__(self, nkv, horizons, seed, spare=3, device="cuda"):
        import torch
        gen = torch.Generator(device=device).manual_seed(seed)
        cpu = torch.Generator().manual_seed(seed)
        need = [-(-h // 64) for h in horizons]
        self.bt_stride = max(need) + 1
        self.n_pages = sum(need) + spare
        shape = (self.n_pages, nkv, 64, 128)
        self.kp, self.vp = _poison(shape, POISON_K, gen, device), _poison(shape, POISON_V, gen, device)
        perm = torch.randperm(self.n_pages, generator=cpu)
        n_rows = len(horizons) + 3
        rows = torch.randperm(n_rows, generator=cpu)[: len(horizons)]
        bt = perm[sum(need):][torch.randint(0, spare, (n_rows, self.bt_stride), generator=cpu)]
        off = 0
        for r, n in zip(rows.tolist(), need):
            bt[r, :n] = perm[off: off + n]
            off += n
        self.bt = bt.to(torch.int32).to(device)
        self.rows = rows.to(torch.int32).to(device)

    def write(self, i, pos0, k, v):
        """K/V of sequence i for positions [pos0, pos0 + len(k))."""
        import torch
        pos = torch.arange(pos0, pos0 + k.shape[0], device=k.device)
        pages = self.bt[int(self.rows[i])][(pos // 64).long()].long()
        self.kp[pages, :, pos % 64] = k
        self.vp[pages, :, pos % 64] = v


def qkv_rows(n, nh, nkv, gen, row0=0):
    """Random bf16 qkv rows, the q heads of row r scaled by SCALES[(row0 + r) % 3]."""
    import torch
    x = torch.randn(n, (nh + 2 * nkv) * 128, generator=gen, device=gen.device)
    x[:, : nh * 128] *= torch.tensor([SCALES[(row0 + r) % len(SCALES)] for r in range(n)], device=gen.device)[:, None]
    return x.to(torch.bfloat16)


def rope_rotate(L, qkv, pos, table, nh, nkv):
    """rope_append's rotation of the rows at `pos`, on a copy (page -1 everywhere: nothing is appended)."""
    import torch
    from gpu_util import ok, p, stream_ptr
    rot = qkv.clone()
    none = torch.full_like(pos, -1)
    scratch = torch.empty(64, dtype=torch.bfloat16, device=qkv.device)
    ok(L.llmlb_op_rope_append(p(rot), p(pos), p(none), p(table), p(scratch), p(scratch), qkv.shape[0], nh, nkv, stream_ptr()))
    return rot


def launch(L, pool, qkv, seq_lens, out_ptr, nh, nkv, table, splits, pdl):
    """llmlb_debug_decode_attention over the whole batch: the engine's launch (pdl: programmatic, as at layers >= 1)."""
    import torch
    from gpu_util import ok, p, stream_ptr
    ws = torch.zeros(256, dtype=torch.uint8, device=qkv.device)
    ok(L.llmlb_debug_decode_attention(p(qkv), p(pool.kp), p(pool.vp), p(pool.bt), pool.bt_stride, p(pool.rows), p(seq_lens),
                                      qkv.shape[0], out_ptr, nh, nkv, p(table), splits, qkv.shape[0], p(ws), int(pdl), stream_ptr()))


def check_launch(L, table, pool, kp0, vp0, qkv, rot, out, ctx_k, ctx_v, seq_lens, nh, nkv, splits, what):
    """rope_append's rotation against fp64, then the decode launch against rope_append and fp64: returns err / bound."""
    n_bad, rratio = rope_check(qkv, rot, seq_lens.long() - 1, table, nh, nkv)
    assert n_bad == 0, "%s: %d rope_append elements wrong (largest err/bound %.3g)" % (what, n_bad, rratio)
    p_round = BF16_U if splits == 1 else 0.0
    n_out, bad_k, bad_v, ratio = decode_rejects(out, pool.kp, pool.vp, kp0, vp0, pool.bt, pool.rows, seq_lens, qkv, rot,
                                                ctx_k, ctx_v, nh, nkv, p_round)
    assert bad_k == 0, "%s: %d K pool words differ from rope_append's k in the new slots / the pool before" % (what, bad_k)
    assert bad_v == 0, "%s: %d V pool words differ from the input v in the new slots / the pool before" % (what, bad_v)
    assert n_out == 0, "%s: %d output elements over the bound (largest err/bound %.3g)" % (what, n_out, ratio)
    return ratio


@pytest.mark.parametrize("splits,nh,nkv,B", DECODE_CASES, ids=["sp%d-h%d-kv%d-B%d" % c for c in DECODE_CASES])
def test_decode_attention_with_the_llama31_table_matches_rope_append_and_fp64(L, rope_table, splits, nh, nkv, B):
    import torch
    from gpu_util import sync
    ratio = 0.0
    for j, lens in enumerate(launch_lens(B)):
        seed = splits * 100000 + nh * 1000 + nkv * 100 + B + j
        pool = Pool(nkv, [n + 1 for n in lens], seed)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        ctx_k = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
        ctx_v = [torch.randn(n - 1, nkv, 128, generator=gen, device="cuda").to(torch.bfloat16) for n in lens]
        for i, n in enumerate(lens):
            if n > 1:
                pool.write(i, 0, ctx_k[i], ctx_v[i])
        for step in (0, 1):
            what = "launch %d step %d, lengths %s" % (j, step, sorted(set(n + step for n in lens)))
            seq_lens = torch.tensor([n + step for n in lens], dtype=torch.int32, device="cuda")
            qkv = qkv_rows(B, nh, nkv, gen, row0=j + step)
            inputs = [t.clone() for t in (qkv, seq_lens, pool.rows, pool.bt)]
            kp0, vp0 = pool.kp.clone(), pool.vp.clone()
            out = _Out(B, nh * 128, torch.bfloat16, pad=0)
            launch(L, pool, qkv, seq_lens, out.ptr(), nh, nkv, rope_table, splits, pdl=step)
            sync()
            assert out.untouched_outside(1) == 0, what + ": stray writes outside the output"
            assert all(torch.equal(a, b) for a, b in zip((qkv, seq_lens, pool.rows, pool.bt), inputs)), what + ": an input changed"
            rot = rope_rotate(L, qkv, seq_lens - 1, rope_table, nh, nkv)
            sync()
            ratio = max(ratio, check_launch(L, rope_table, pool, kp0, vp0, qkv, rot, out.slot(0), ctx_k, ctx_v, seq_lens, nh, nkv,
                                            splits, what))
            del kp0, vp0
            for b in range(B):                  # the next step attends over the k and v this one appended
                ctx_k[b] = torch.cat([ctx_k[b], rot[b, nh * 128:(nh + nkv) * 128].view(1, nkv, 128)])
                ctx_v[b] = torch.cat([ctx_v[b], qkv[b, (nh + nkv) * 128:].view(1, nkv, 128)])
        del pool, ctx_k, ctx_v
    _report("decode, cluster %d, %d/%d heads" % (cluster_size(splits), nh, nkv), ratio)
