"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD) with FAKE_CUDART_LAUNCH_LOG set, so that the
log holds the engine's LAUNCH PLAN — kernel, grid, block, shared memory, cluster, PDL — for every prefill width 1..2048 and
every decode batch width 1..128 of a model geometry / tensor-parallel degree.  Two layers only: launch shapes do not depend
on the depth.  All `tp` ranks live in this one process (the fake runtime's IPC handles work within a process too) and run one
after the other: nothing executes, so nobody waits for a peer.
usage: launch_plan_sweep.py 8b|mid|70b|tiny <tp> [max_width]
  max_width: only prefill widths and decode batches up to it (the long-context batches too), and no 131072-token context —
  enough to see every decode GEMV launch (those run at 1..4 rows only) without the cost of the whole sweep."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ["FAKE_CUDART_LAUNCH_LOG"]
MODELS = {"8b": ffi.LLAMA3_8B, "mid": ffi.LLAMA_MID, "70b": ffi.LLAMA3_70B, "tiny": ffi.LLAMA_TINY}


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


def drain(e, rid):
    while True:
        ev = e.poll(rid, timeout_ms=-1)
        if ev and ev[-1]["finish_reason"]:
            break
    e.release(rid)


def main():
    model = dict(MODELS[sys.argv[1]], n_layers=2)
    tp = int(sys.argv[2])
    max_width = int(sys.argv[3]) if len(sys.argv) > 3 else None
    engs = [ffi.Engine(model, tp_rank=r, tp_size=tp, max_seqs=128, max_ctx=4096, max_step_tokens=2048) for r in range(tp)]
    if tp > 1:
        hs = [e.tp_export() for e in engs]
        for e in engs:
            e.tp_import(hs)
    for T in range(1, min(2048, max_width or 2048) + 1):
        mark("prefill T=%d" % T)
        for e in engs:
            drain(e, e.submit([1] * T, 1, ignore_eos=True))
    for B in range(1, min(128, max_width or 128) + 1):
        mark("decode B=%d" % B)
        for e in engs:
            e.pause(True)
            rids = [e.submit([1] * 8, 3, ignore_eos=True) for _ in range(B)]
            e.pause(False)
            for r in rids:
                drain(e, r)
    # long contexts: prompts chunked over two prefill steps (the second attends to cached pages), then decode over ~3900 tokens
    for B in (1, 3, 5, 32):
        if max_width and B > max_width:
            continue
        mark("long B=%d" % B)
        for e in engs:
            e.pause(True)
            rids = [e.submit([1] * (3800 + 7 * i), 4, ignore_eos=True) for i in range(B)]
            e.pause(False)
            for r in rids:
                drain(e, r)
    for e in engs:
        e.close()
    if max_width:
        return
    # a 131072-token context: 64 prefill chunks over ever longer cached contexts, then decode over 130 k tokens
    engs = [ffi.Engine(model, tp_rank=r, tp_size=tp, max_seqs=2, max_ctx=131072, max_step_tokens=2048) for r in range(tp)]
    if tp > 1:
        hs = [e.tp_export() for e in engs]
        for e in engs:
            e.tp_import(hs)
    mark("ctx131072")
    for e in engs:
        drain(e, e.submit([i % 1000 for i in range(130000)], 8, ignore_eos=True))
    for e in engs:
        e.close()


if __name__ == "__main__":
    main()
