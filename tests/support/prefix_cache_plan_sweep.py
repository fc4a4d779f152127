"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) so that
tests/test_prefix_cache_cpu.py can compare launch plans with the prefix cache off and on.  Llama-3-8B widths, two layers.
usage: prefix_cache_plan_sweep.py unique off|on graphs|eager
         prefills of several widths and decode batches, every prompt distinct from the first token on (no prefix to share)
       prefix_cache_plan_sweep.py shared off|on <k>
         max_step_tokens 64k, one token generated.  off: prompt P of 64k + 37 tokens (two prefill steps, split at 64k).
         on: P[:64k + 1] first, then P (a hit on k pages, then one prefill step of the 37-token suffix).
Prints one JSON line: per section, the prefill tokens and the cached_tokens of its last request."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ.get("FAKE_CUDART_LAUNCH_LOG")
PREFILL_WIDTHS = (1, 2, 5, 63, 64, 65, 129, 300, 2048)
DECODE_BATCHES = (1, 3, 8)
SUFFIX = 37


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


def main():
    kind, on = sys.argv[1], sys.argv[2] == "on"
    model = dict(ffi.LLAMA3_8B, n_layers=2)
    out = {}

    def run(e, section, prompts, max_tokens):
        mark(section)
        t0 = e.health()["tokens_prefill"]
        e.pause(True)
        rids = [e.submit(p, max_tokens, ignore_eos=True) for p in prompts]
        e.pause(False)
        for r in rids:
            while True:
                ev = e.poll(r, timeout_ms=-1)
                if ev and ev[-1]["finish_reason"]:
                    assert ev[-1]["finish_reason"] == ffi.FINISH_LENGTH, ev[-1]
                    break
        out[section] = (e.health()["tokens_prefill"] - t0, e.cached_tokens(rids[-1]))
        for r in rids:
            e.release(r)

    if kind == "unique":
        graphs = sys.argv[3] == "graphs"
        with ffi.Engine(model, max_seqs=8, max_ctx=4096, max_step_tokens=2048, use_cuda_graphs=graphs, prefix_cache=on) as e:
            for T in PREFILL_WIDTHS:
                run(e, "prefill T=%d" % T, [[(131 * T + 7 * j) % 1000 + 1 for j in range(T)]], 2)
            for B in DECODE_BATCHES:
                run(e, "decode B=%d" % B, [[(1000 + 17 * B + 5 * i + 3 * j) % 2000 + 1 for j in range(70 + i)] for i in range(B)], 3)
    else:
        k = int(sys.argv[3])
        P = [(11 * j) % 3000 + 1 for j in range(64 * k + SUFFIX)]
        with ffi.Engine(model, max_seqs=4, max_ctx=2048, max_step_tokens=64 * k, use_cuda_graphs=False, prefix_cache=on) as e:
            if on:
                run(e, "prefix", [P[:64 * k + 1]], 1)
            run(e, "P", [P], 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
