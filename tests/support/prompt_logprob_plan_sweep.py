"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) through one fixed
workload of logprob requests — prefills of several widths, a prompt chunked over three prefill steps, decode batches — so that
tests/test_prompt_logprobs_cpu.py can compare the launch plans of the same workload submitted with and without prompt
logprobs.  Llama-3-8B widths, two layers (launch shapes do not depend on the depth).  Every request is drained to its end;
in prompt mode its prompt records are read after its first event, and there must be exactly n_prompt - 1 of them.
usage: prompt_logprob_plan_sweep.py lp|prompt graphs|eager <max_seqs> [tp]
  lp:     llmlb_request_submit_logprobs (top_logprobs 5 and 0 alternately)
  prompt: the same through llmlb_request_submit_prompt_logprobs"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ.get("FAKE_CUDART_LAUNCH_LOG")   # read by the test for the workload constants, without a log
PREFILL_WIDTHS = (1, 2, 5, 9, 64, 300, 2048)
CHUNKED = 4500          # three prefill steps of max_step_tokens 2048
DECODE_BATCHES = (1, 3, 8)


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


def main():
    mode, graphs, max_seqs = sys.argv[1], sys.argv[2] == "graphs", int(sys.argv[3])
    tp = int(sys.argv[4]) if len(sys.argv) > 4 else 1
    prompt_lp = mode == "prompt"
    model = dict(ffi.LLAMA3_8B, n_layers=2)
    engs = [ffi.Engine(model, tp_rank=r, tp_size=tp, max_seqs=max_seqs, max_ctx=8192, max_step_tokens=2048, use_cuda_graphs=graphs)
            for r in range(tp)]
    if tp > 1:
        hs = [e.tp_export() for e in engs]
        for e in engs:
            e.tp_import(hs)

    def drain(e, rid, n_prompt):
        recs, first = None, True
        while True:
            ev = e.poll_logprobs(rid, timeout_ms=-1)
            if prompt_lp and first and ev:
                recs = e.poll_prompt_logprobs(rid, cap=8192)
                assert len(recs) == n_prompt - 1, (len(recs), n_prompt)
                first = False
            if ev and ev[-1]["finish_reason"]:
                assert ev[-1]["finish_reason"] == ffi.FINISH_LENGTH, ev[-1]
                break
        if prompt_lp:
            assert e.poll_prompt_logprobs(rid) == []
        e.release(rid)

    def run(prompts, max_tokens):
        for e in engs:
            e.pause(True)
            rids = [e.submit(p, max_tokens, ignore_eos=True, logprobs=5 if i % 2 == 0 else 0, prompt_logprobs=prompt_lp)
                    for i, p in enumerate(prompts)]
            e.pause(False)
            for r, p in zip(rids, prompts):
                drain(e, r, len(p))

    for T in PREFILL_WIDTHS:
        mark("prefill T=%d" % T)
        run([[(7 * j) % 1000 + 1 for j in range(T)]], 2)
    mark("chunked T=%d" % CHUNKED)
    run([[(3 * j) % 1000 + 1 for j in range(CHUNKED)]], 2)
    for B in DECODE_BATCHES:
        mark("decode B=%d" % B)
        run([[(5 * i + j) % 1000 + 1 for j in range(8 + i)] for i in range(B)], 3)
    for e in engs:
        e.close()


if __name__ == "__main__":
    main()
