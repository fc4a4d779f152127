"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) through one fixed
workload — prefill steps of several widths, then decode batches of width 1..64 — so that tests/test_penalties_cpu.py can
compare the launch plans of the same workload submitted three ways.  Llama-3-8B widths, two layers (launch shapes do not
depend on the depth).
usage: penalty_plan_sweep.py plain|neutral|mixed graphs|eager
  plain:   llmlb_request_submit
  neutral: llmlb_request_submit_penalized with both penalties 0 and no bias
  mixed:   every even-numbered request of a batch penalised (frequency, presence and a bias), the others not"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ["FAKE_CUDART_LAUNCH_LOG"]
PREFILL_WIDTHS = (1, 2, 4, 5, 64, 300, 2048)
DECODE_WIDTHS_EAGER = (1, 2, 3, 4, 5, 8, 17, 33, 63, 64)


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


def drain(e, rid):
    while True:
        ev = e.poll(rid, timeout_ms=-1)
        if ev and ev[-1]["finish_reason"]:
            assert ev[-1]["finish_reason"] == ffi.FINISH_LENGTH, ev[-1]
            break
    e.release(rid)


def main():
    mode, graphs = sys.argv[1], sys.argv[2] == "graphs"

    def submit(e, prompt, n, i):
        if mode == "plain":
            return e.submit(prompt, n, ignore_eos=True)
        if mode == "neutral" or i % 2:
            return e.submit(prompt, n, ignore_eos=True, frequency_penalty=0.0, presence_penalty=0.0, logit_bias={})
        return e.submit(prompt, n, ignore_eos=True, frequency_penalty=0.5, presence_penalty=-0.25, logit_bias={5: 1.0, 7: -2.0})

    model = dict(ffi.LLAMA3_8B, n_layers=2)
    with ffi.Engine(model, max_seqs=64, max_ctx=4096, max_step_tokens=2048, use_cuda_graphs=graphs) as e:
        for T in PREFILL_WIDTHS:
            mark("prefill T=%d" % T)
            drain(e, submit(e, [1] * T, 1, 0))
        for B in (range(1, 65) if graphs else DECODE_WIDTHS_EAGER):
            mark("decode B=%d" % B)
            e.pause(True)
            rids = [submit(e, [1] * 8, 3, i) for i in range(B)]
            e.pause(False)
            for r in rids:
                drain(e, r)


if __name__ == "__main__":
    main()
