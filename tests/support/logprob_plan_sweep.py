"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) through one fixed
workload — prefill steps of several widths, then decode batches of width 1..64 — so that tests/test_logprobs_cpu.py can
compare the launch plans of the same workload submitted three ways.  Llama-3-8B widths, two layers (launch shapes do not
depend on the depth).
usage: logprob_plan_sweep.py plain|nolp|mixed graphs|eager
  plain: llmlb_request_submit, drained with llmlb_request_poll
  nolp:  llmlb_request_submit_penalized with no penalties (NULL), drained with llmlb_request_poll_logprobs
  mixed: every even-numbered request of a batch reports logprobs (top_logprobs 20 and 0 alternately), the others not"""
import ctypes as C
import math
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


def main():
    mode, graphs = sys.argv[1], sys.argv[2] == "graphs"

    def submit(e, prompt, n, i):
        if mode == "plain":
            return e.submit(prompt, n, ignore_eos=True)
        if mode == "nolp" or i % 2:
            arr = (C.c_int32 * len(prompt))(*prompt)
            s = ffi.Sampling(max_tokens=n, ignore_eos=1)
            rid = C.c_uint64()
            ffi.check(ffi.lib().llmlb_request_submit_penalized(e._h, arr, len(prompt), C.byref(s), None, C.byref(rid)))
            return rid.value
        return e.submit(prompt, n, ignore_eos=True, logprobs=20 if i % 4 == 0 else 0)

    def drain(e, rid, i):
        while True:
            ev = e.poll(rid, timeout_ms=-1) if mode == "plain" else e.poll_logprobs(rid, timeout_ms=-1)
            if mode == "mixed":     # the fake runtime computes nothing: the records are whatever the pinned ring holds,
                for x in ev:        # but an event of a request without logprobs must say so
                    if i % 2 and x["token_id"] >= 0:
                        assert math.isnan(x["logprob"]) and x["top_logprobs"] == [], x
            if ev and ev[-1]["finish_reason"]:
                assert ev[-1]["finish_reason"] == ffi.FINISH_LENGTH, ev[-1]
                break
        e.release(rid)

    model = dict(ffi.LLAMA3_8B, n_layers=2)
    with ffi.Engine(model, max_seqs=64, max_ctx=4096, max_step_tokens=2048, use_cuda_graphs=graphs) as e:
        for T in PREFILL_WIDTHS:
            mark("prefill T=%d" % T)
            drain(e, submit(e, [1] * T, 1, 0), 0)
        for B in (range(1, 65) if graphs else DECODE_WIDTHS_EAGER):
            mark("decode B=%d" % B)
            e.pause(True)
            rids = [submit(e, [1] * 8, 3, i) for i in range(B)]
            e.pause(False)
            for i, r in enumerate(rids):
                drain(e, r, i)


if __name__ == "__main__":
    main()
