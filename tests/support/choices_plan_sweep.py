"""Drives the product engine over tests/support/fake_cudart.cpp (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) so that
tests/test_choices_cpu.py can read the launch plans of requests with n choices.  Llama-3-8B widths, two layers, eager
decode steps (every kernel of every step in the log).
usage: choices_plan_sweep.py one submit|choices off|on
         the same requests through llmlb_request_submit (and its penalised / logprob variants) or through
         llmlb_request_submit_choices with n = 1
       choices_plan_sweep.py group off|on
         one group per section "L=<prompt tokens> n=<choices>", each alone in the engine, 4 tokens out
Prints one JSON line: per section, the prefill tokens it caused and its prefill and decode steps."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ.get("FAKE_CUDART_LAUNCH_LOG")
GROUPS = [(L, n) for L in (65, 81, 104, 127, 128, 1000) for n in (2, 3, 8, 16)]
ONE = [dict(), dict(logprobs=2), dict(frequency_penalty=0.5, logit_bias={7: 3.0}), dict(logprobs=1, prompt_logprobs=True)]
M_OUT = 4


def mark(s):
    with open(LOG, "a") as f:
        f.write("### %s\n" % s)


def drain(e, rids):
    for r in rids:
        while True:
            ev = e.poll(r, timeout_ms=-1)
            if ev and ev[-1]["finish_reason"]:
                assert ev[-1]["finish_reason"] == ffi.FINISH_LENGTH, ev[-1]
                break
    for r in rids:
        e.release(r)


def main():
    kind, on = sys.argv[1], sys.argv[-1] == "on"
    model = dict(ffi.LLAMA3_8B, n_layers=2)
    out = {}
    with ffi.Engine(model, max_seqs=16, max_ctx=2048, max_step_tokens=1024, use_cuda_graphs=False, prefix_cache=on) as e:
        def run(section, submit):
            mark(section)
            h0 = e.health()
            e.pause(True)
            rids = submit()
            e.pause(False)
            drain(e, rids)
            h = e.health()
            out[section] = [h[k] - h0[k] for k in ("tokens_prefill", "steps_prefill", "steps_decode")]

        if kind == "one":
            api = sys.argv[2]
            for i, kw in enumerate(ONE):
                P = [(37 * i + 11 * j) % 3000 + 1 for j in range(90 + 70 * i)]
                if api == "submit":
                    run("one %d" % i, lambda: [e.submit(P, M_OUT, ignore_eos=True, seed=5, **kw)])
                else:
                    run("one %d" % i, lambda: e.submit_choices(P, M_OUT, 1, ignore_eos=True, seed=5, **kw))
        else:
            for i, (L, n) in enumerate(GROUPS):
                P = [(131 * i + 7 * j) % 3000 + 1 for j in range(L)]
                run("L=%d n=%d" % (L, n), lambda: e.submit_choices(P, M_OUT, n, ignore_eos=True, temperature=0.7, seed=3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
