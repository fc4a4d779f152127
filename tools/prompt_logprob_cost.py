"""What prompt logprobs cost a prefill: a 2048-token prompt at Llama-3-8B shapes (synthetic weights), one request at a
time, max_tokens 1, with logprobs (top 1, lm-eval's request) and without prompt logprobs, then with them; at max_seqs 8 and
64.  The time is the engine's own CUDA-event time of the prefill step (health: gpu_ms_prefill), which includes the prompt
groups; the cases alternate, three runs each after one warm-up of each.  Prints one JSON line with the card's name and power
limit.
usage: python tools/prompt_logprob_cost.py [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

N_PROMPT = 2048


def prefill_ms(e, prompt_lp):
    h0 = e.health()
    rid = e.submit([(7 * j) % 128000 + 1 for j in range(N_PROMPT)], 1, ignore_eos=True, logprobs=1, prompt_logprobs=prompt_lp)
    while True:
        ev = e.poll_logprobs(rid, timeout_ms=-1)
        if ev and ev[-1]["finish_reason"]:
            break
    n_rec = len(e.poll_prompt_logprobs(rid, cap=N_PROMPT))
    assert n_rec == (N_PROMPT - 1 if prompt_lp else 0), n_rec
    e.release(rid)
    h1 = e.health()
    assert h1["steps_prefill"] - h0["steps_prefill"] == 1
    return h1["gpu_ms_prefill"] - h0["gpu_ms_prefill"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "n_prompt": N_PROMPT, "prefill_ms": {}}
    for max_seqs in (8, 64):
        with ffi.Engine(ffi.LLAMA3_8B, max_seqs=max_seqs, max_ctx=N_PROMPT + 64, max_step_tokens=N_PROMPT, seed=0) as e:
            prefill_ms(e, False)
            prefill_ms(e, True)
            runs = {"without": [], "with": []}
            for _ in range(3):
                runs["without"].append(round(prefill_ms(e, False), 3))
                runs["with"].append(round(prefill_ms(e, True), 3))
            res["prefill_ms"]["max_seqs%d" % max_seqs] = runs
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print("wall %.1f s" % (time.time() - t0), file=sys.stderr)
