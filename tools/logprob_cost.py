"""What logprobs cost a decode step: Llama-3-8B shapes (synthetic weights), batch 1 and batch 64, every request with
top_logprobs 20, every request with top_logprobs 0, or no logprobs.  The step time is the engine's own CUDA-event time
per decode step (health: gpu_ms_decode / steps_decode) over a window that starts after every sequence is decoding; the
three cases alternate, twice each.  Also times logprob_kernel alone (llmlb_op_logprobs, CUDA events over 200 launches)
on 1 and 64 rows of 128256 LM-like logits, with 20 and with 0 alternatives.
usage: python tools/logprob_cost.py [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

CASES = {"none": None, "top0": 0, "top20": 20}


def step_ms(e, batch, logprobs, n_new=160, warm=32):
    e.pause(True)
    rids = [e.submit([(7 * i + j) % 128256 for j in range(128)], n_new, ignore_eos=True, logprobs=logprobs) for i in range(batch)]
    e.pause(False)
    poll = e.poll if logprobs is None else e.poll_logprobs
    seen = 0
    while seen < warm:                     # every sequence is past prefill and the graphs of this width are captured
        seen += sum(x["token_id"] >= 0 for x in poll(rids[0], timeout_ms=-1))
    h0 = e.health()
    for r in rids:
        while True:
            ev = poll(r, timeout_ms=-1)
            if ev and ev[-1]["finish_reason"]:
                break
        if r == rids[0]:
            h1 = e.health()                # the window ends when the first request finishes (all run the same length)
    for r in rids:
        e.release(r)
    return (h1["gpu_ms_decode"] - h0["gpu_ms_decode"]) / max(1, h1["steps_decode"] - h0["steps_decode"])


def kernel_us(rows, n, vocab=128256, reps=200):
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    logits = torch.randn(rows, vocab, device="cuda", generator=g) * 2
    logits[:, :8] += 10                    # a few tokens well above the bulk, as a language model's row has
    tokens = torch.zeros(rows, device="cuda", dtype=torch.int32)
    top = torch.full((rows,), n, device="cuda", dtype=torch.int32)
    rec = torch.empty(rows * 42, device="cuda", dtype=torch.int32)
    args = (logits.data_ptr(), rows, vocab, tokens.data_ptr(), top.data_ptr(), rec.data_ptr(), None)
    L = ffi.lib()
    for _ in range(10):
        assert L.llmlb_op_logprobs(*args) == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        L.llmlb_op_logprobs(*args)
    b.record()
    torch.cuda.synchronize()
    return {"rows": rows, "top_logprobs": n, "us": round(a.elapsed_time(b) * 1e3 / reps, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "kernel": [kernel_us(r, n) for r in (1, 64) for n in (20, 0)], "decode_step_ms": {}}
    with ffi.Engine(ffi.LLAMA3_8B, max_seqs=64, max_ctx=1024, seed=0) as e:
        for batch in (1, 64):
            runs = {k: [] for k in CASES}
            for _ in range(2):
                for k, lp in CASES.items():
                    runs[k].append(round(step_ms(e, batch, lp), 4))
            res["decode_step_ms"]["batch%d" % batch] = runs
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print("wall %.1f s" % (time.time() - t0), file=sys.stderr)
