"""What frequency / presence penalties cost a decode step: Llama-3-8B shapes (synthetic weights), batch 1 and batch 64,
every request penalised or none.  The step time is the engine's own CUDA-event time per decode step (health:
gpu_ms_decode / steps_decode) over a window that starts after every sequence is decoding; the two cases alternate, twice
each.  Also times penalize_kernel alone (llmlb_op_penalize, CUDA events over 200 launches) on 1 and 64 rows of 128256
logits, against the bytes it moves: counts read, logits read and written.
usage: python tools/penalty_cost.py [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

PEN = dict(frequency_penalty=0.5, presence_penalty=0.5, logit_bias={13: 1.0, 42: -1.0})


def step_ms(e, batch, penalised, n_new=160, warm=32):
    kw = PEN if penalised else {}
    e.pause(True)
    rids = [e.submit([(7 * i + j) % 128256 for j in range(128)], n_new, ignore_eos=True, **kw) for i in range(batch)]
    e.pause(False)
    seen = 0
    while seen < warm:                     # every sequence is past prefill and the graphs of this width are captured
        seen += sum(x["token_id"] >= 0 for x in e.poll(rids[0], timeout_ms=-1))
    h0 = e.health()
    for r in rids:
        while True:
            ev = e.poll(r, timeout_ms=-1)
            if ev and ev[-1]["finish_reason"]:
                break
        if r == rids[0]:
            h1 = e.health()                # the window ends when the first request finishes (all run the same length)
    for r in rids:
        e.release(r)
    return (h1["gpu_ms_decode"] - h0["gpu_ms_decode"]) / max(1, h1["steps_decode"] - h0["steps_decode"])


def kernel_us(rows, vocab=128256, reps=200):
    import torch
    logits = torch.randn(rows * vocab, device="cuda")
    counts = torch.randint(0, 3, (rows * vocab,), device="cuda", dtype=torch.int32)
    f = torch.full((rows,), 0.5, device="cuda")
    nb = torch.zeros(rows, device="cuda", dtype=torch.int32)
    args = (logits.data_ptr(), rows, vocab, counts.data_ptr(), vocab, f.data_ptr(), f.data_ptr(), None, None, nb.data_ptr(), 0, None)
    L = ffi.lib()
    for _ in range(10):
        assert L.llmlb_op_penalize(*args) == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        L.llmlb_op_penalize(*args)
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1e3 / reps
    nbytes = rows * vocab * 12
    return {"rows": rows, "us": round(us, 2), "MB": round(nbytes / 1e6, 2), "GB_per_s": round(nbytes / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "kernel": [kernel_us(1), kernel_us(64)], "decode_step_ms": {}}
    with ffi.Engine(ffi.LLAMA3_8B, max_seqs=64, max_ctx=1024, seed=0) as e:
        for batch in (1, 64):
            runs = {"none": [], "penalised": []}
            for _ in range(2):
                for pen in (False, True):
                    runs["penalised" if pen else "none"].append(round(step_ms(e, batch, pen), 4))
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
