"""What serving n choices of one prompt costs, three ways, at Llama-3-8B shapes (synthetic weights, max_ctx 4096, max_seqs 16):
  group:  one llmlb_request_submit_choices of n (one prefill, then a kv_fork of the prompt's tail page);
  lone:   n llmlb_request_submit of the same prompt with seeds s + i, prefix cache off;
  cached: the same n lone requests with the prefix cache on (requests admitted in one iteration match before any publishes).
Prompts of 512 and 2000 tokens, 128 tokens out, n in 1, 2, 4, 8, 16, temperature 0.8.  Per case: wall ms until every choice has
its first token, total wall ms, and the engine's tokens_prefill.  Separately, the kv_fork kernel alone (llmlb_op_kv_fork) at
8 KV heads and 32 layers, rows 63, for 1..15 destinations, timed with CUDA events.  Prints one JSON line with the card's name
and power limit.
usage: python tools/choices_cost.py [--out file.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

CFG = ffi.LLAMA3_8B
KW = dict(max_seqs=16, max_ctx=4096, max_step_tokens=2048, seed=0)
M_OUT = 128


def serve(e, submit):
    """submit() -> ids, all at once; returns (ms until every id has a token, total ms)"""
    t0 = time.perf_counter()
    rids = submit()
    first, pending = {}, set(rids)
    while pending:
        for r in list(pending):
            for ev in e.poll(r, timeout_ms=1):
                if ev["token_id"] >= 0:
                    first.setdefault(r, time.perf_counter())
                if ev["finish_reason"]:
                    pending.discard(r)
    t1 = time.perf_counter()
    for r in rids:
        e.release(r)
    return 1e3 * (max(first.values()) - t0), 1e3 * (t1 - t0)


def run_mode(mode):
    """every (L, n) case on one engine, each on a prompt of its own (so that the cache only shares within a case)"""
    out = []
    with ffi.Engine(CFG, prefix_cache=mode == "cached", **KW) as e:
        warm = np.random.RandomState(1).randint(0, CFG["vocab"], 300).tolist()
        serve(e, lambda: e.submit_choices(warm, 8, 16, ignore_eos=True))     # graphs of every decode width
        for L in (512, 2000):
            for n in (1, 2, 4, 8, 16):
                P = np.random.RandomState(L * 100 + n).randint(0, CFG["vocab"], L).tolist()
                t0 = e.health()["tokens_prefill"]
                kw = dict(ignore_eos=True, temperature=0.8, seed=11)
                if mode == "group":
                    ttf, tot = serve(e, lambda: e.submit_choices(P, M_OUT, n, **kw))
                else:
                    ttf, tot = serve(e, lambda: [e.submit(P, M_OUT, **dict(kw, seed=11 + i)) for i in range(n)])
                out.append(dict(L=L, n=n, mode=mode, first_token_ms=round(ttf, 2), total_ms=round(tot, 2),
                                tokens_prefill=e.health()["tokens_prefill"] - t0))
                print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def kv_fork_us():
    import torch
    n_layers, n_kv, n_pages = 32, 8, 64
    k = torch.zeros((n_layers, n_pages, n_kv, 64, 128), dtype=torch.bfloat16, device="cuda")
    v = torch.zeros_like(k)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for nd in (1, 3, 7, 15):
        d = torch.arange(1, nd + 1, dtype=torch.int32, device="cuda")
        call = lambda: ffi.check(ffi.lib().llmlb_op_kv_fork(C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()), n_layers, n_pages,
                                                            n_kv, 0, C.c_void_p(d.data_ptr()), nd, 63, st))
        for _ in range(5):
            call()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(50):
            call()
        b.record()
        torch.cuda.synchronize()
        out[nd] = round(1e3 * a.elapsed_time(b) / 50, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(card=card, model="Llama-3-8B synthetic", max_tokens=M_OUT, kv_fork_us_rows63_32layers_8kv=kv_fork_us(), cases=[])
    for mode in ("group", "lone", "cached"):
        res["cases"] += run_mode(mode)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
