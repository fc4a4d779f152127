"""What the prefix cache saves and costs, cache off against cache on, alternating, at Llama-3-8B shapes (synthetic weights,
max_ctx 8192, max_seqs 32).  Each round creates one engine per setting and runs three workloads on it:
  (a) shared prefix: 32 requests share a 4000-token prefix, each with its own 100-token suffix, 64 generated tokens;
  (b) chat: 8 conversations x 4 turns, each turn's prompt = the previous prompt + its reply + 50 new tokens, 64 generated;
  (c) no reuse: bench.py's shape, 32 unique 512-token prompts, 128 generated.
Per workload: the CUDA-event time of its prefill steps (health: gpu_ms_prefill), mean time to first token, generated tokens
per second of wall time, and prefill / decode tokens per second of CUDA-event time.  Prints one JSON line with the card's name
and power limit.
--host: instead, the host cost of one scheduling iteration, cache off and on, over the fake CUDA runtime (no GPU): batches
of 1 / 8 / 64 / 128 sequences decoding after a hit, wall time per decode step (the fake steps take no time).
usage: python tools/prefix_cache_cost.py [--rounds 2] [--host] [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

V = ffi.LLAMA3_8B["vocab"]


def serve(e, prompts, m):
    """all prompts at once; returns (wall s, first-token ms per request, generated tokens)"""
    t0 = time.time()
    rids = [e.submit(p, m, ignore_eos=True) for p in prompts]
    first, toks, out = {}, 0, {}
    pending = set(rids)
    while pending:
        for r in list(pending):
            for ev in e.poll(r, timeout_ms=1):
                if ev["token_id"] >= 0:
                    toks += 1
                    first.setdefault(r, ev["t_ms"])
                    out.setdefault(r, []).append(ev["token_id"])
                if ev["finish_reason"]:
                    pending.discard(r)
    wall = time.time() - t0
    for r in rids:
        e.release(r)
    return wall, [first[r] for r in rids], toks, [out[r] for r in rids]


def measure(e, fn):
    h0 = e.health()
    wall, ttft, toks = fn()
    h1 = e.health()
    d = {k: h1[k] - h0[k] for k in ("gpu_ms_prefill", "gpu_ms_decode", "tokens_prefill", "tokens_decode")}
    return dict(prefill_ms=round(d["gpu_ms_prefill"], 1), ttft_ms=round(float(np.mean(ttft)), 1), tok_s=round(toks / wall, 1),
                tokens_prefill=d["tokens_prefill"],
                prefill_tok_s=round(d["tokens_prefill"] / (d["gpu_ms_prefill"] / 1e3), 1) if d["gpu_ms_prefill"] else None,
                decode_tok_s=round(d["tokens_decode"] / (d["gpu_ms_decode"] / 1e3), 1) if d["gpu_ms_decode"] else None)


def workloads(e, rs):
    res = {}
    prefix = rs.randint(0, V, 4000).tolist()

    def shared():
        w, t, n, _ = serve(e, [prefix + rs.randint(0, V, 100).tolist() for _ in range(32)], 64)
        return w, t, n
    res["a_shared_prefix"] = measure(e, shared)

    hist = [rs.randint(0, V, 1000).tolist() for _ in range(8)]

    def chat():
        wall, ttft, n = 0.0, [], 0
        for _ in range(4):
            w, t, k, outs = serve(e, hist, 64)
            wall, ttft, n = wall + w, ttft + t, n + k
            for i in range(8):
                hist[i] = hist[i] + outs[i] + rs.randint(0, V, 50).tolist()
        return wall, ttft, n
    res["b_chat"] = measure(e, chat)

    def unique():
        w, t, n, _ = serve(e, [rs.randint(0, V, 512).tolist() for _ in range(32)], 128)
        return w, t, n
    res["c_no_reuse"] = measure(e, unique)
    return res


def gpu(rounds):
    name = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": name, "model": "llama-3-8b synthetic", "max_ctx": 8192, "max_seqs": 32, "rounds": []}
    for rnd in range(rounds):
        row = {}
        for on in (False, True):
            with ffi.Engine(ffi.LLAMA3_8B, max_seqs=32, max_ctx=8192, seed=0, prefix_cache=on) as e:
                serve(e, [np.random.RandomState(99).randint(0, V, 600).tolist()], 4)    # warm-up: first launches, graphs
                row["on" if on else "off"] = workloads(e, np.random.RandomState(1000 + rnd))   # the same tokens for both
                if on:
                    row["on"]["cache"] = e.prefix_cache_stats()
        res["rounds"].append(row)
    return res


def host():
    """re-executes itself over the fake CUDA runtime"""
    if os.environ.get("LLMLB_FAKE_CUDART") != "1":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import test_engine_host_logic_cpu as HL
        env = dict(os.environ, LD_PRELOAD=HL.build_fake(), LLMLB_FAKE_CUDART="1")
        return json.loads(subprocess.run([sys.executable, __file__, "--host"], env=env, capture_output=True, text=True, check=True).stdout)
    res = {"fake_cuda_runtime": True, "us_per_decode_step": {"off": {}, "on": {}}}
    model = dict(ffi.LLAMA3_8B, n_layers=2)
    for B, on in [(B, on) for B in (1, 8, 64, 128) for on in (False, True)]:
        with ffi.Engine(model, max_seqs=128, max_ctx=1024, prefix_cache=on) as e:
            prompts = [[(7 * i + 3 * j) % 1000 + 1 for j in range(200)] for i in range(B)]   # 200 tokens: pages to publish
            serve(e, prompts, 2)
            e.pause(True)
            rids = [e.submit(p, 400, ignore_eos=True) for p in prompts]                      # every sequence hits 3 pages
            h0, t0 = e.health(), time.time()
            e.pause(False)
            for r in rids:                                                                   # one blocking waiter at a time
                while not any(ev["finish_reason"] for ev in e.poll(r, cap=512, timeout_ms=-1)):
                    pass
            h1 = e.health()
            for r in rids:
                e.release(r)
            res["us_per_decode_step"]["on" if on else "off"][B] = round((time.time() - t0) * 1e6 / (h1["steps_decode"] - h0["steps_decode"]), 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = host() if a.host else gpu(a.rounds)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
