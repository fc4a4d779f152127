"""Per-CTA timeline of one batch-1 decode step (debug hook llmlb_debug_trace_*): where the time
between the HBM-bound GEMVs goes.  Run on the GPU box: python tools/decode_timeline.py"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from llmlb_b200 import ffi  # noqa: E402


def main():
    L = ffi.lib()
    L.llmlb_debug_trace_enable.argtypes = [C.c_uint32]
    L.llmlb_debug_trace_dump.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    model = ffi.LLAMA3_8B
    eng = ffi.Engine(model, max_seqs=4, max_ctx=1024, use_cuda_graphs=os.environ.get("GRAPHS", "1") == "1")
    prompt = np.random.RandomState(0).randint(0, model["vocab"], 512).tolist()
    eng.generate(prompt, 8, ignore_eos=True)           # warm
    cap = 400000
    L.llmlb_debug_trace_enable(cap)
    eng.generate(prompt, 6, ignore_eos=True)
    buf = np.zeros((cap, 6), dtype=np.uint64)
    n = C.c_uint32()
    L.llmlb_debug_trace_dump(buf.ctypes.data, cap, C.byref(n))
    L.llmlb_debug_trace_enable(0)
    eng.close()
    r = buf[: n.value]
    if os.environ.get("TRACE_OUT"):
        np.save(os.environ["TRACE_OUT"], r)
    # group records into launches: per tag, records sorted by start time come in blocks of one
    # grid (PDL lets adjacent kernels overlap in time, so grouping must be per kernel type)
    launches = []
    for tag in np.unique(r[:, 0]):
        rows = r[r[:, 0] == tag]
        rows = rows[np.argsort(rows[:, 5])]
        grid = 128 if int(tag) == 1 else 132
        for i in range(0, len(rows) - grid + 1, grid):
            blk = rows[i:i + grid]
            launches.append({"tag": int(tag), "rows": list(blk), "mid": float(np.median(blk[:, 5].astype(np.float64)))})
    launches.sort(key=lambda l: l["mid"])
    # keep the last full decode step: launches after the last lm_head (n_out=128256)
    def name(tag):
        if tag == 1:
            return "attention"
        return "gemv %dx%d" % (tag >> 32, tag & 0xFFFFFFFF)
    idx = [i for i, l in enumerate(launches) if name(l["tag"]).startswith("gemv 128256")]
    if len(idx) >= 2:
        launches = launches[idx[-2] + 1: idx[-1] + 1]
    t_base = min(int(x[2]) for x in launches[0]["rows"])
    print("%-22s %5s %9s %9s %9s %9s %9s %9s" % ("kernel", "ctas", "start", "first_go", "last_go", "first_end", "end", "gap_prev"))
    prev_end = None
    tot = {}
    for l in launches[:12] + launches[-6:]:
        a = np.array(l["rows"], dtype=np.int64)
        t0, t1, t2, t3 = a[:, 2], a[:, 3], a[:, 4], a[:, 5]
        gap = (t0.min() - prev_end) if prev_end is not None else 0
        print("%-22s %5d %9.2f %9.2f %9.2f %9.2f %9.2f %9.2f" % (name(l["tag"]), len(a), (t0.min() - t_base) / 1e3, (t1.min() - t_base) / 1e3,
              (t1.max() - t_base) / 1e3, (t3.min() - t_base) / 1e3, (t3.max() - t_base) / 1e3, gap / 1e3))
        prev_end = t3.max()
    # aggregate over the step
    prev_end = None
    for l in launches:
        a = np.array(l["rows"], dtype=np.int64)
        k = name(l["tag"])
        d = tot.setdefault(k, {"n": 0, "span": 0.0, "busy": 0.0, "wait": 0.0, "overlap": 0.0})
        d["n"] += 1
        d["span"] += (a[:, 5].max() - a[:, 2].min()) / 1e3           # first CTA start -> last CTA end
        d["busy"] += (a[:, 5] - a[:, 3]).mean() / 1e3                # mean CTA time after the dependency wait
        d["wait"] += (a[:, 3] - a[:, 2]).mean() / 1e3                # mean time parked in griddepcontrol.wait
        if prev_end is not None:
            d["overlap"] += max(0, prev_end - a[:, 2].min()) / 1e3   # started before the previous kernel ended
        prev_end = a[:, 5].max()
    att = np.array([row for l in launches if l["tag"] == 1 for row in l["rows"]], dtype=np.int64)
    if len(att):
        print("\nattention CTA phases (us, mean / max): start->prologue done %.2f / %.2f, loop %.2f / %.2f, merge+cluster %.2f / %.2f"
              % ((att[:, 3] - att[:, 2]).mean() / 1e3, (att[:, 3] - att[:, 2]).max() / 1e3, (att[:, 4] - att[:, 3]).mean() / 1e3,
                 (att[:, 4] - att[:, 3]).max() / 1e3, (att[:, 5] - att[:, 4]).mean() / 1e3, (att[:, 5] - att[:, 4]).max() / 1e3))
    step = (max(int(x[5]) for x in launches[-1]["rows"]) - t_base) / 1e3
    print("\nstep (first GEMV start -> lm_head end): %.1f us" % step)
    print("%-22s %4s %10s %10s %10s %10s" % ("kernel", "n", "span_us", "busy_us", "wait_us", "early_us"))
    for k, d in tot.items():
        print("%-22s %4d %10.1f %10.1f %10.1f %10.1f" % (k, d["n"], d["span"], d["busy"], d["wait"], d["overlap"]))


if __name__ == "__main__":
    main()
