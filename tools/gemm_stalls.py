"""Where the wgmma prefill GEMM's cycles go (debug hook llmlb_debug_trace_*): per kernel type,
the share of CTA lifetime the TMA producer waited for a free smem slot and each of the two consumer
warpgroups waited for data.  Run with LLMLB_GEMM_NO_2CTA=1 (the 1-CTA
kernel is the instrumented one)."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("LLMLB_GEMM_NO_2CTA", "1")
from llmlb_b200 import ffi  # noqa: E402


def main():
    L = ffi.lib()
    L.llmlb_debug_trace_enable.argtypes = [C.c_uint32]
    L.llmlb_debug_trace_dump.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    model = ffi.LLAMA3_8B
    eng = ffi.Engine(model, max_seqs=4, max_ctx=1024)
    prompt = np.random.RandomState(0).randint(0, model["vocab"], 512).tolist()
    eng.generate(prompt, 2, ignore_eos=True)
    cap = 200000
    L.llmlb_debug_trace_enable(cap)
    eng.generate(prompt, 1, ignore_eos=True)
    buf = np.zeros((cap, 6), dtype=np.uint64)
    n = C.c_uint32()
    L.llmlb_debug_trace_dump(buf.ctypes.data, cap, C.byref(n))
    L.llmlb_debug_trace_enable(0)
    eng.close()
    r = buf[: n.value]
    r = r[(r[:, 0] >> np.uint64(60)) == 2]
    names = {0: "store_bf16", 1: "resid_f32", 2: "silu_mul", 3: "store_f32"}
    print("%-34s %6s %10s %9s %9s %9s" % ("kernel", "ctas", "cycles", "prod_wait", "wg1_wait", "wg2_wait"))
    for tag in np.unique(r[:, 0]):
        rows = r[r[:, 0] == tag].astype(np.float64)
        t = int(tag)
        name = "gemm_tc n_out=%d k=%d %s" % ((t >> 32) & 0xFFFFFFF, t & 0xFFFFFFF, names[(t >> 28) & 0xF])
        tot = rows[:, 2]
        print("%-34s %6d %10.0f %8.1f%% %8.1f%% %8.1f%%" % (name, len(rows), tot.mean(), 100 * (rows[:, 3] / tot).mean(),
                                                           100 * (rows[:, 4] / tot).mean(), 100 * (rows[:, 5] / tot).mean()))


if __name__ == "__main__":
    main()
