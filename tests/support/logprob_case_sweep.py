"""Launches llmlb_op_logprobs over the fake CUDA runtime (LD_PRELOAD, FAKE_CUDART_LAUNCH_LOG set) for each (rows, vocab)
case of the GPU op test (tests/test_logprobs_gpu.py), one "### logprob R V" mark before each, so that
tests/test_logprobs_cpu.py can check which vocabularies the GPU cases launch logprob_kernel with.
usage: logprob_case_sweep.py R:V [R:V ...]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from llmlb_b200 import ffi  # noqa: E402

LOG = os.environ["FAKE_CUDART_LAUNCH_LOG"]
L = ffi.lib()
cudart = C.CDLL("libcudart.so.12")
buf = C.c_void_p()
assert cudart.cudaMalloc(C.byref(buf), C.c_size_t(1 << 20)) == 0
for case in sys.argv[1:]:
    R, V = (int(x) for x in case.split(":"))
    with open(LOG, "a") as f:
        f.write("### logprob %d %d\n" % (R, V))
    ffi.check(L.llmlb_op_logprobs(buf, R, V, buf, buf, buf, None))
