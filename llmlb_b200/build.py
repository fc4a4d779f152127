"""Builds libllmlb_b200.so (CUDA kernels + engine + C ABI) in-tree with nvcc for sm_90a (H100).

No torch involvement: the library links only against the CUDA runtime.  The .so lands next to
this file so that it travels with the repo snapshot to the GPU box.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libllmlb_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SOURCES = ["elementwise.cu", "gemv.cu", "gemv_ks.cu", "gemm_tc.cu", "gemm_tc2.cu", "attention.cu", "attention_tc.cu",
           "sampling.cu", "penalty.cu", "logprob.cu", "tp_exchange.cu", "kv_fork.cu", "engine.cu"]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest(path):
    h = hashlib.sha256()
    for dep in [path, os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "tc_common.cuh"), os.path.join(CSRC, "tp_common.cuh"),
                os.path.join(CSRC, "wgmma.cuh"),
                os.path.join(HERE, "..", "include", "llmlb_b200.h"), __file__]:
        with open(dep, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _compile(src):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    stamp = obj + ".sha"
    dig = _digest(path)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False, ""
    cmd = [NVCC, *FLAGS, "-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    with open(stamp, "w") as f:
        f.write(dig)
    with open(obj + ".ptxas.log", "w") as f:
        f.write(r.stderr)
    return obj, True, r.stderr


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(_compile, SOURCES))
    objs = [o for o, _, _ in results]
    changed = any(c for _, c, _ in results)
    if changed or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
               "-lcudart", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    if verbose:
        for _, c, log in results:
            if c:
                sys.stderr.write(log)
    return LIB


HOST_LIB = os.path.join(HERE, "libllmlb_host.so")
SERVER = os.path.join(HERE, "llmlb_b200_server")


def _newer(target, deps):
    return (not os.path.exists(target)) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def build_host():
    """Gateway-side C++ (no CUDA): libllmlb_host.so, plus the HTTP shim linked to the engine."""
    hd = os.path.join(HERE, "host")
    deps = [os.path.join(hd, f) for f in ("gateway.cpp", "gateway.hpp", "json.hpp", "tokenizer.cpp", "tokenizer.hpp",
                                          "unicode_tables.inc", "anthropic.cpp", "anthropic.hpp", "checkpoint.cpp", "checkpoint.hpp",
                                          "download.cpp", "download.hpp")]
    deps += [os.path.join(HERE, "..", "include", h) for h in ("llmlb_host.h", "llmlb_gateway.h")]
    if _newer(HOST_LIB, deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-pthread",
                               os.path.join(hd, "gateway.cpp"), os.path.join(hd, "tokenizer.cpp"),
                               os.path.join(hd, "anthropic.cpp"), os.path.join(hd, "checkpoint.cpp"), os.path.join(hd, "download.cpp"),
                               "-o", HOST_LIB])
    sdeps = deps + [os.path.join(hd, "server.cpp"), LIB, os.path.join(HERE, "..", "include", "llmlb_b200.h")]
    if os.path.exists(LIB) and _newer(SERVER, sdeps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", os.path.join(hd, "server.cpp"),
                               os.path.join(hd, "gateway.cpp"), os.path.join(hd, "tokenizer.cpp"),
                               os.path.join(hd, "anthropic.cpp"), os.path.join(hd, "checkpoint.cpp"), os.path.join(hd, "download.cpp"),
                               "-o", SERVER,
                               "-L" + HERE, "-lllmlb_b200",
                               "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + "/usr/local/cuda/lib64"])
    return HOST_LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
    print(build_host())
