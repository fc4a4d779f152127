"""Sanitizer pass over the engine's HOST code (scheduler thread, page allocator, C-ABI locking) without a GPU.

    python tools/sanitize_engine_host.py thread     # ThreadSanitizer
    python tools/sanitize_engine_host.py address    # AddressSanitizer + UBSan

Builds libllmlb_b200.so from the product sources with the host compiler's -fsanitize=<kind> (device code unchanged), then
runs the scenarios of tests/test_engine_host_logic_cpu.py against it over tests/support/fake_cudart.cpp (a test double of
libcudart: host memory, no-op launches).  Python itself is not instrumented, so the sanitizer runtime is preloaded ahead of
the fake runtime.  Output: the pytest tail and every sanitizer report found in the log; exit status 1 if there was one."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from llmlb_b200 import build as B  # noqa: E402


def main():
    kind = sys.argv[1] if len(sys.argv) > 1 else "thread"
    sans = {"thread": ["-fsanitize=thread"], "address": ["-fsanitize=address", "-fsanitize=undefined"]}[kind]
    host = [x for f in sans + ["-fno-omit-frame-pointer"] for x in ("-Xcompiler", f)]          # nvcc splits -Xcompiler arguments at commas
    out = os.path.join(ROOT, "tests", "support", "_build", "san_" + kind)
    os.makedirs(out, exist_ok=True)
    flags = [f for f in B.FLAGS if f not in ("-Xptxas", "-v")] + ["-g", *host]

    def comp(src):
        obj = os.path.join(out, src.replace(".cu", ".o"))
        path = os.path.join(B.CSRC, src)
        deps = [path] + [os.path.join(B.CSRC, h) for h in os.listdir(B.CSRC) if h.endswith(".cuh")]
        if not os.path.exists(obj) or any(os.path.getmtime(d) > os.path.getmtime(obj) for d in deps):
            subprocess.check_call([B.NVCC, *flags, "-c", path, "-o", obj])
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(comp, B.SOURCES))
    lib = os.path.join(out, "libllmlb_b200.so")
    subprocess.check_call([B.NVCC, "-shared", "-o", lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a", *host, "-lcudart", "-lpthread"])
    # the HTTP shim over the same library, same sanitizer
    hd = os.path.join(ROOT, "llmlb_b200", "host")
    server = os.path.join(out, "llmlb_b200_server")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", *sans, "-fno-omit-frame-pointer", "-pthread",
                           *[os.path.join(hd, f) for f in ("server.cpp", "gateway.cpp", "tokenizer.cpp", "anthropic.cpp", "checkpoint.cpp", "download.cpp")],
                           "-o", server, "-L" + out, "-lllmlb_b200", "-Wl,-rpath," + out, "-Wl,-rpath,/usr/local/cuda/lib64"])
    import test_engine_host_logic_cpu as T
    fake = T.build_fake()
    for stale in ("server_stderr.log",):
        if os.path.exists(os.path.join(out, stale)):
            os.remove(os.path.join(out, stale))
    rt = subprocess.check_output(["gcc", "-print-file-name=" + ("libtsan.so" if kind == "thread" else "libasan.so")], text=True).strip()
    env = dict(os.environ, LD_PRELOAD=rt + ":" + fake, LLMLB_FAKE_CUDART="1", LLMLB_HOST_LOGIC_LIB=lib,
               TSAN_OPTIONS="halt_on_error=0 second_deadlock_stack=1 history_size=4", ASAN_OPTIONS="detect_leaks=0:abort_on_error=0",
               UBSAN_OPTIONS="print_stacktrace=1")
    log = os.path.join(out, "run.log")
    with open(log, "w") as f:
        # -s: sanitizer reports are written to fd 2; under pytest's capture they would go to a temp file and vanish with _exit(1)
        r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_engine_host_logic_cpu.py"), "-q", "-s", "-p", "no:cacheprovider",
                            "-k", "scenario and not slowstep"], stdout=f, stderr=subprocess.STDOUT, env=env, cwd=ROOT, timeout=3000)
        r1 = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_engine_host_logic_cpu.py"), "-q", "-s", "-p", "no:cacheprovider",
                             "-k", "slowstep"], stdout=f, stderr=subprocess.STDOUT, env=dict(env, FAKE_CUDART_STEP_US="2000"), cwd=ROOT, timeout=3000)
        r.returncode = r.returncode or r1.returncode
    with open(log, "a") as f:        # the server is instrumented itself: only the fake runtime is preloaded (by the test module)
        r2 = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_server_real_engine_cpu.py"), "-q", "-s", "-p", "no:cacheprovider"],
                            stdout=f, stderr=subprocess.STDOUT, cwd=ROOT, timeout=3000,
                            env=dict(os.environ, LLMLB_SERVER_BIN=server, LLMLB_SERVER_STDERR=os.path.join(out, "server_stderr.log"),
                                     LLMLB_SERVER_PRELOAD_FIRST=rt if kind == "address" else "",       # ASan insists on being first in the list
                                     TSAN_OPTIONS=env["TSAN_OPTIONS"], ASAN_OPTIONS=env["ASAN_OPTIONS"], UBSAN_OPTIONS=env["UBSAN_OPTIONS"]))
    r.returncode = r.returncode or r2.returncode
    text = open(log).read() + (open(os.path.join(out, "server_stderr.log")).read() if os.path.exists(os.path.join(out, "server_stderr.log")) else "")
    reports = text.count("WARNING: ThreadSanitizer") + text.count("ERROR: AddressSanitizer") + text.count("runtime error:")
    print("\n".join(text.strip().splitlines()[-6:]))
    print("%s: pytest rc=%d, sanitizer reports: %d (log: %s)" % (kind, r.returncode, reports, log))
    sys.exit(1 if (r.returncode or reports) else 0)


if __name__ == "__main__":
    main()
