"""examples/inprocess_host.c against the REAL engine on an H100: a C99 host over the three public headers serving the
gateway's hot path in-process (gate -> TPS router -> lease -> submit/poll -> SSE -> relay accounting -> TPS update), no HTTP.
Checked two ways: the gateway oracle over the client-visible bytes and the router state (as in the CPU test against the
scripted engine), and token-for-token against the Python ctypes host driving the same library with the same prompts.
(File name: runs after the kernel / engine / server suites — it compiles a program first.)"""
import json
import os
import re
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import gateway_ref as G  # noqa: E402

pytestmark = pytest.mark.gpu
MODEL = dict(hidden=512, n_layers=2, n_heads=8, n_kv_heads=2, head_dim=128, ffn=1024, vocab=3072, rope_theta=500000.0, rms_eps=1e-5)   # the program's defaults


def _prompt(index, n, vocab):
    """the xorshift of examples/inprocess_host.c::serve_one"""
    s = (0x9E3779B97F4A7C15 * (index + 1)) & (2 ** 64 - 1)
    out = []
    for _ in range(n):
        s ^= (s << 13) & (2 ** 64 - 1); s ^= s >> 7; s ^= (s << 17) & (2 ** 64 - 1)
        out.append(s % vocab)
    return out


def test_c_host_serves_in_process_and_agrees_with_the_ctypes_host(built_lib, tmp_path):
    from llmlb_b200 import build, ffi
    host = build.build_host()
    exe = str(tmp_path / "inprocess_host")
    d = os.path.dirname(built_lib)
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "inprocess_host.c"),
                           "-L" + d, "-lllmlb_b200", "-lllmlb_host", "-Wl,-rpath," + d, "-Wl,-rpath,/usr/local/cuda/lib64", "-o", exe])
    n_req, n_in, n_out = 3, 40, 24
    r = subprocess.run([exe, "--api", "responses", "--requests", str(n_req), "--prompt-len", str(n_in), "--max-tokens", str(n_out)], capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()[-3000:]
    streams = r.stdout.decode().split("### request ")[1:]
    recs = [json.loads(l) for l in r.stderr.decode().splitlines() if l.startswith("{")]
    per, final = recs[:-1], recs[-1]
    state = G.ModelTpsState()
    got_tokens = []
    for i, (s, rec) in enumerate(zip(streams, per)):
        sse = s.split("\n", 1)[1]
        acc = G.StreamingTokenAccumulator("llama-tiny")
        assert G.process_sse_lines(sse, acc) == "" and acc.done
        assert acc.finalize() == {"input_tokens": n_in, "output_tokens": n_out, "total_tokens": n_in + n_out}
        assert rec["usage"] == [n_in, n_out, n_in + n_out] and rec["finish"] == 2        # LLMLB_FINISH_LENGTH (EOS ignored)
        got_tokens.append([int(x) for x in re.findall(r"<(\d+)> ", acc.accumulated_content)])
        assert len(got_tokens[-1]) == n_out
        state.update_tps(n_out, rec["ms"])
    assert final["request_count"] == n_req and final["stats"][:4] == [0, n_req, n_req, 0] and final["in_flight"] == 0
    assert all(x["ms"] >= 1 for x in per) and final["tps_ema"] == state.tps_ema          # durations are clamped to >= 1 ms (proxy.rs:157)
    # the same requests through the Python host of the same library
    with ffi.Engine(MODEL, model_id="llama-tiny", max_seqs=8, max_ctx=1024, seed=0) as eng:
        for i in range(n_req):
            toks, _ = eng.generate(_prompt(i, n_in, MODEL["vocab"]), n_out, ignore_eos=True)
            assert toks == got_tokens[i], i
