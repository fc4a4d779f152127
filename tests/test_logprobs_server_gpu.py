"""-m gpu: the HTTP shim serving logprobs from the real engine (LLAMA_TINY, synthetic weights) on the chat and completions
routes: entries for every generated token, greedy tokens at the top of their alternatives, values that are
log-probabilities, and streamed entries that concatenate to the non-streamed list of the same greedy request."""
import json
import math
import os
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_server_gpu as S  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def server(built_lib):
    from llmlb_b200 import build
    build.build_host()
    port = S._free_port()
    proc = subprocess.Popen([S.BIN, "--port", str(port), "--model", "tiny", "--model-id", "tiny-llama",
                             "--max-seqs", "8", "--max-ctx", "512"], stderr=subprocess.PIPE)
    deadline = time.time() + 120
    while time.time() < deadline:
        try:
            st, _, _ = S.call(port, "GET", "/v1/models")
            break
        except OSError:
            assert proc.poll() is None, proc.stderr.read().decode()
            time.sleep(0.2)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


def _post(port, route, body):
    st, _, d = S.call(port, "POST", route, body)
    assert st == 200, d
    return d


def _chunks(d):
    return [json.loads(l[6:]) for l in d.decode().split("\n") if l.startswith("data: ") and l != "data: [DONE]"]


def test_chat_logprobs_from_the_engine(server):
    body = {"model": "tiny-llama", "messages": [{"role": "user", "content": "logprobs please"}], "max_tokens": 12,
            "temperature": 0, "ignore_eos": True, "logprobs": True, "top_logprobs": 5}
    j = json.loads(_post(server, "/v1/chat/completions", body))
    content = j["choices"][0]["logprobs"]["content"]
    assert len(content) == j["usage"]["completion_tokens"] == 12
    for e in content:
        assert len(e["top_logprobs"]) == 5 and e["logprob"] <= 0 and math.isfinite(e["logprob"])
        vals = [a["logprob"] for a in e["top_logprobs"]]
        assert vals == sorted(vals, reverse=True) and sum(math.exp(v) for v in vals) <= 1 + 1e-5
        assert e["logprob"] == vals[0]                     # greedy: the token is (tied with) the most probable
    streamed = []
    for c in _chunks(_post(server, "/v1/chat/completions", dict(body, stream=True))):
        lp = c["choices"][0].get("logprobs") if c.get("choices") else None
        streamed += lp["content"] if lp else []
    assert streamed == content


def test_completions_logprobs_from_the_engine(server):
    body = {"model": "tiny-llama", "prompt": [5, 6, 7, 8], "max_tokens": 10, "temperature": 0, "ignore_eos": True, "logprobs": 3}
    j = json.loads(_post(server, "/v1/completions", body))
    lp = j["choices"][0]["logprobs"]
    assert len(lp["tokens"]) == len(lp["token_logprobs"]) == len(lp["top_logprobs"]) == len(lp["text_offset"]) == 10
    for v, top in zip(lp["token_logprobs"], lp["top_logprobs"]):
        assert v <= 0 and 1 <= len(top) <= 3 and max(top.values()) == v
    assert lp["text_offset"] == sorted(lp["text_offset"]) and lp["text_offset"][0] == 0
    streamed = {"tokens": [], "token_logprobs": [], "top_logprobs": [], "text_offset": []}
    for c in _chunks(_post(server, "/v1/completions", dict(body, stream=True))):
        x = c["choices"][0].get("logprobs") if c.get("choices") else None
        for k in streamed:
            streamed[k] += x[k] if x else []
    assert streamed == lp
