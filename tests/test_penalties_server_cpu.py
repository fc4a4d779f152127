"""frequency_penalty, presence_penalty and logit_bias through the HTTP shim (llmlb_b200/host/server.cpp) on the chat and
completions routes, against the scripted engine of tests/support/fake_engine_penalties.cpp (a +100 bias forces its token
there, as greedy decoding would): every refusal is a 400 invalid_request_error, null means the default, a forcing bias
reaches the engine, and a server linked to the scripted engine without the entry point (tests/support/fake_engine.cpp, an
engine library that predates it) refuses penalised requests."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_server_fake_engine_cpu as F  # noqa: E402
from test_server_fake_engine_cpu import fake_bin  # noqa: E402,F401  (fixture: the server on the engine without the entry point)

T = F.T
VOCAB = 2048   # --model tiny
PEN_DIR = os.path.join(F.BUILD, "penalties")


@pytest.fixture(scope="module")
def built_lib():
    return None


def _serve(binary):
    port, proc = F._start(binary, "--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8", "--max-ctx", "512")
    return port, proc


@pytest.fixture(scope="module")
def server():
    """The server linked to the scripted engine with llmlb_request_submit_penalized."""
    os.makedirs(PEN_DIR, exist_ok=True)
    hd = os.path.join(ROOT, "llmlb_b200", "host")
    lib, binary = os.path.join(PEN_DIR, "libllmlb_b200.so"), os.path.join(PEN_DIR, "llmlb_b200_server")
    srcs = [os.path.join(hd, f) for f in ("server.cpp", "gateway.cpp", "tokenizer.cpp", "anthropic.cpp", "checkpoint.cpp", "download.cpp")]
    fake_srcs = [os.path.join(HERE, "support", f) for f in ("fake_engine_penalties.cpp", "fake_engine.cpp")]
    hdr = os.path.join(ROOT, "include", "llmlb_b200.h")
    if F._newer(lib, fake_srcs + [hdr]):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wall", "-pthread", fake_srcs[0], "-o", lib])
    deps = srcs + [lib, hdr] + [os.path.join(hd, f) for f in os.listdir(hd) if f.endswith((".hpp", ".inc"))]
    if F._newer(binary, deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-pthread", *srcs, "-o", binary, "-L" + PEN_DIR, "-lllmlb_b200",
                               "-Wl,-rpath," + PEN_DIR])
    assert "llmlb_request_submit_penalized" in subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    port, proc = _serve(binary)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


@pytest.fixture(scope="module")
def old_engine_server(fake_bin):
    """The server linked to the scripted engine without the entry point, as tests/test_server_fake_engine_cpu.py builds it."""
    assert "llmlb_request_submit_penalized" not in subprocess.check_output(["nm", "-D", "--defined-only", F.FAKE_LIB], text=True)
    port, proc = _serve(fake_bin)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


def _body(route, **kw):
    if route == "/v1/chat/completions":
        b = {"model": "tiny-llama", "messages": [{"role": "user", "content": "hello there"}], "max_tokens": 6, "temperature": 0}
    else:
        b = {"model": "tiny-llama", "prompt": "hello there", "max_tokens": 6, "temperature": 0}
    b.update(kw)
    return b


def _post(port, route, **kw):
    st, _, data = T.call(port, "POST", route, _body(route, **kw))
    return st, json.loads(data)


def _text(port, route, **kw):
    """the generated text of a request on a fixed token prompt, ignore_eos so that it runs max_tokens long"""
    st, body = _post(port, route, prompt_token_ids=[5, 6, 7], ignore_eos=True, **kw)
    assert st == 200, body
    assert body["usage"]["completion_tokens"] == kw.get("max_tokens", 6)
    return body["choices"][0]["message"]["content"] if route == "/v1/chat/completions" else body["choices"][0]["text"]


ROUTES = ["/v1/chat/completions", "/v1/completions"]
BAD = [
    dict(frequency_penalty="0.5"), dict(frequency_penalty=2.5), dict(frequency_penalty=-2.01), dict(presence_penalty=True),
    dict(presence_penalty=3), dict(presence_penalty=[1]), dict(logit_bias=[1, 2]), dict(logit_bias="x"),
    dict(logit_bias={"abc": 1}), dict(logit_bias={"-1": 1}), dict(logit_bias={"1.5": 1}), dict(logit_bias={" 1": 1}),
    dict(logit_bias={str(VOCAB): 1}), dict(logit_bias={"99999999999": 1}), dict(logit_bias={"3": 100.5}),
    dict(logit_bias={"3": -101}), dict(logit_bias={"3": "1"}), dict(logit_bias={"3": None}), dict(logit_bias={"3": 1, "03": 2}),
    dict(logit_bias={str(i): 1 for i in range(1025)}),
]


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("bad", range(len(BAD)))
def test_out_of_range_or_malformed_penalties_are_400(server, route, bad):
    st, body = _post(server, route, **BAD[bad])
    assert st == 400, (BAD[bad], body)
    assert body["error"]["type"] == "invalid_request_error"
    assert any(k in body["error"]["message"] for k in ("frequency_penalty", "presence_penalty", "logit_bias")), body


@pytest.mark.parametrize("route", ROUTES)
def test_null_penalties_are_the_defaults(server, route):
    assert _text(server, route, frequency_penalty=None, presence_penalty=None, logit_bias=None) == _text(server, route)
    # neutral values and limits are accepted
    for kw in (dict(frequency_penalty=0, presence_penalty=0.0, logit_bias={}), dict(frequency_penalty=2, presence_penalty=-2),
               dict(logit_bias={str(i): (100 if i % 2 else -100) for i in range(1024)}), dict(logit_bias={"0": 1, str(VOCAB - 1): -1.5})):
        assert _post(server, route, **kw)[0] == 200, kw


@pytest.mark.parametrize("route", ROUTES)
def test_a_forcing_bias_reaches_the_engine(server, route):
    # ids 68 and 69 are the bytes "A" and "B" of the byte-level placeholder tokenizer (id = byte + 3)
    assert _text(server, route, logit_bias={"68": 100}, max_tokens=5) == "AAAAA"
    assert _text(server, route, logit_bias={"69": 100, "68": -100}, max_tokens=5) == "BBBBB"
    assert _text(server, route, max_tokens=5) not in ("AAAAA", "BBBBB")


@pytest.mark.parametrize("route", ROUTES)
def test_a_server_on_an_engine_without_penalties_refuses_penalised_requests(old_engine_server, route):
    for kw in (dict(frequency_penalty=0.5), dict(presence_penalty=-1), dict(logit_bias={"3": 1})):
        st, body = _post(old_engine_server, route, **kw)
        assert st == 400 and "not supported" in body["error"]["message"], body
    # unpenalised requests, and neutral or null penalties, are still served
    for kw in ({}, dict(frequency_penalty=0, presence_penalty=None, logit_bias={})):
        assert _post(old_engine_server, route, **kw)[0] == 200
