"""OpenAI's n through the HTTP shim (llmlb_b200/host/server.cpp) against the scripted engine of
tests/support/fake_engine_choices.cpp, where choice i is the scripted request with seed + i:
- body and stream shapes for n = 1, 2 and 5 on chat and completions, with logprobs, echo, stop and include_usage: n choices
  in index order, each with its own text, finish_reason and logprobs; each stream chunk carries one choice and its index,
  and chat sends a role delta for every index first; every choice's text is the scripted request's with seed + i;
- usage counts the prompt once and sums the choices' completion tokens;
- a stop string ends only the choice whose text reaches it;
- a client that hangs up cancels every choice;
- n outside [1, 128] is a 400 on chat and completions, n above the engine's max_seqs a 400 with the engine's message, any
  n != 1 a 400 on responses (Anthropic's messages have no n: the translation drops it, as before); a server on an engine
  library without llmlb_request_submit_choices refuses n > 1;
- with n absent or 1, every response is byte for byte what the server of the parent commit sends (built from git)."""
import json
import os
import re
import socket
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_logprobs_server_cpu as LS  # noqa: E402

T, F = LS.T, LS.F
CHAT, COMP, RESP, MSG = "/v1/chat/completions", "/v1/completions", "/v1/responses", "/v1/messages"
ARGS = ["--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8", "--max-ctx", "512"]
DIR = os.path.join(LS.LP_DIR, "choices")


@pytest.fixture(scope="module")
def built_lib():
    return None


def _bin(name, engine_src, host_dir=os.path.join(ROOT, "llmlb_b200", "host")):
    return LS._build(os.path.join(DIR, name), os.path.join(HERE, "support", engine_src), host_dir)


@pytest.fixture(scope="module")
def choices_bin():
    lib, binary = _bin("n", "fake_engine_choices.cpp")
    assert "llmlb_request_submit_choices" in subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    return binary


def _server(binary, *extra, env=None):
    port, proc = F._start(binary, *ARGS, *extra, env=env)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


@pytest.fixture(scope="module")
def srv(choices_bin):
    yield from _server(choices_bin)


def _body(route, n=None, stream=False, **kw):
    b = {"model": "tiny-llama", "max_tokens": 6, "temperature": 0.8, "seed": 41, "ignore_eos": True, "stream": stream}
    if route == COMP:
        b["prompt"] = "count: one two three"
    else:
        b["messages"] = [{"role": "user", "content": "count: one two three"}]
    if n is not None:
        b["n"] = n
    if stream:
        b["stream_options"] = {"include_usage": True}
    b.update(kw)
    return b


def _post(port, route, body, headers=None):
    st, _, data = T.call(port, "POST", route, body, headers)
    return st, data


def _events(data):
    return [json.loads(l[6:]) for l in data.decode().split("\n") if l.startswith("data: ") and l != "data: [DONE]"]


def _single(port, route, seed, **kw):
    """the body of the one-choice request with this seed"""
    st, data = _post(port, route, _body(route, seed=seed, **kw))
    assert st == 200, data
    return json.loads(data)


def _text(route, choice):
    return choice["text"] if route == COMP else choice["message"]["content"]


@pytest.mark.parametrize("route", [CHAT, COMP])
@pytest.mark.parametrize("n", [1, 2, 5])
def test_a_body_holds_n_choices_each_the_request_with_seed_plus_i(srv, route, n):
    lp = {"logprobs": True, "top_logprobs": 2} if route == CHAT else {"logprobs": 2, "echo": True}
    st, data = _post(srv, route, _body(route, n, **lp))
    assert st == 200, data
    b = json.loads(data)
    assert [c["index"] for c in b["choices"]] == list(range(n))
    for i, c in enumerate(b["choices"]):
        one = _single(srv, route, 41 + i, **lp)["choices"][0]
        assert c["finish_reason"] == "length" and _text(route, c) == _text(route, one) and c["logprobs"] == one["logprobs"]
        if route == COMP:
            assert c["text"].startswith("count: one two three")
    one_usage = _single(srv, route, 41, **lp)["usage"]
    assert b["usage"]["prompt_tokens"] == one_usage["prompt_tokens"]
    assert b["usage"]["completion_tokens"] == n * 6 and b["usage"]["total_tokens"] == one_usage["prompt_tokens"] + n * 6
    if n > 1:
        assert len({_text(route, c) for c in b["choices"]}) > 1


@pytest.mark.parametrize("route", [CHAT, COMP])
@pytest.mark.parametrize("n", [1, 2, 5])
def test_a_stream_carries_one_choice_per_chunk_with_its_index(srv, route, n):
    lp = {"logprobs": True} if route == CHAT else {"logprobs": 1, "echo": True}
    st, data = _post(srv, route, _body(route, n, stream=True, **lp))
    assert st == 200, data
    evs = _events(data)
    assert data.decode().endswith("data: [DONE]\n\n")
    chunks, usage = [e for e in evs if e["choices"]], [e for e in evs if e.get("usage")]
    assert all(len(e["choices"]) == 1 for e in chunks)
    if route == CHAT:
        assert [e["choices"][0]["index"] for e in chunks[:n]] == list(range(n))
        assert all(e["choices"][0]["delta"] == {"role": "assistant"} for e in chunks[:n])
    texts, finish = {}, {}
    for e in chunks:
        c = e["choices"][0]
        piece = c["text"] if route == COMP else c["delta"].get("content", "")
        texts[c["index"]] = texts.get(c["index"], "") + (piece or "")
        if c["finish_reason"]:
            assert c["index"] not in finish
            finish[c["index"]] = c["finish_reason"]
    assert finish == {i: "length" for i in range(n)}
    st, body = _post(srv, route, _body(route, n, **lp))
    assert [_text(route, c) for c in json.loads(body)["choices"]] == [texts[i] for i in range(n)]
    assert len(usage) == 1 and usage[0]["usage"]["completion_tokens"] == n * 6 and evs[-1] is usage[0]


@pytest.mark.parametrize("route", [CHAT, COMP])
def test_a_stop_string_ends_only_its_own_choice(srv, route):
    base = json.loads(_post(srv, route, _body(route, 2, max_tokens=40))[1])["choices"]
    t0, t1 = _text(route, base[0]), _text(route, base[1])
    stop = next(t0[i:i + 2] for i in range(4, len(t0) - 2) if t0[i:i + 2] not in t1 and t0[i:i + 2].strip())
    b = json.loads(_post(srv, route, _body(route, 2, max_tokens=40, stop=stop))[1])
    c0, c1 = b["choices"]
    assert c0["finish_reason"] == "stop" and _text(route, c0) == t0[:t0.index(stop)]
    assert c1["finish_reason"] == "length" and _text(route, c1) == t1
    assert b["usage"]["completion_tokens"] < 80


def _active(port):
    return json.loads(T.call(port, "GET", "/api/health")[2])["load"]["active_requests"]


def test_a_client_that_hangs_up_cancels_every_choice(choices_bin):
    for port in _server(choices_bin, env={"FAKE_ENGINE_TOKEN_US": "20000"}):
        for stream in (True, False):
            body = json.dumps(_body(CHAT, 4, stream=stream, max_tokens=400)).encode()
            s = socket.create_connection(("127.0.0.1", port))
            s.sendall(b"POST /v1/chat/completions HTTP/1.1\r\nHost: x\r\nContent-Type: application/json\r\nContent-Length: %d\r\n\r\n"
                      % len(body) + body)
            deadline = time.time() + 10
            while _active(port) < 4 and time.time() < deadline:
                time.sleep(0.02)
            assert _active(port) == 4
            s.close()
            deadline = time.time() + 10
            while _active(port) and time.time() < deadline:
                time.sleep(0.05)
            assert _active(port) == 0


@pytest.mark.parametrize("route", [CHAT, COMP])
@pytest.mark.parametrize("n", [0, -1, 129, 1.5, "2", True, [2]])
def test_n_outside_1_to_128_is_refused_on_chat_and_completions(srv, route, n):
    st, data = _post(srv, route, _body(route, n))
    assert st == 400 and "n must be an integer in [1, 128]" in json.loads(data)["error"]["message"], data


@pytest.mark.parametrize("route", [CHAT, COMP])
def test_n_above_the_engines_max_seqs_is_refused_with_its_message(srv, route):
    st, data = _post(srv, route, _body(route, 9))
    assert st == 400 and "n must be in [1, max_seqs = 8]" in json.loads(data)["error"]["message"], data


def test_responses_keep_refusing_n_and_messages_have_none(srv):
    st, data = _post(srv, RESP, {"model": "tiny-llama", "input": "hi", "max_output_tokens": 4, "n": 2})
    assert st == 400 and "n must be 1" in data.decode()
    # Anthropic's Messages API has no n: the request's translation does not carry one, as before, and one message comes back
    st, data = _post(srv, MSG, {"model": "tiny-llama", "max_tokens": 4, "n": 2, "messages": [{"role": "user", "content": "hi"}]},
                     {"anthropic-version": "2023-06-01"})
    assert st == 200 and json.loads(data)["type"] == "message"


def test_an_engine_library_without_choices_refuses_n_above_1(tmp_path):
    lib, binary = _bin("no_entry", "fake_engine_prefix_cache.cpp")
    assert "llmlb_request_submit_choices" not in subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    for port in _server(binary):
        st, data = _post(port, CHAT, _body(CHAT, 2))
        assert st == 400 and "cannot fork a prompt" in data.decode()
        assert _post(port, CHAT, _body(CHAT, 1))[0] == 200


# ---- n absent: the parent commit's bytes --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def parent_bin(tmp_path_factory):
    host = tmp_path_factory.mktemp("parent_host")
    base = subprocess.run(["git", "-C", ROOT, "rev-parse", "HEAD"], capture_output=True, text=True)
    # the commit before the one that added n to the server: the newest commit whose server.cpp has no submit_choices
    revs = subprocess.run(["git", "-C", ROOT, "log", "--format=%H", "-n", "50", "--", "llmlb_b200/host/server.cpp"],
                          capture_output=True, text=True)
    if base.returncode or revs.returncode:
        pytest.skip("no git history")
    rev = None
    for h in revs.stdout.split():
        src = subprocess.run(["git", "-C", ROOT, "show", h + ":llmlb_b200/host/server.cpp"], capture_output=True, text=True).stdout
        if "llmlb_request_submit_choices" not in src:
            rev = h
            break
    if rev is None:
        pytest.skip("no server without n in the history")
    os.makedirs(str(host / "llmlb_b200" / "host"))
    os.makedirs(str(host / "include"))
    for d in ("llmlb_b200/host/", "include/"):
        for f in subprocess.run(["git", "-C", ROOT, "ls-tree", "--name-only", rev, d], capture_output=True, text=True).stdout.split():
            with open(str(host / f), "wb") as out:
                out.write(subprocess.run(["git", "-C", ROOT, "show", rev + ":" + f], capture_output=True).stdout)
    return _bin("parent", "fake_engine_choices.cpp", str(host / "llmlb_b200" / "host"))[1]


def _normalise(data):
    return re.sub(rb'"created":\d+', b'"created":0', data)


def test_without_n_every_response_is_the_parent_servers_byte_for_byte(choices_bin, parent_bin):
    reqs = []
    for route in (CHAT, COMP):
        for stream in (False, True):
            for kw in ({}, {"logprobs": True, "top_logprobs": 3} if route == CHAT else {"logprobs": 3, "echo": True},
                       {"stop": "e"}, {"temperature": 0}):
                reqs.append((route, _body(route, None, stream, **kw)))
                reqs.append((route, _body(route, 1, stream, **kw)))
    reqs.append((RESP, {"model": "tiny-llama", "input": "hi", "max_output_tokens": 5, "seed": 3}))
    got = {}
    for name, binary in (("now", choices_bin), ("parent", parent_bin)):
        for port in _server(binary):
            got[name] = [_normalise(_post(port, route, body)[1]) for route, body in reqs]
    assert got["now"] == got["parent"]
