"""OpenAI's cached_tokens through the HTTP shim (llmlb_b200/host/server.cpp) against the scripted engine of
tests/support/fake_engine_prefix_cache.cpp, which reports 64 * floor((n - 1) / 64) cached tokens for an n-token prompt when
the server sets llmlb_engine_config.prefix_cache: with --prefix-cache, usage carries prompt_tokens_details (chat,
completions) or input_tokens_details (responses), in bodies and in the streams' usage; /v1/messages keeps its shapes;
without the flag no response mentions it; and a server on an engine library without the prefix cache refuses the flag at
start-up."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_logprobs_server_cpu as LS  # noqa: E402

T, F = LS.T, LS.F
CHAT, COMP, RESP, MSG = "/v1/chat/completions", "/v1/completions", "/v1/responses", "/v1/messages"
ARGS = ["--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8", "--max-ctx", "512"]
LONG = "the quick brown fox jumps over the lazy dog; " * 5     # 225 bytes: 225 placeholder tokens


@pytest.fixture(scope="module")
def built_lib():
    return None


@pytest.fixture(scope="module")
def pc_bin():
    lib, binary = LS._build(os.path.join(LS.LP_DIR, "prefix_cache"), os.path.join(HERE, "support", "fake_engine_prefix_cache.cpp"),
                            os.path.join(ROOT, "llmlb_b200", "host"))
    assert "llmlb_request_cached_tokens" in subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    return binary


def _server(binary, *extra):
    port, proc = F._start(binary, *ARGS, *extra)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


@pytest.fixture(scope="module")
def on(pc_bin):
    yield from _server(pc_bin, "--prefix-cache")


@pytest.fixture(scope="module")
def off(pc_bin):
    yield from _server(pc_bin)


def _body(route, stream=False):
    b = {"model": "tiny-llama", "max_tokens": 4, "temperature": 0, "stream": stream}
    if route == COMP:
        b["prompt"] = LONG
    elif route == RESP:
        b = {"model": "tiny-llama", "input": LONG, "max_output_tokens": 4, "temperature": 0, "stream": stream}
    else:
        b["messages"] = [{"role": "user", "content": LONG}]
    if stream and route in (CHAT, COMP):
        b["stream_options"] = {"include_usage": True}
    return b


def _usage(port, route, stream):
    st, _, data = T.call(port, "POST", route, _body(route, stream), {"anthropic-version": "2023-06-01"} if route == MSG else None)
    assert st == 200, data
    if not stream:
        return LS.json.loads(data)["usage"], data
    events = [LS.json.loads(l[6:]) for l in data.decode().split("\n") if l.startswith("data: ") and l != "data: [DONE]"]
    if route == RESP:
        done = [e for e in events if e.get("type") == "response.done"]
        return done[-1]["response"]["usage"], data
    return [e for e in events if e.get("usage")][-1]["usage"], data


def _cached(n):
    return 64 * ((n - 1) // 64)


@pytest.mark.parametrize("stream", [False, True])
@pytest.mark.parametrize("route", [CHAT, COMP])
def test_usage_reports_cached_prompt_tokens(on, route, stream):
    u, _ = _usage(on, route, stream)
    assert u["prompt_tokens"] >= 225 and u["prompt_tokens_details"] == {"cached_tokens": _cached(u["prompt_tokens"])}, u
    assert u["prompt_tokens_details"]["cached_tokens"] > 0
    assert u["total_tokens"] == u["prompt_tokens"] + u["completion_tokens"]


@pytest.mark.parametrize("stream", [False, True])
def test_responses_usage_reports_cached_input_tokens(on, stream):
    u, _ = _usage(on, RESP, stream)
    assert u["input_tokens_details"] == {"cached_tokens": _cached(u["input_tokens"])} and u["input_tokens_details"]["cached_tokens"] > 0, u


@pytest.mark.parametrize("stream", [False, True])
@pytest.mark.parametrize("route", [CHAT, COMP, RESP, MSG])
def test_without_the_flag_and_on_messages_usage_has_no_details(on, off, route, stream):
    for port in ((off, on) if route == MSG else (off,)):
        u, data = _usage(port, route, stream)
        assert b"cached_tokens" not in data and b"_tokens_details" not in data, data
        keys = {"input_tokens", "output_tokens"} if route == MSG else \
               {"input_tokens", "output_tokens", "total_tokens"} if route == RESP else {"prompt_tokens", "completion_tokens", "total_tokens"}
        assert set(u) == keys or (route == MSG and set(u) <= keys | {"cache_creation_input_tokens", "cache_read_input_tokens"}), u


def test_without_the_flag_bytes_match_an_engine_library_without_the_cache(off):
    """The same requests against the server linked to the engine library that predates the prefix cache: the same bytes,
    once the per-request id and creation time are masked."""
    import re
    _, old_bin = LS._build(os.path.join(LS.LP_DIR, "prompt"), os.path.join(HERE, "support", "fake_engine_prompt_logprobs.cpp"),
                           os.path.join(ROOT, "llmlb_b200", "host"))
    gen = _server(old_bin)
    old = next(gen)
    try:
        for route in (CHAT, COMP, RESP):
            for stream in (False, True):
                got = [_usage(p, route, stream)[1] for p in (off, old)]
                mask = [re.sub(rb'"(id|created|created_at)":("[^"]*"|\d+)', b"", g) for g in got]
                assert mask[0] == mask[1], (route, stream)
    finally:
        next(gen, None)


def test_an_engine_library_without_the_cache_refuses_the_flag_at_start_up():
    _, old_bin = LS._build(os.path.join(LS.LP_DIR, "prompt"), os.path.join(HERE, "support", "fake_engine_prompt_logprobs.cpp"),
                           os.path.join(ROOT, "llmlb_b200", "host"))
    r = subprocess.run([old_bin, "--port", "0", *ARGS, "--prefix-cache"], capture_output=True, text=True, timeout=30)
    assert r.returncode == 2 and "--prefix-cache" in r.stderr and "llmlb_request_cached_tokens" in r.stderr, r.stderr
