"""OpenAI logprobs through the HTTP shim (llmlb_b200/host/server.cpp) on the chat and completions routes, against the
scripted engine of tests/support/fake_engine_logprobs.cpp (its records are exact binary fractions the test restates):
every refusal is a 400 invalid_request_error; both response shapes carry OpenAI's field names and the engine's values;
streamed entries, concatenated, equal the non-streamed list of the same seeded request, also with a stop string and with
UTF-8 split over tokens; stop-id tokens are not listed; a server linked to an engine without the entry points refuses
logprob requests; and a request without logprobs gives the same bytes as the shim before logprobs existed (built from
the git history when it is there)."""
import json
import os
import re
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_server_fake_engine_cpu as F  # noqa: E402

T = F.T
VOCAB = 2048   # --model tiny
LP_DIR = os.path.join(F.BUILD, "logprobs")
HOST_SRCS = ("server.cpp", "gateway.cpp", "tokenizer.cpp", "anthropic.cpp", "checkpoint.cpp", "download.cpp")
TOKENIZER = os.path.join(HERE, "golden", "tokenizer_llama3_style.json")


@pytest.fixture(scope="module")
def built_lib():
    return None


def _build(out_dir, engine_src, host_dir):
    """libllmlb_b200.so from a scripted engine source and the server from host_dir's sources, in out_dir."""
    os.makedirs(out_dir, exist_ok=True)
    lib, binary = os.path.join(out_dir, "libllmlb_b200.so"), os.path.join(out_dir, "llmlb_b200_server")
    srcs = [os.path.join(host_dir, f) for f in HOST_SRCS]
    fake_srcs = [os.path.join(HERE, "support", f) for f in ("fake_engine_logprobs.cpp", "fake_engine_penalties.cpp", "fake_engine.cpp")]
    hdr = os.path.join(ROOT, "include", "llmlb_b200.h")
    if F._newer(lib, fake_srcs + [hdr]):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wall", "-pthread", engine_src, "-o", lib])
    deps = srcs + [lib, hdr] + [os.path.join(host_dir, f) for f in os.listdir(host_dir) if f.endswith((".hpp", ".inc"))]
    if F._newer(binary, deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-pthread", "-I" + host_dir, *srcs, "-o", binary,
                               "-L" + out_dir, "-lllmlb_b200", "-Wl,-rpath," + out_dir])
    return lib, binary


def _serve(binary, tokenizer=False):
    args = ["--model", "tiny", "--model-id", "tiny-llama", "--max-seqs", "8", "--max-ctx", "512"]
    if tokenizer:
        args += ["--vocab", "3072", "--tokenizer", TOKENIZER]
    return F._start(binary, *args)


def _fixture(binary, tokenizer=False):
    port, proc = _serve(binary, tokenizer)
    yield port
    proc.terminate()
    proc.wait(timeout=20)


@pytest.fixture(scope="module")
def lp_bin():
    lib, binary = _build(LP_DIR, os.path.join(HERE, "support", "fake_engine_logprobs.cpp"), os.path.join(ROOT, "llmlb_b200", "host"))
    syms = subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    assert "llmlb_request_submit_logprobs" in syms and "llmlb_request_poll_logprobs" in syms
    return binary


@pytest.fixture(scope="module")
def server(lp_bin):
    yield from _fixture(lp_bin)


@pytest.fixture(scope="module")
def tok_server(lp_bin):
    yield from _fixture(lp_bin, tokenizer=True)


@pytest.fixture(scope="module")
def old_engine_server():
    """The server linked to the scripted engine with penalties but without the logprob entry points."""
    lib, binary = _build(os.path.join(LP_DIR, "no_entry"), os.path.join(HERE, "support", "fake_engine_penalties.cpp"),
                         os.path.join(ROOT, "llmlb_b200", "host"))
    assert "llmlb_request_poll_logprobs" not in subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    yield from _fixture(binary)


def _body(route, **kw):
    if route == "/v1/chat/completions":
        b = {"model": "tiny-llama", "messages": [{"role": "user", "content": "hello there"}], "max_tokens": 8, "temperature": 0}
    else:
        b = {"model": "tiny-llama", "prompt": "hello there", "max_tokens": 8, "temperature": 0}
    b.update(kw)
    return b


def _post(port, route, **kw):
    st, _, data = T.call(port, "POST", route, _body(route, **kw))
    return st, json.loads(data)


def _stream(port, route, **kw):
    st, _, data = T.call(port, "POST", route, _body(route, stream=True, **kw))
    assert st == 200, data
    chunks = [json.loads(l[6:]) for l in data.decode().split("\n") if l.startswith("data: ") and l != "data: [DONE]"]
    return chunks, data


CHAT, COMP = "/v1/chat/completions", "/v1/completions"
BAD = [
    (CHAT, dict(logprobs="yes")), (CHAT, dict(logprobs=1)), (CHAT, dict(logprobs=[True])),
    (CHAT, dict(logprobs=True, top_logprobs=21)), (CHAT, dict(logprobs=True, top_logprobs=-1)),
    (CHAT, dict(logprobs=True, top_logprobs=2.5)), (CHAT, dict(logprobs=True, top_logprobs="3")),
    (CHAT, dict(logprobs=True, top_logprobs=True)), (CHAT, dict(top_logprobs=3)), (CHAT, dict(logprobs=False, top_logprobs=0)),
    (CHAT, dict(logprobs=None, top_logprobs=2)),
    (COMP, dict(logprobs=True)), (COMP, dict(logprobs=6)), (COMP, dict(logprobs=-1)), (COMP, dict(logprobs=2.5)),
    (COMP, dict(logprobs="2")), (COMP, dict(logprobs=[1])), (COMP, dict(logprobs=1, echo=True)), (COMP, dict(logprobs=0, echo=True)),
]


@pytest.mark.parametrize("bad", range(len(BAD)))
def test_malformed_or_out_of_range_logprobs_are_400(server, bad):
    route, kw = BAD[bad]
    st, body = _post(server, route, **kw)
    assert st == 400, (kw, body)
    assert body["error"]["type"] == "invalid_request_error"
    assert any(k in body["error"]["message"] for k in ("logprobs", "top_logprobs", "echo")), body


def _want_record(t, n):
    lp = -(1 + t % 7) / 4
    return lp, [((t + 7 * j) % VOCAB, lp - j) for j in range(n)]


def _placeholder(t):
    """byte_detokenize of the server without a tokenizer: printable ASCII bytes as themselves, anything else <|id|>"""
    c = t - 3
    return chr(c) if 3 <= t < 259 and c < 0x80 and (c >= 0x20 or c in (9, 10)) else "<|%d|>" % t


def test_chat_body_shape_and_values(server):
    st, body = _post(server, CHAT, prompt_token_ids=[5, 6, 7], ignore_eos=True, logprobs=True, top_logprobs=3)
    assert st == 200, body
    ch = body["choices"][0]
    assert list(ch) == ["index", "message", "logprobs", "finish_reason"]
    assert ch["logprobs"]["refusal"] is None and list(ch["logprobs"]) == ["content", "refusal"]
    content = ch["logprobs"]["content"]
    assert len(content) == 8 and "".join(e["token"] for e in content) == ch["message"]["content"]
    for e in content:
        assert list(e) == ["token", "logprob", "bytes", "top_logprobs"]
        assert e["bytes"] == list(e["token"].encode())
        t = next(i for i in range(VOCAB) if _placeholder(i) == e["token"])
        lp, top = _want_record(t, 3)
        assert e["logprob"] == lp
        assert [(a["token"], a["logprob"]) for a in e["top_logprobs"]] == [(_placeholder(i), v) for i, v in top]
        assert all(list(a) == ["token", "logprob", "bytes"] for a in e["top_logprobs"])
    # logprobs: true without top_logprobs lists no alternatives
    st, body = _post(server, CHAT, prompt_token_ids=[5, 6, 7], ignore_eos=True, logprobs=True)
    assert all(e["top_logprobs"] == [] for e in body["choices"][0]["logprobs"]["content"])


def test_completions_body_shape_and_values(server):
    st, body = _post(server, COMP, prompt_token_ids=[5, 6, 7], ignore_eos=True, logprobs=2)
    assert st == 200, body
    ch = body["choices"][0]
    assert list(ch) == ["index", "text", "logprobs", "finish_reason"]
    lpj = ch["logprobs"]
    assert list(lpj) == ["tokens", "token_logprobs", "top_logprobs", "text_offset"]
    assert len(lpj["tokens"]) == 8 and "".join(lpj["tokens"]) == ch["text"]
    off = 0
    for tok, v, top, o in zip(lpj["tokens"], lpj["token_logprobs"], lpj["top_logprobs"], lpj["text_offset"]):
        t = next(i for i in range(VOCAB) if _placeholder(i) == tok)
        lp, alts = _want_record(t, 2)
        assert v == lp and o == off
        assert top == {_placeholder(i): a for i, a in alts}
        off += len(tok)
    st, body = _post(server, COMP, prompt_token_ids=[5, 6, 7], ignore_eos=True, logprobs=0)
    assert all(t == {} for t in body["choices"][0]["logprobs"]["top_logprobs"])


def _stream_entries(chunks, route):
    out = []
    for c in chunks:
        if not c.get("choices"):
            continue
        lp = c["choices"][0].get("logprobs")
        if lp is None:
            continue
        if route == CHAT:
            out += lp["content"]
        else:
            out += [list(x) for x in zip(lp["tokens"], lp["token_logprobs"], lp["top_logprobs"], lp["text_offset"])]
    return out


def _body_entries(body, route):
    lp = body["choices"][0]["logprobs"]
    if route == CHAT:
        return lp["content"]
    return [list(x) for x in zip(lp["tokens"], lp["token_logprobs"], lp["top_logprobs"], lp["text_offset"])]


def _text_of(body, route):
    ch = body["choices"][0]
    return ch["message"]["content"] if route == CHAT else ch["text"]


def _stream_text(chunks, route):
    key = "delta" if route == CHAT else None
    return "".join((c["choices"][0]["delta"].get("content") or "") if key else c["choices"][0]["text"] for c in chunks if c.get("choices"))


CASES = [dict(max_tokens=24, ignore_eos=True), dict(max_tokens=40, stop=None), dict(max_tokens=40, ignore_eos=True, seed=3, temperature=0.8)]


@pytest.mark.parametrize("tok", [False, True])
@pytest.mark.parametrize("route", [CHAT, COMP])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_streamed_entries_concatenate_to_the_body_list(server, tok_server, route, tok, case):
    port = tok_server if tok else server
    kw = dict(CASES[case], prompt_token_ids=[9, 8, 7, 6])
    kw.update(dict(logprobs=True, top_logprobs=4) if route == CHAT else dict(logprobs=4))
    if kw.get("stop", 0) is None:           # a stop string: a piece of the unstopped text, so that the match happens
        st, full = _post(port, route, **dict(kw, stop=None))
        text = _text_of(full, route)
        kw["stop"] = text[len(text) // 2: len(text) // 2 + 2] if len(text) > 4 else "zz"
    st, body = _post(port, route, **kw)
    assert st == 200, body
    chunks, raw = _stream(port, route, **kw)
    entries = _body_entries(body, route)
    assert entries and _stream_entries(chunks, route) == entries
    assert _stream_text(chunks, route) == _text_of(body, route)
    if route == CHAT and not tok:   # token texts add up to the text, which a stop string may cut short
        joined = "".join(e["token"] for e in entries)
        assert joined.startswith(_text_of(body, route)) and (kw.get("stop") or joined == _text_of(body, route))
    elif route == COMP:               # text_offset counts the code points released before each token
        text = _text_of(body, route)
        assert all(0 <= e[3] <= len(text) for e in entries) and [e[3] for e in entries] == sorted(e[3] for e in entries)


def test_split_utf8_and_stop_ids_with_a_tokenizer(tok_server):
    """Byte-level tokens split characters: a held-back piece still streams its entries (with empty text); the bytes of
    every entry are the token's raw bytes.  A stop id (<|eot_id|> and the like) ends generation without an entry."""
    seen_split = seen_stop = False
    for seed in range(40):
        kw = dict(prompt_token_ids=[100 + seed, 7, 9], max_tokens=30, temperature=0.9, seed=seed, logprobs=True, top_logprobs=2)
        st, body = _post(tok_server, CHAT, **kw)
        assert st == 200, body
        content = body["choices"][0]["logprobs"]["content"]
        chunks, _ = _stream(tok_server, CHAT, **kw)
        assert _stream_entries(chunks, CHAT) == content
        for e in content:
            assert bytes(e["bytes"]).decode("utf-8", "replace") == e["token"]
            if len(e["bytes"]) == 1 and e["bytes"][0] >= 0x80:
                seen_split = True
        for c in chunks:
            d = c["choices"][0] if c.get("choices") else None
            if d and d.get("logprobs") and d["delta"].get("content") == "":
                seen_split = True
        fin = body["choices"][0]["finish_reason"]
        n_out = body["usage"]["completion_tokens"]
        if fin == "stop":
            seen_stop = True
            assert len(content) == n_out - 1               # the stop id is not listed
        else:
            assert len(content) == n_out
    assert seen_split and seen_stop


def test_a_server_on_an_engine_without_logprobs_refuses_logprob_requests(old_engine_server):
    for route, kw in ((CHAT, dict(logprobs=True)), (CHAT, dict(logprobs=True, top_logprobs=2)), (COMP, dict(logprobs=0))):
        st, body = _post(old_engine_server, route, **kw)
        assert st == 400 and "not supported" in body["error"]["message"], body
    for route, kw in ((CHAT, {}), (CHAT, dict(logprobs=False)), (CHAT, dict(logprobs=None, top_logprobs=None)), (COMP, dict(logprobs=None))):
        assert _post(old_engine_server, route, **kw)[0] == 200


def _normalise(data):
    return re.sub(rb'"created":\d+', b'"created":0', re.sub(rb'"(chatcmpl|cmpl)-\d+"', rb'"\1-0"', data))


def _parent_host_dir(tmp_root):
    """The host sources of the last commit before the shim served logprobs, from git; None without the history."""
    try:
        intro = subprocess.run(["git", "-C", ROOT, "log", "-n1", "--format=%H", "-S", "llmlb_request_poll_logprobs", "--",
                                "llmlb_b200/host/server.cpp"], capture_output=True, text=True, timeout=30)
        if intro.returncode != 0:
            return None
        rev = intro.stdout.strip() + "~1" if intro.stdout.strip() else "HEAD"
        d = os.path.join(tmp_root, "parent", "llmlb_b200", "host")   # the sources include "../../include/..."
        for sub in ("llmlb_b200/host", "include"):
            os.makedirs(os.path.join(tmp_root, "parent", sub), exist_ok=True)
            for f in os.listdir(os.path.join(ROOT, sub)):
                r = subprocess.run(["git", "-C", ROOT, "show", "%s:%s/%s" % (rev, sub, f)], capture_output=True, timeout=30)
                if r.returncode == 0:
                    open(os.path.join(tmp_root, "parent", sub, f), "wb").write(r.stdout)
        src = open(os.path.join(d, "server.cpp")).read() if os.path.exists(os.path.join(d, "server.cpp")) else ""
        return d if src and "llmlb_request_poll_logprobs" not in src else None
    except (OSError, subprocess.SubprocessError):
        return None


def test_requests_without_logprobs_give_the_bytes_of_the_shim_before_logprobs(server, tmp_path):
    d = _parent_host_dir(str(tmp_path))
    if d is None:
        pytest.skip("no git history to build the earlier shim from")
    _, binary = _build(str(tmp_path / "parent_bin"), os.path.join(HERE, "support", "fake_engine_logprobs.cpp"), d)
    port, proc = _serve(binary)
    try:
        for route in (CHAT, COMP):
            for kw in (dict(ignore_eos=True), dict(stream=True, ignore_eos=True), dict(stream=True, stream_options={"include_usage": True}),
                       dict(stop=["e"], max_tokens=20), dict(logprobs=None) if route == COMP else dict(logprobs=False)):
                body = _body(route, prompt_token_ids=[5, 6, 7], **kw)
                new = T.call(server, "POST", route, body)
                old = T.call(port, "POST", route, body)
                assert new[0] == old[0] == 200
                assert _normalise(new[2]) == _normalise(old[2]), (route, kw)
                assert b'"logprobs":{' not in new[2]
    finally:
        proc.terminate()
        proc.wait(timeout=20)
