"""OpenAI completions' echo, alone and with logprobs, through the HTTP shim (llmlb_b200/host/server.cpp) against the
scripted engine of tests/support/fake_engine_prompt_logprobs.cpp (its prompt records are exact binary fractions the test
restates): the echoed text in bodies and streams, for string and token-id prompts; the prompt entries first, with a null
first entry, the engine's values and code-point text offsets into the echoed text; streamed entries that concatenate to the
body's list; a string prompt that round-trips through the tokenizer, multi-byte UTF-8 included; and a server on an engine
library without the prompt entry points, which keeps answering echo with logprobs with a 400."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_logprobs_server_cpu as LS  # noqa: E402

T = LS.T
COMP, CHAT = LS.COMP, LS.CHAT
VOCAB = LS.VOCAB


@pytest.fixture(scope="module")
def built_lib():
    return None


@pytest.fixture(scope="module")
def plp_bin():
    lib, binary = LS._build(os.path.join(LS.LP_DIR, "prompt"), os.path.join(HERE, "support", "fake_engine_prompt_logprobs.cpp"),
                            os.path.join(ROOT, "llmlb_b200", "host"))
    syms = subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    assert "llmlb_request_submit_prompt_logprobs" in syms and "llmlb_request_poll_prompt_logprobs" in syms
    return binary


@pytest.fixture(scope="module")
def server(plp_bin):
    yield from LS._fixture(plp_bin)


@pytest.fixture(scope="module")
def tok_server(plp_bin):
    yield from LS._fixture(plp_bin, tokenizer=True)


@pytest.fixture(scope="module")
def old_server():
    """The server linked to the scripted engine with logprobs but without the prompt entry points."""
    _, binary = LS._build(LS.LP_DIR, os.path.join(HERE, "support", "fake_engine_logprobs.cpp"), os.path.join(ROOT, "llmlb_b200", "host"))
    yield from LS._fixture(binary)


def _post(port, **kw):
    return LS._post(port, COMP, **kw)


def _stream(port, **kw):
    return LS._stream(port, COMP, **kw)


def _entries(lp):
    return [list(x) for x in zip(lp["tokens"], lp["token_logprobs"], lp["top_logprobs"], lp["text_offset"])]


def _stream_entries(chunks):
    out = []
    for c in chunks:
        if c.get("choices") and c["choices"][0].get("logprobs") is not None:
            out += _entries(c["choices"][0]["logprobs"])
    return out


def _text(chunks):
    return "".join(c["choices"][0]["text"] for c in chunks if c.get("choices"))


IDS = [40, 70, 75, 76, 79]    # placeholder text "EKHIL"


@pytest.mark.parametrize("prompt", ["string", "ids"])
def test_echo_alone_prepends_the_prompt_text(server, prompt):
    kw = dict(prompt="hello there") if prompt == "string" else dict(prompt=IDS)
    want = "hello there" if prompt == "string" else "".join(LS._placeholder(t) for t in IDS)
    st, plain = _post(server, ignore_eos=True, **kw)
    st2, body = _post(server, ignore_eos=True, echo=True, **kw)
    assert st == st2 == 200
    ch = body["choices"][0]
    assert ch["text"] == want + plain["choices"][0]["text"] and ch.get("logprobs") is None
    assert body["usage"] == plain["usage"]                                         # the prompt counts once
    chunks, _ = _stream(server, ignore_eos=True, echo=True, **kw)
    assert chunks[0]["choices"][0]["text"] == want                                 # the prompt text leads the stream
    assert _text(chunks) == ch["text"]
    assert _post(server, ignore_eos=True, echo=False, **kw)[1]["choices"][0]["text"] == plain["choices"][0]["text"]


@pytest.mark.parametrize("n", [0, 1, 5])
def test_echo_with_logprobs_lists_the_prompt_first(server, n):
    st, body = _post(server, prompt=IDS, ignore_eos=True, echo=True, logprobs=n)
    assert st == 200, body
    ch = body["choices"][0]
    lp = ch["logprobs"]
    assert list(lp) == ["tokens", "token_logprobs", "top_logprobs", "text_offset"]
    assert len(lp["tokens"]) == len(IDS) + 8
    assert lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None     # the first token has no record
    assert "".join(lp["tokens"]) == ch["text"]
    off = 0
    for k, (tok, v, top, o) in enumerate(_entries(lp)):
        assert o == off
        off += len(tok)
        if k == 0:
            continue
        t = IDS[k] if k < len(IDS) else next(i for i in range(VOCAB) if LS._placeholder(i) == tok)
        want, alts = LS._want_record(t, n)
        assert tok == LS._placeholder(t) and v == want
        assert top == {LS._placeholder(i): a for i, a in alts}
    # the generated entries are those of the request without echo
    st, plain = _post(server, prompt=IDS, ignore_eos=True, logprobs=n)
    gen = _entries(plain["choices"][0]["logprobs"])
    shift = len("".join(LS._placeholder(t) for t in IDS))
    assert _entries(lp)[len(IDS):] == [[a, b, c, d + shift] for a, b, c, d in gen]


@pytest.mark.parametrize("case", [dict(max_tokens=12, ignore_eos=True), dict(max_tokens=30, stop="e"),
                                  dict(max_tokens=20, temperature=0.8, seed=3, ignore_eos=True)])
@pytest.mark.parametrize("tok", [False, True])
def test_streamed_prompt_and_token_entries_concatenate_to_the_body(server, tok_server, case, tok):
    port = tok_server if tok else server
    kw = dict(case, prompt=[9, 8, 7, 300, 301], echo=True, logprobs=3)
    st, body = _post(port, **kw)
    assert st == 200, body
    chunks, _ = _stream(port, **kw)
    assert _stream_entries(chunks) == _entries(body["choices"][0]["logprobs"])
    assert _text(chunks) == body["choices"][0]["text"]
    first = chunks[0]["choices"][0]
    assert len(first["logprobs"]["tokens"]) == 5 and first["logprobs"]["token_logprobs"][0] is None


def test_string_prompt_round_trips_through_the_tokenizer(tok_server):
    """The echoed text of a string prompt is the string itself; with logprobs, the prompt tokens' texts (BOS included: a
    special token with no text) and offsets line up with it, multi-byte UTF-8 included."""
    for prompt in ("hello there", "naïve café — 東京 🙂 done", "  spaces\tand\nlines "):
        st, body = _post(tok_server, prompt=prompt, ignore_eos=True, max_tokens=4, echo=True, logprobs=1)
        assert st == 200, body
        ch = body["choices"][0]
        assert ch["text"].startswith(prompt)
        lp = ch["logprobs"]
        n_prompt = body["usage"]["prompt_tokens"]
        offs = lp["text_offset"][:n_prompt]
        assert offs == sorted(offs) and offs[0] == 0 and all(o <= len(prompt) for o in offs)
        assert lp["token_logprobs"][0] is None and all(v is not None for v in lp["token_logprobs"][1:])
        assert lp["text_offset"][n_prompt] == len(prompt)                         # the first generated token starts after it
        st, alone = _post(tok_server, prompt=prompt, ignore_eos=True, max_tokens=4, echo=True)
        assert alone["choices"][0]["text"] == ch["text"]


def test_chat_ignores_echo_and_non_echo_requests_keep_their_shape(server):
    st, a = LS._post(server, CHAT, prompt_token_ids=[5, 6, 7], ignore_eos=True)
    st2, b = LS._post(server, CHAT, prompt_token_ids=[5, 6, 7], ignore_eos=True, echo=True)
    assert st == st2 == 200 and a["choices"] == b["choices"]


def test_a_server_on_an_engine_without_prompt_logprobs_refuses_echo_with_logprobs(old_server):
    for n in (0, 1, 5):
        st, body = _post(old_server, prompt=IDS, echo=True, logprobs=n)
        assert st == 400 and "echo" in body["error"]["message"] and body["error"]["type"] == "invalid_request_error", body
    st, body = _post(old_server, prompt=IDS, echo=True, ignore_eos=True)                 # echo alone needs no entry point
    assert st == 200 and body["choices"][0]["text"].startswith("".join(LS._placeholder(t) for t in IDS))
    chunks, raw = _stream(old_server, prompt=IDS, echo=True, ignore_eos=True)
    assert json.loads(json.dumps(chunks))[0]["choices"][0]["text"] == "".join(LS._placeholder(t) for t in IDS)


def _string_offsets(s, n_bytes):
    """text_offset of each prompt token of string s, whose tokens are made of n_bytes[i] bytes of it: the code points of s
    before the token, a character cut by a token boundary counting from the token that completes it."""
    b, at, out = s.encode(), 0, []
    for n in n_bytes:
        start = sum(1 for c in b[:at] if c & 0xC0 != 0x80)
        out.append(start - (1 if at < len(b) and b[at] & 0xC0 == 0x80 else 0))
        at = min(len(b), at + n)
    return out


def test_string_prompt_offsets_point_into_the_string_itself(server):
    """Without a tokenizer, every byte of a string is one placeholder token, and bytes outside printable ASCII detokenize to
    "<|id|>": the echoed text is still the string, and the prompt offsets count its code points, not the placeholder's."""
    prompt = "aé\tb€\x01c"
    st, body = _post(server, prompt=prompt, ignore_eos=True, max_tokens=3, echo=True, logprobs=1)
    assert st == 200, body
    ch = body["choices"][0]
    n = len(prompt.encode())
    assert ch["text"].startswith(prompt) and body["usage"]["prompt_tokens"] == n
    offs = ch["logprobs"]["text_offset"]
    assert offs[:n] == _string_offsets(prompt, [1] * n) == [0, 1, 1, 2, 3, 4, 4, 4, 5, 6]
    assert offs[n] == len(prompt)
