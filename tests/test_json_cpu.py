"""CPU: the JSON grammar of `format: "json"` -- the Python restatement (tests/json_oracle.py) against Python's own json module and
hand-written answers, the device automaton (gridllm_b200/csrc/json_fsm.h, compiled for the host) against the restatement state
for state, the C ABI layout of gl_sample_opts.format, and the service's mapping of `format` end to end over an engine double
that applies the restated mask."""
import asyncio
import ctypes
import json
import os
import random
import re
import subprocess

import numpy as np
import pytest

import json_oracle as J
from conftest import ROOT


# ---- a seeded corpus -------------------------------------------------------------------------------------------------
_WORDS = ["alpha", "beta", "naïve", "café", "✓ ok", "日本語", "emoji 😀", "quote \" and \\ slash /", "tab\tnew\nline", "\u0001ctl",
          "", "x" * 40, "é́", "\U0010fffd"]


def _value(rnd, depth, max_depth):
    r = rnd.random()
    if depth < max_depth and r < 0.25:
        return {rnd.choice(_WORDS) + str(i): _value(rnd, depth + 1, max_depth) for i in range(rnd.randint(0, 4))}
    if depth < max_depth and r < 0.45:
        return [_value(rnd, depth + 1, max_depth) for _ in range(rnd.randint(0, 4))]
    r = rnd.random()
    if r < 0.2:
        return rnd.choice(_WORDS)
    if r < 0.35:
        return rnd.randint(-10**12, 10**12)
    if r < 0.5:
        return rnd.choice([0, -0, 1, -1, 7, 10, 120])
    if r < 0.7:
        return rnd.uniform(-1e6, 1e6) * (10.0 ** rnd.randint(-30, 30))
    return rnd.choice([True, False, None])


def corpus(seed=7, n=60):
    rnd = random.Random(seed)
    docs = []
    for i in range(n):
        d = {f"k{j}": _value(rnd, 2, 2 + (i % 9)) for j in range(rnd.randint(0, 5))}
        docs.append(json.dumps(d).encode())                                       # default separators, ASCII escapes
        docs.append(json.dumps(d, ensure_ascii=False).encode("utf-8"))            # raw UTF-8 in strings
        docs.append(json.dumps(d, indent=2, ensure_ascii=i % 2 == 0).encode("utf-8"))      # depth <= 10: indent <= 20
    return docs


def _no_constants(name):
    raise ValueError(name)


def _loads_dict(data):
    try:
        v = json.loads(data, parse_constant=_no_constants)
    except (ValueError, UnicodeDecodeError, RecursionError):
        return None
    return v if isinstance(v, dict) else None


def _meets_rules(data):
    """the whitespace / depth rules of the language, checked on text json.loads accepted: no whitespace before the root, every
    run of whitespace between tokens is "" / " " / "\\n" [ \\t]{0,20}, depth <= 64"""
    s = data.decode("utf-8")
    if not s.startswith("{"):
        return False
    depth, i, in_str = 0, 0, False
    while i < len(s):
        c = s[i]
        if in_str:
            if c == "\\":
                i += 2
                continue
            in_str = c != '"'
            i += 1
            continue
        if c == '"':
            in_str = True
        elif c in "{[":
            depth += 1
            if depth > J.MAX_DEPTH:
                return False
        elif c in "}]":
            depth -= 1
        elif c in " \t\n\r":
            m = re.match(r"[ \t\n\r]+", s[i:]).group(0)
            if not re.fullmatch(r" |\n[ \t]{0,20}", m):
                return False
            i += len(m)
            continue
        i += 1
    return True


def test_corpus_documents_are_complete_and_every_prefix_viable():
    n = 0
    for doc in corpus():
        st = J.INITIAL
        for k, c in enumerate(doc):
            st = J.step(st, c)
            assert st is not None, (doc[: k + 1],)
            if k < len(doc) - 1:
                assert not J.done(st) or doc[k + 1:].strip(b" \n\t") == b""
        assert J.done(st), doc
        n += 1
    assert n == 180


def _mutations(rnd, doc):
    b = bytearray(doc)
    k = rnd.randrange(6)
    if k == 0 and len(b) > 1:
        return bytes(b[: rnd.randrange(1, len(b))])                     # truncation
    p = rnd.randrange(len(b) + 1)
    if k == 1:
        return bytes(b[:p] + bytes([rnd.randrange(256)]) + b[p:])        # random byte inserted
    if k == 2:
        return bytes(b[:p] + rnd.choice([b" ", b"\n", b"  ", b"\r", b"\t", b"\n" + b" " * 21, b",", b"}", b"]", b"0", b"-", b'"']) + b[p:])
    if k == 3 and len(b):
        b[min(p, len(b) - 1)] = rnd.randrange(256)                        # random byte replaced
        return bytes(b)
    if k == 4:
        return bytes(b) + rnd.choice([b" ", b"\n\t\t", b"\n" + b" " * 20, b"\n" + b" " * 21, b"x", b"{}"])
    return bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 12)))


def test_fuzz_agrees_with_python_json():
    rnd = random.Random(11)
    docs = corpus(seed=3, n=30)
    accepted = parsed = 0
    for _ in range(6000):
        m = _mutations(rnd, rnd.choice(docs))
        ok = J.complete(m)
        d = _loads_dict(m)
        if ok:
            assert d is not None, m                                       # the language is JSON
            accepted += 1
        if d is not None and _meets_rules(m):
            assert ok, m                                                   # ... all of it that meets the stated rules
            parsed += 1
    assert accepted > 500 and parsed > 500


def test_utf8_in_strings_agrees_with_the_strict_decoder():
    rnd = random.Random(5)
    pool = list(range(0x80, 0x100)) + [ord(c) for c in "abc xyz"]
    agree = valid = 0
    for _ in range(20000):
        body = bytes(rnd.choice(pool) for _ in range(rnd.randint(1, 6)))
        try:
            body.decode("utf-8", "strict")
            ok = True
        except UnicodeDecodeError:
            ok = False
        assert J.complete(b'{"k": "' + body + b'"}') == ok, body
        agree += 1
        valid += ok
    assert valid > 200 and agree == 20000
    # the edges of RFC 3629: overlongs, surrogates, above U+10FFFF, truncated sequences
    for bad in (b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xf0\x80\x80\x80", b"\xf4\x90\x80\x80",
                b"\xf5\x80\x80\x80", b"\xe2\x82", b"\x80"):
        assert not J.complete(b'{"k": "' + bad + b'"}'), bad
    for good in (b"\xc2\x80", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf", b"\x7f"):
        assert J.complete(b'{"k": "' + good + b'"}'), good
    assert J.viable(b'{"k": "\xe2\x82')                                     # a piece may end inside a character


def test_known_answers():
    ok = [b"{}", b'{"a": 1}', b'{"a":-0}', b'{"a": 1e5}', b'{"a": 1E+5}', b'{"a": -0.25e-3}', b'{"a": [true, false, null]}',
          b'{"a": "\\u00e9\\n\\"\\\\\\/\\b\\f\\r\\t"}', b'{\n' + b"\t" * 20 + b'"a": {}}', b"{} ", b"{}\n" + b" " * 20,
          b'{"a" : {"b":[]}}', b'{ }', b'{"":""}']
    bad = [b"", b" {}", b"[]", b'"a"', b"{}x", b"{}{}", b'{"a": 01}', b'{"a": 1.}', b'{"a": .5}', b'{"a": +1}', b'{"a": 1e}',
           b'{"a": tru}', b'{"a": True}', b"{,}", b'{"a": 1,}', b'{"a" 1}', b"{a: 1}", b'{"a": "\\x"}', b'{"a": "\\u12g4"}',
           b'{"a": "\x1f"}', b"{  }", b"{\n" + b" " * 21 + b"}", b"{\n\n}", b"{ \n}", b"{}  ", b"{}\n" + b" " * 21, b'{"a": NaN}']
    for d in ok:
        assert J.complete(d), d
    for d in bad:
        assert not J.complete(d), d
    # viable but not complete: a stop token is masked there
    for d in (b"{", b'{"a"', b'{"a": 1', b'{"a": [', b'{"a": "x', b'{"a": -', b'{"a": 1e', b'{"a": {}'):
        assert J.viable(d) and not J.complete(d), d
    # depth 64, root included: the 64th bracket opens, the 65th is masked
    assert J.viable(b'{"a":' + b"[" * 63) and not J.viable(b'{"a":' + b"[" * 64)
    assert J.complete(b'{"a":' + b"[" * 63 + b"]" * 63 + b"}")
    # stop tokens: only once the root has closed, anywhere in its trailing ws; ws budget 20 after a newline
    pieces = [bytes([i]) for i in range(128)] + [b"", b""]                   # ids 128, 129: a stop token and a control token
    for gen, stop_ok in ((b"", False), (b"{", False), (b'{"a":1', False), (b"{}", True), (b"{} ", True), (b"{}\n\t", True)):
        m = J.mask(pieces, [128], list(gen))
        assert m[128] == stop_ok and not m[129], gen
    m = J.mask(pieces, [128], list(b"{}\n" + b" " * 20))
    assert np.flatnonzero(m).tolist() == [128]                              # nothing but the stop token is left
    m = J.mask(pieces, [128], list(b"{}\n" + b" " * 19))
    assert sorted(np.flatnonzero(m).tolist()) == [9, 32, 128]
    assert np.flatnonzero(J.mask(pieces, [128], [])).tolist() == [ord("{")]


# ---- the device automaton, compiled for the host ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def json_fsm_lib(tmp_path_factory):
    """CPU build of json_fsm.h through tests/hostcheck/json_shim.cpp -- test infrastructure only"""
    out = str(tmp_path_factory.mktemp("jsonfsm") / "libjsonfsm.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "json_shim.cpp")])
    lib = ctypes.CDLL(out)
    lib.jf_trace.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    assert lib.jf_state_bytes() == 16
    return lib


def _c_trace(lib, data):
    buf = np.zeros((max(1, len(data)), 16), np.uint8)
    done = ctypes.c_int(0)
    n = lib.jf_trace(bytes(data), len(data), buf.ctypes.data_as(ctypes.c_void_p), ctypes.byref(done))
    states = []
    for row in buf[:n]:
        lo, hi = int(row[:4].view(np.uint32)[0]), int(row[4:8].view(np.uint32)[0])
        mode, depth, cnt, aux, key = (int(x) for x in row[8:13])
        states.append((mode, depth, lo | (hi << 32), cnt, aux, key))
    return n, states, bool(done.value)


def _py_trace(data):
    st, states = J.INITIAL, []
    for c in data:
        st = J.step(st, c)
        if st is None:
            break
        states.append(st)
    return len(states), states


def _same(a, b):
    """the stack bits above the depth are not part of the state"""
    mask = (1 << a[1]) - 1
    return a[:2] == b[:2] and (a[2] & mask) == (b[2] & mask) and a[3:] == b[3:]


def test_device_automaton_matches_the_oracle_state_for_state(json_fsm_lib):
    rnd = random.Random(17)
    docs = corpus(seed=9, n=40)
    inputs = list(docs) + [_mutations(rnd, rnd.choice(docs)) for _ in range(3000)]
    inputs += [b'{"a":' + b"[" * 70, b"{}\n" + b" " * 25, b'{"k": "\xf4\x8f\xbf\xbf\xf4\x90"}']
    for data in inputs:
        n_c, s_c, done_c = _c_trace(json_fsm_lib, data)
        n_p, s_p = _py_trace(data)
        assert n_c == n_p, data
        for k, (a, b) in enumerate(zip(s_c, s_p)):
            assert _same(a, b), (data[: k + 1], a, b)
        if n_c == len(data):
            assert done_c == J.done(s_p[-1] if s_p else J.INITIAL), data


# ---- C ABI ---------------------------------------------------------------------------------------------------------------
def test_sample_opts_format_field():
    from gridllm_b200 import native as N
    S = N.SampleOpts
    assert ctypes.sizeof(S) == 72
    old = {"num_predict": 0, "temperature": 4, "top_k": 8, "top_p": 12, "seed": 16, "ignore_eos": 24, "n_stop_ids": 28, "stop_ids": 32,
           "want_logits": 40, "repeat_penalty": 44, "repeat_last_n": 48, "presence_penalty": 52, "frequency_penalty": 56, "min_p": 60}
    assert {k: getattr(S, k).offset for k in old} == old
    assert S.format.offset == 64 and S.reserved.offset == 64
    z = S()
    assert z.format == 0 and list(z.reserved) == [0]                       # a zeroed struct: off
    z.format = N.GL_FORMAT_JSON
    assert list(z.reserved) == [1]
    assert "gl_constrain_logits" in N.ABI_SYMBOLS
    hdr = open(os.path.join(ROOT, "include", "gridllm_native.h")).read()
    assert "#define GL_FORMAT_JSON 1" in hdr and "gl_constrain_logits(" in hdr
    assert N._format_code(None) == 0 and N._format_code("") == 0 and N._format_code("json") == 1
    with pytest.raises(ValueError):
        N._format_code("yaml")


# ---- service mapping -----------------------------------------------------------------------------------------------------
def _service(**kw):
    from gridllm_b200 import service as SV
    return SV.NativeInferenceService({}, **kw)


def test_service_format_mapping():
    s = _service()
    F = s._format
    assert F({}) == {} and F({"options": {}}) == {} and F({"metadata": {}}) == {}
    assert F({"metadata": {"format": "json"}}) == {"format": "json"}
    assert F({"options": {"format": "json"}}) == {"format": "json"}                       # the OpenAI route's place
    schema = {"type": "object", "properties": {"a": {"type": "integer"}}}
    assert F({"metadata": {"format": schema}}) == {"format": "json"}                      # valid JSON; the schema is not enforced
    assert F({"options": {"format": schema}}) == {"format": "json"}
    assert F({"metadata": {"format": None}}) == {} and F({"metadata": {"format": ""}}) == {}
    assert F({"metadata": {"format": ""}, "options": {"format": "json"}}) == {"format": "json"}
    assert F({"metadata": {"format": "json"}, "options": {"format": "bogus"}}) == {"format": "json"}     # metadata first
    for bad in ("yaml", "JSON", 1, True, ["json"]):
        with pytest.raises(RuntimeError):
            F({"metadata": {"format": bad}})
    # the sampling and penalty maps do not see it
    assert s._sampling({"format": "json"}) == {} and s._penalties({"format": "json"}) == {}


# ---- end to end over the engine double -----------------------------------------------------------------------------------
def _json_double():
    import oracle_engine
    from oracle import llama_oracle as O, sampler as SM

    class JsonDouble(oracle_engine.OracleEngine):
        """the oracle-backed engine double with the `format` keyword of native.Engine: before every draw the restated mask
        (json_oracle.apply_mask).  bias: a bonus on the closing bytes and eos, standing in for a model that wants to finish."""
        bias = 0.0

        def _pieces(self):
            if not hasattr(self, "_pc"):
                self._pc = [self.token_piece(t) for t in range(self.info.n_vocab)]
                self._bonus = np.zeros(self.info.n_vocab, np.float32)
                for t, p in enumerate(self._pc):
                    if p in (b"}", b"]", b'"'):
                        self._bonus[t] = 1.0
                self._bonus[self.info.eos_id] = 1.0
            return self._pc

        def _draw(self, logits, gen, stops, opts, i, fmt):
            if fmt == "json":
                pieces = self._pieces()
                logits = J.apply_mask(logits + self.bias * self._bonus, pieces, stops, gen)
            return SM.sample(logits, *opts, i)

        def generate(self, prompt, num_predict=128, ignore_eos=False, on_token=None, want_logits=False, stop_ids=(), temperature=0.0,
                     top_k=0, top_p=1.0, seed=0, format=None):
            self.formats = getattr(self, "formats", []) + [format]
            assert not (format and ignore_eos)
            orc = O.LlamaOracle(self.m, act="i16", kv_f16=True)
            logits = None
            for t in prompt:
                logits = orc.step(int(t))
            stops = set(int(s) for s in stop_ids) | ({self.info.eos_id, self.info.eot_id} if not ignore_eos else set())
            ids, lps, reason = [], [], 1
            for i in range(num_predict):
                tok, lp, _ = self._draw(logits, ids, stops, (temperature, top_k, top_p, seed), i, format)
                if tok in stops:
                    reason = 0
                    break
                ids.append(tok)
                lps.append(lp)
                if on_token is not None and on_token(tok, lp, self._bytes([tok])):
                    reason = 2
                    break
                logits = orc.step(tok)
            from types import SimpleNamespace
            st = SimpleNamespace(prompt_eval_count=len(prompt), eval_count=len(ids), prompt_eval_duration_ns=1, eval_duration_ns=1,
                                 total_duration_ns=2, load_duration_ns=1, done_reason=reason, kernel_launches=0)
            return SimpleNamespace(ids=np.array(ids, dtype=np.int32), logprobs=np.array(lps, dtype=np.float32), stats=st)

        def seq_open(self, prompt, num_predict=128, ignore_eos=False, temperature=0.0, top_k=0, top_p=1.0, seed=0, stop_ids=(), format=None):
            self.formats = getattr(self, "formats", []) + [format]
            slot = super().seq_open(prompt, num_predict, ignore_eos, temperature, top_k, top_p, seed, stop_ids)
            self._seqs[slot].fmt, self._seqs[slot].gen = format, []
            return slot

        def batch_step(self, cap=128):
            out = []
            for slot, q in sorted(getattr(self, "_seqs", {}).items()):
                if q.done:
                    continue
                tok, lp, _ = self._draw(q.logits, q.gen, q.stops, q.opts, q.n, q.fmt)
                if tok in q.stops:
                    q.done = q.stopped = True
                    out.append((slot, -1, 0.0, True))
                    continue
                q.n += 1
                q.gen.append(int(tok))
                q.done = q.n >= q.n_pred
                out.append((slot, int(tok), float(lp), q.done))
                if not q.done:
                    q.logits = q.orc.step(int(tok))
            return out

    return JsonDouble


def _run(coro):
    return asyncio.new_event_loop().run_until_complete(coro)


@pytest.mark.parametrize("max_batch", [0, 4])
def test_json_requests_end_to_end(tiny_gguf, hostcheck_lib, monkeypatch, max_batch):
    import oracle_engine
    from gridllm_b200 import service as SV
    oracle_engine.use_hostcheck(hostcheck_lib)
    Double = _json_double()
    monkeypatch.setattr(SV.N, "Engine", Double)
    monkeypatch.setattr(SV.N, "device_count", lambda: 1)
    svc = SV.NativeInferenceService({"tiny:latest": tiny_gguf}, device=0, max_batch=max_batch)
    try:
        eng = svc._engine("tiny:latest")
        req = {"id": "j1", "model": "tiny:latest", "prompt": "the rain in spain", "priority": "medium",
               "options": {"num_predict": 24, "temperature": 0}, "metadata": {"format": "json"}}
        # free-running model: a viable prefix cut by num_predict
        res = _run(svc.generateResponse(req))
        assert eng.formats[-1] == "json" and res["done_reason"] == "length"
        assert J.viable(res["response"].encode("utf-8")) and res["response"].startswith("{")

        async def collect(r):
            return [c async for c in svc.generateStreamResponse(r)]
        chunks = _run(collect(dict(req, id="j2")))
        acc = b""
        for c in chunks:
            acc += c["response"].encode("utf-8")
            assert J.viable(acc), acc                                         # every streamed concatenation
        assert acc.decode("utf-8") == res["response"]
        # a model that wants to finish: the document closes, the stop token ends it, the response parses
        Double.bias = 50.0
        for r in (dict(req, id="j3"), dict(req, id="j4", metadata={}, options=dict(req["options"], format={"type": "object"}))):
            out = _run(svc.generateResponse(r))
            assert out["done_reason"] == "stop" and isinstance(json.loads(out["response"]), dict), out["response"]
        chat = {"id": "c1", "model": "tiny:latest", "priority": "low", "options": {"num_predict": 24},
                "metadata": {"messages": [{"role": "user", "content": "reply in JSON"}], "format": "json"}}
        out = _run(svc.generateChatResponse(chat))
        assert isinstance(json.loads(out["message"]["content"]), dict)
        async def collect_chat(r):
            return [c async for c in svc.generateChatStreamResponse(r)]
        chunks = _run(collect_chat(dict(chat, id="c2")))
        text = "".join(c["response"] for c in chunks)
        assert text == out["message"]["content"]
        Double.bias = 0.0
        # without format: no keyword reaches the engine (a request without format is unchanged)
        _run(svc.generateResponse(dict(req, id="j5", metadata={})))
        assert eng.formats[-1] is None
        # refusals
        with pytest.raises(RuntimeError):
            _run(svc.generateResponse(dict(req, id="j6", options={"ignore_eos": True}, metadata={"format": "json"})))
        with pytest.raises(RuntimeError):
            _run(svc.generateResponse(dict(req, id="j7", metadata={"format": "xml"})))
        # embeddings ignore it
        emb = _run(svc.generateEmbedding({"id": "e1", "model": "tiny:latest", "input": ["hi"], "metadata": {"format": "json"}}))
        assert len(emb["embeddings"]) == 1
    finally:
        Double.bias = 0.0
        svc.close()
