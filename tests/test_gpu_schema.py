"""GPU: the JSON schema mask (gridllm_b200/csrc/schema_mask.cu, automaton schema_fsm.h) against the restatement in
tests/schema_oracle.py, through the C ABI.

Stated bars: gl_constrain_logits with a schema code masks exactly the tokens schema_oracle.mask refuses and leaves every other
logit bit-unchanged; greedy gl_generate follows the oracle model's decode loop with the oracle mask (ids equal wherever the
masked top-1/top-2 margin > 5e-2); a finite schema ends on a stop token with a document jsonschema accepts; sampled draws never
take a masked token; rows with different schemas, "json" rows and free rows share a batch and give the tokens they give alone
and from gl_generate; a schema request runs one kernel more per draw; the registry keeps codes, keeps schemas in use and
refuses evicted codes."""
import json

import numpy as np
import pytest

import schema_oracle as SO

pytestmark = pytest.mark.gpu

PERSON = {"$defs": {"Address": {"properties": {"street": {"title": "Street", "type": "string", "maxLength": 12},
                                               "zip": {"anyOf": [{"type": "string"}, {"type": "null"}], "default": None}},
                                "required": ["street"], "title": "Address", "type": "object"}},
          "properties": {"name": {"type": "string", "maxLength": 8}, "age": {"type": "integer"},
                         "tags": {"items": {"type": "string", "maxLength": 4}, "type": "array", "maxItems": 2},
                         "home": {"$ref": "#/$defs/Address"}},
          "required": ["name", "age", "tags"], "title": "Person", "type": "object"}
FINITE = {"type": "object", "properties": {"ok": {"type": "boolean"}, "color": {"enum": ["red", "green", "blue"]}, "n": {"enum": [1, 22, None]}},
          "required": ["ok", "color", "n"]}
TREE = {"$defs": {"T": {"type": "object", "properties": {"v": {"type": "integer"}, "kids": {"type": "array", "items": {"$ref": "#/$defs/T"}}},
                        "required": ["v"]}}, "$ref": "#/$defs/T"}


def _engine(path, **kw):
    from gridllm_b200 import native as N
    return N.Engine(path, **kw)


def _pieces(e):
    return [e.token_piece(t) for t in range(e.info.n_vocab)]


def _stops(e):
    return [s for s in (e.info.eos_id, e.info.eot_id) if s >= 0]


DOCS = [(PERSON, {"name": "Ann", "age": 41, "tags": ["a", "bc"], "home": {"street": "Main St", "zip": None}}),
        (PERSON, {"name": "Bo", "age": -7, "tags": []}),
        (FINITE, {"ok": True, "color": "green", "n": 22}),
        (TREE, {"v": 1, "kids": [{"v": 2}, {"v": 3, "kids": []}]})]


def _check_constrain(e, rng, every=1):
    from gridllm_b200 import native as N
    pieces, stops, n = _pieces(e), _stops(e), e.info.n_vocab
    cases = 0
    for schema, doc in DOCS:
        code = e.format_schema(schema)
        root = SO.compile_schema(schema)
        for indent in (None, 1):
            ids = [int(t) for t in e.tokenize(json.dumps(doc, indent=indent), add_bos=False)]
            for cut in range(0, len(ids) + 1, every):
                logits = (rng.standard_normal(n) * 3).astype(np.float32)
                got = e.constrain_logits(logits, ids[:cut], format=code)
                want = SO.mask(root, pieces, stops, ids[:cut])
                assert np.array_equal(np.isneginf(got), ~want), (schema.get("title"), cut, np.flatnonzero(np.isneginf(got) != ~want)[:10])
                assert np.array_equal(got[want].view(np.uint32), logits[want].view(np.uint32))
                assert want.any()
                cases += 1
    byte_tok = {p[0]: t for t, p in enumerate(pieces) if len(p) == 1}
    with pytest.raises(N.NativeError) as ei:                       # a history outside the schema
        e.constrain_logits(np.zeros(n, np.float32), [byte_tok[c] for c in b'{"x'], format=e.format_schema(FINITE))
    assert ei.value.code == -1
    return cases


def test_constrain_logits_matches_the_oracle_mask(tiny_gguf):
    e = _engine(tiny_gguf)
    assert _check_constrain(e, np.random.Generator(np.random.PCG64(3))) > 100
    e.close()


def test_constrain_logits_on_a_llama3_sized_vocabulary(tmp_models):
    from oracle import gguf_synth as S
    path = str(tmp_models / "json_vocab_128k.gguf")
    S.build_model(path, S.LlamaShape("json-vocab-synth", 1, 256, 4, 2, 512, 128256, 10000.0, 1e-5, 512), "q8_0", seed=5)
    e = _engine(path)
    assert e.info.n_vocab == 128256
    assert _check_constrain(e, np.random.Generator(np.random.PCG64(4)), every=9) > 10
    e.close()


def _oracle_greedy(m, prompt, n, root, pieces, stops):
    from oracle import llama_oracle as O
    orc = O.LlamaOracle(m, act="i16", kv_f16=True)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    out = []
    for _ in range(n):
        ml = SO.apply_mask(root, logits, pieces, stops, [t for t, _ in out])
        tok = int(np.argmax(ml))
        srt = np.sort(ml)
        out.append((tok, float(srt[-1] - srt[-2])))
        if tok in stops:
            break
        logits = orc.step(tok)
    return out


def test_greedy_schema_generate_follows_the_oracle(tiny_gguf):
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    e = _engine(tiny_gguf, prefill_mode=1)
    pieces, stops = _pieces(e), _stops(e)
    root = SO.compile_schema(PERSON)
    compared = 0
    for seed in (2000, 2001):
        prompt = np.random.Generator(np.random.PCG64(seed)).integers(0, m.n_vocab - 3, size=20)
        g = e.generate(prompt, num_predict=20, want_logits=True, format=PERSON)
        assert SO.viable(root, b"".join(pieces[t] for t in g.ids))
        ref = _oracle_greedy(m, prompt, len(g.ids), root, pieces, stops)
        for i, (tok, margin) in enumerate(ref[: len(g.ids)]):
            assert np.array_equal(~np.isneginf(e.last_logits(i)), SO.mask(root, pieces, stops, list(g.ids[:i]))), (seed, i)
            compared += 1
            if int(g.ids[i]) != tok:
                assert margin <= 5e-2, (seed, i, margin)
                break
    assert compared >= 10
    e.close()


def test_finite_schema_ends_on_a_stop_token(tiny_gguf):
    import jsonschema
    e = _engine(tiny_gguf)
    pieces = _pieces(e)
    prompt = np.arange(10, 30)
    g = e.generate(prompt, num_predict=200, format=FINITE)
    text = b"".join(pieces[t] for t in g.ids)
    assert g.stats.done_reason == 0, text
    jsonschema.validate(json.loads(text), FINITE)
    e.close()


def test_sampled_schema_draws_never_take_a_masked_token(tiny_gguf):
    e = _engine(tiny_gguf)
    pieces, stops = _pieces(e), _stops(e)
    root = SO.compile_schema(PERSON)
    prompt = np.random.Generator(np.random.PCG64(23)).integers(0, e.info.n_vocab - 3, size=16)
    draws = 0
    for seed in range(4):
        kw = dict(num_predict=20, temperature=0.9, top_k=40, seed=seed, format=PERSON, repeat_penalty=1.3, presence_penalty=0.2)
        g = e.generate(prompt, want_logits=True, **kw)
        for i, t in enumerate(g.ids):
            mk = SO.mask(root, pieces, stops, list(g.ids[:i]))
            assert mk[t] and np.array_equal(~np.isneginf(e.last_logits(i)), mk), (seed, i)
            draws += 1
    assert draws > 40
    e.close()


def test_one_launch_more_per_draw(tiny_gguf):
    e = _engine(tiny_gguf)
    prompt = np.random.Generator(np.random.PCG64(31)).integers(0, e.info.n_vocab - 3, size=20)
    a = e.generate(prompt, num_predict=6, ignore_eos=True)
    b = e.generate(prompt, num_predict=10, ignore_eos=True)
    per = (b.stats.kernel_launches - a.stats.kernel_launches) // 4
    base = a.stats.kernel_launches - 6 * per
    j = e.generate(prompt, num_predict=12, format="json")
    assert j.stats.kernel_launches == base + max(j.stats.eval_count, 1) * (per + 1)
    for samp in ({}, dict(temperature=0.8, top_k=40, seed=3)):
        g = e.generate(prompt, num_predict=12, format=PERSON, **samp)
        assert g.stats.kernel_launches == base + max(g.stats.eval_count, 1) * (per + 1), samp
        x = e.generate(prompt, num_predict=10, ignore_eos=True)      # a request without format: unchanged
        assert np.array_equal(x.ids, b.ids) and x.stats.kernel_launches == b.stats.kernel_launches
        y = e.generate(prompt, num_predict=12, format="json")
        assert np.array_equal(y.ids, j.ids) and y.stats.kernel_launches == j.stats.kernel_launches
    e.close()


def _drain(e, want):
    out = {s: ([], []) for s in want}
    guard = 0
    while any(len(out[s][0]) < want[s] for s in want):
        guard += 1
        assert guard < 10000
        for slot, tok, lp, done in e.batch_step():
            if slot in out and len(out[slot][0]) < want[slot]:
                out[slot][1].append(e.seq_logits(slot))
                out[slot][0].append(int(tok))
                if done and tok < 0:
                    want[slot] = len(out[slot][0])
    return out


@pytest.mark.parametrize("mode", [1, 2])
def test_batched_schemas(tiny128_gguf, mode):
    e = _engine(tiny128_gguf, max_batch=8, max_ctx=1024, batch_weights=mode)
    pieces, stops = _pieces(e), _stops(e)
    rng = np.random.Generator(np.random.PCG64(41))
    prompts = [rng.integers(0, e.info.n_vocab - 3, size=k) for k in (40, 25, 30, 5, 33)]       # 5: the single-sequence open
    N_TOK = 14
    opts = [dict(num_predict=N_TOK, format=PERSON), dict(num_predict=N_TOK, format=TREE), dict(num_predict=N_TOK, format="json"),
            dict(num_predict=N_TOK, format=FINITE), dict(num_predict=N_TOK, ignore_eos=True)]
    alone = []
    for p, o in zip(prompts, opts):
        s = e.seq_open(p, **o)
        alone.append(_drain(e, {s: N_TOK})[s])
        e.seq_close(s)
    slots = e.seq_open_many([prompts[0], prompts[1], prompts[2]], opts[:3])
    slots += [e.seq_open(prompts[3], **opts[3]), e.seq_open(prompts[4], **opts[4])]
    got = _drain(e, {s: len(a[0]) for s, a in zip(slots, alone)})
    for s, a in zip(slots, alone):
        assert got[s][0] == a[0]
        assert all(np.array_equal(x, y) for x, y in zip(got[s][1], a[1]))
        e.seq_close(s)
    for (ids, lgs), o in zip(alone[:4], opts[:4]):
        real = [t for t in ids if t >= 0]
        if isinstance(o["format"], dict):
            root = SO.compile_schema(o["format"])
            for i, lg in enumerate(lgs[: len(real)]):
                assert np.array_equal(~np.isneginf(lg), SO.mask(root, pieces, stops, real[:i])), i
    for p, o, (ids, _) in zip(prompts, opts, alone):
        g = e.generate(p, want_logits=True, **o)
        for i in range(min(len(g.ids), len([t for t in ids if t >= 0]))):
            if int(g.ids[i]) != ids[i]:
                lgi = e.last_logits(i)
                srt = np.sort(lgi)
                assert srt[-1] - srt[-2] <= 2e-2 * float(np.abs(lgi[np.isfinite(lgi)]).max()), (i, srt[-1] - srt[-2])
                break
    e.close()


def test_registry(tiny128_gguf, monkeypatch):
    from gridllm_b200 import native as N
    e = _engine(tiny128_gguf, max_batch=4, max_ctx=512)
    a = e.format_schema(FINITE)
    assert a >= N.GL_FORMAT_SCHEMA_BASE and e.format_schema(FINITE) == a
    assert e.format_schema(json.dumps(FINITE, ensure_ascii=False, separators=(",", ":"))) == a
    prompt = np.arange(10, 40)
    slot = e.seq_open(prompt, num_predict=4, format=a)               # in use: never evicted
    codes = [e.format_schema({"type": "object", "properties": {"k%d" % i: {"type": "integer"}}}) for i in range(70)]
    assert len(set(codes)) == 70 and a not in codes
    assert e.format_schema(FINITE) == a
    _drain(e, {slot: 4})
    e.seq_close(slot)
    with pytest.raises(N.NativeError) as ei:                         # the first of the 70: evicted
        e.generate(prompt, num_predict=2, format=codes[0])
    assert ei.value.code == -1
    with pytest.raises(N.NativeError) as ei:
        e.format_schema({"type": "object", "properties": {"zip": {"type": "string", "pattern": "x"}}})
    assert ei.value.code == -4 and "'pattern' is not supported at /properties/zip" in ei.value.detail
    with pytest.raises(N.NativeError) as ei:
        e.format_schema(b'{"type":')
    assert ei.value.code == -1
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=2, format=N.GL_FORMAT_SCHEMA_BASE + 100000)
    assert ei.value.code == -1
    e.close()
    monkeypatch.setenv("GL_MEGA", "1")
    m = _engine(tiny128_gguf, prefill_mode=1)
    with pytest.raises(N.NativeError) as ei:
        m.generate(prompt, num_predict=2, format=FINITE)
    assert ei.value.code == -4
    m.close()
