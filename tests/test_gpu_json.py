"""GPU: the JSON grammar mask (gridllm_b200/csrc/json_mask.cu, automaton json_fsm.h) against the restatement in
tests/json_oracle.py, through the C ABI.

Stated bars: gl_constrain_logits masks exactly the tokens json_oracle.mask refuses and leaves every other logit bit-unchanged;
a greedy JSON gl_generate follows the oracle model's decode loop with the oracle mask (ids equal wherever the masked top-1/top-2
margin > 5e-2, logits within 2e-3 * max|logit| of the i16 oracle, logprob within 2e-2); sampled JSON draws lie inside the
oracle's interval of the masked logits to 1e-4 and never take a masked token; a JSON request runs one kernel more per draw; rows
without JSON are bit-identical beside JSON rows, and JSON rows give the same tokens however they are admitted."""
import json

import numpy as np
import pytest

import json_oracle as J

pytestmark = pytest.mark.gpu


def _engine(path, **kw):
    from gridllm_b200 import native as N
    return N.Engine(path, **kw)


def _pieces(e):
    return [e.token_piece(t) for t in range(e.info.n_vocab)]


def _stops(e):
    return [s for s in (e.info.eos_id, e.info.eot_id) if s >= 0]


def _histories(e, pieces, rng, n_docs=6):
    """token histories the mask is checked after: every cut point of tokenised seeded documents, in-string partial UTF-8 (byte
    tokens), depth 64, complete documents with and without ws budget left"""
    byte_tok = {p[0]: t for t, p in enumerate(pieces) if len(p) == 1}
    docs = []
    for i in range(n_docs):
        d = {"name": "café ✓", "n": [1, -0.5, 3e8, True, None], "k%d" % i: {"x": "quote \" \\ é", "y": []}}
        docs.append(json.dumps(d, ensure_ascii=i % 2 == 0, indent=2 if i % 3 == 0 else None))
    hist = []
    for text in docs:
        ids = [int(t) for t in e.tokenize(text, add_bos=False)]
        for cut in range(0, len(ids) + 1, max(1, len(ids) // 40)):
            hist.append(ids[:cut])
        hist.append(ids)
    by = lambda bs: [byte_tok[b] for b in bs]
    hist.append(by(b'{"s": "\xe2'))                       # inside a 3-byte character
    hist.append(by(b'{"s": "\xf0\x9f'))                   # inside a 4-byte character
    hist.append(by(b'{"s": "\xed'))                       # surrogate range excluded next
    hist.append(by(b'{"s": "\\u00'))
    hist.append(by(b'{"a":' + b"[" * 63))                 # depth 64: no bracket opens
    hist.append(by(b'{"a":' + b"[" * 62))
    hist.append(by(b"{}"))                                # complete, the whole ws budget left
    hist.append(by(b"{}\n" + b"\t" * 19))                 # one ws byte left
    hist.append(by(b"{}\n" + b" " * 20))                  # none left: only the stop tokens
    hist.append(by(b'{"a": 12'))
    return hist


def _check_constrain(e, rng):
    from gridllm_b200 import native as N
    pieces = _pieces(e)
    stops = _stops(e)
    n = e.info.n_vocab
    cases = 0
    for h in _histories(e, pieces, rng):
        logits = (rng.standard_normal(n) * 3).astype(np.float32)
        got = e.constrain_logits(logits, h)
        want = J.mask(pieces, stops, h)
        assert np.array_equal(np.isneginf(got), ~want), (h, np.flatnonzero(np.isneginf(got) != ~want)[:10])
        assert np.array_equal(got[want].view(np.uint32), logits[want].view(np.uint32))
        assert want.any()
        cases += 1
    # format off: nothing changes; an invalid history is refused
    logits = rng.standard_normal(n).astype(np.float32)
    assert np.array_equal(e.constrain_logits(logits, [], format=None), logits)
    byte_tok = {p[0]: t for t, p in enumerate(pieces) if len(p) == 1}
    for bad in ([byte_tok[ord("[")]], [byte_tok[ord("{")], byte_tok[ord("}")], byte_tok[ord("}")]], [byte_tok[ord("{")], stops[0]],
                [byte_tok[ord("{")], byte_tok[ord("\n")], byte_tok[ord("\n")]]):
        with pytest.raises(N.NativeError) as ei:
            e.constrain_logits(logits, bad)
        assert ei.value.code == -1
    return cases


def test_constrain_logits_matches_the_oracle_mask(tiny_gguf):
    e = _engine(tiny_gguf)
    assert _check_constrain(e, np.random.Generator(np.random.PCG64(3))) > 100
    e.close()


def test_constrain_logits_on_a_llama3_sized_vocabulary(tmp_models):
    """128 256 entries: 501 CTAs per row"""
    from oracle import gguf_synth as S
    path = str(tmp_models / "json_vocab_128k.gguf")
    S.build_model(path, S.LlamaShape("json-vocab-synth", 1, 256, 4, 2, 512, 128256, 10000.0, 1e-5, 512), "q8_0", seed=5)
    e = _engine(path)
    assert e.info.n_vocab == 128256
    assert _check_constrain(e, np.random.Generator(np.random.PCG64(4))) > 100
    e.close()


def _oracle_json_greedy(m, prompt, n, pieces, stops, act, pen=None):
    import penalty_oracle as PO
    from oracle import llama_oracle as O
    orc = O.LlamaOracle(m, act=act, kv_f16=True)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    hist, out = [int(t) for t in prompt], []
    for _ in range(n):
        lg = PO.penalize(logits, hist, **pen) if pen else logits
        ml = J.apply_mask(lg, pieces, stops, [t for t, *_ in out])
        tok = int(np.argmax(ml))
        srt = np.sort(ml)
        lse = float(ml.max()) + float(np.log(np.exp(ml.astype(np.float64) - ml.max()).sum()))
        out.append((tok, float(ml[tok]) - lse, float(srt[-1] - srt[-2]), ml))
        if tok in stops:
            break
        hist.append(tok)
        logits = orc.step(tok)
    return out


def test_greedy_json_generate_follows_the_oracle(tiny_gguf):
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    e = _engine(tiny_gguf, prefill_mode=1)
    pieces, stops = _pieces(e), _stops(e)
    compared = 0
    for seed in (2000, 2001, 2002):
        prompt = np.random.Generator(np.random.PCG64(seed)).integers(0, m.n_vocab - 3, size=20)
        g = e.generate(prompt, num_predict=24, want_logits=True, format="json")
        assert J.viable(b"".join(pieces[t] for t in g.ids))
        ref = _oracle_json_greedy(m, prompt, len(g.ids), pieces, stops, "i16")
        for i, (tok, lp, margin, ml) in enumerate(ref[: len(g.ids)]):
            lg = e.last_logits(i)
            assert np.array_equal(np.isneginf(lg), np.isneginf(ml)), (seed, i)          # the same mask
            fin = np.isfinite(ml)
            assert np.abs(lg[fin] - ml[fin]).max() <= 2e-3 * np.abs(ml[fin]).max(), (seed, i)
            assert int(np.argmax(lg)) == int(g.ids[i])
            assert abs(float(g.logprobs[i]) - lp) <= 2e-2, (seed, i)
            compared += 1
            if int(g.ids[i]) != tok:
                assert margin <= 5e-2, (seed, i, margin)
                break
    assert compared >= 10
    e.close()


def test_json_document_ends_on_a_stop_token(tiny_gguf):
    """the first draw is '{' whatever the prompt ends with; a generation that ends on a stop token is a complete document"""
    e = _engine(tiny_gguf)
    pieces = _pieces(e)
    byte_tok = {p[0]: t for t, p in enumerate(pieces) if len(p) == 1}
    # the first token after the prompt is masked too: only '{' may start the output, whatever the prompt ends with
    prompt = np.array([byte_tok[c] for c in b'answer: {"a": '], np.int32)
    for seed in range(8):
        g = e.generate(prompt, num_predict=200, temperature=1.0, top_k=0, top_p=1.0, seed=seed, format="json")
        text = b"".join(pieces[t] for t in g.ids)
        assert text.startswith(b"{") and J.viable(text)
        if g.stats.done_reason == 0:
            assert J.complete(text) and isinstance(json.loads(text), dict)
    e.close()


def test_sampled_json_draws_never_take_a_masked_token(tiny_gguf):
    import penalty_oracle as PO
    e = _engine(tiny_gguf)
    pieces, stops = _pieces(e), _stops(e)
    rng = np.random.Generator(np.random.PCG64(23))
    prompt = rng.integers(0, e.info.n_vocab - 3, size=16)
    draws = 0
    for top_k, top_p, min_p in ((40, 0.95, 0.0), (0, 1.0, 0.0), (10, 1.0, 0.05), (1000, 0.5, 0.0)):
        for seed in range(6):
            kw = dict(num_predict=24, temperature=0.9, top_k=top_k, top_p=top_p, seed=seed, min_p=min_p, format="json")
            g = e.generate(prompt, want_logits=True, **kw)
            assert list(e.generate(prompt, **kw).ids) == list(g.ids)
            for i, t in enumerate(g.ids):
                lg = e.last_logits(i)
                assert J.mask(pieces, stops, list(g.ids[:i]))[t]
                assert np.array_equal(np.isneginf(lg), ~J.mask(pieces, stops, list(g.ids[:i])))
                assert PO.interval_error(lg, int(t), 0.9, top_k, top_p, seed, i, min_p=min_p) <= 1e-4, (top_k, seed, i)
                draws += 1
    assert draws > 150
    e.close()


def test_penalties_then_mask(tiny_gguf):
    import penalty_oracle as PO
    e = _engine(tiny_gguf, prefill_mode=1)
    pieces, stops = _pieces(e), _stops(e)
    prompt = np.random.Generator(np.random.PCG64(5)).integers(0, e.info.n_vocab - 3, size=30)
    pen = dict(repeat_penalty=1.4, repeat_last_n=-1, presence_penalty=0.3, frequency_penalty=0.2)
    e.generate(prompt, num_predict=1, ignore_eos=True, want_logits=True)
    u0 = e.last_logits(0)
    e.generate(prompt, num_predict=1, want_logits=True, format="json", **pen)
    assert np.array_equal(e.last_logits(0).view(np.uint32), J.apply_mask(PO.penalize(u0, prompt, **pen), pieces, stops, []).view(np.uint32))
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    g = e.generate(prompt, num_predict=16, want_logits=True, format="json", **pen)
    ref = _oracle_json_greedy(m, prompt, len(g.ids), pieces, stops, "i16", pen)
    for i, (tok, lp, margin, ml) in enumerate(ref[: len(g.ids)]):
        assert np.array_equal(np.isneginf(e.last_logits(i)), np.isneginf(ml)), i
        if int(g.ids[i]) != tok:
            assert margin <= 5e-2, (i, margin)
            break
    e.close()


def test_one_launch_more_per_draw_and_nothing_else_changes(tiny_gguf):
    e = _engine(tiny_gguf)
    prompt = np.random.Generator(np.random.PCG64(31)).integers(0, e.info.n_vocab - 3, size=20)
    a = e.generate(prompt, num_predict=6, ignore_eos=True)
    b = e.generate(prompt, num_predict=10, ignore_eos=True)
    per = (b.stats.kernel_launches - a.stats.kernel_launches) // 4
    base = a.stats.kernel_launches - 6 * per
    for samp in ({}, dict(temperature=0.8, top_k=40, top_p=0.9, seed=3)):
        g = e.generate(prompt, num_predict=12, format="json", **samp)
        assert g.stats.kernel_launches == base + max(g.stats.eval_count, 1) * (per + 1), samp
        # a request without format afterwards: the same bits as before any JSON request
        x = e.generate(prompt, num_predict=10, ignore_eos=True)
        assert np.array_equal(x.ids, b.ids) and np.array_equal(x.logprobs.view(np.uint32), b.logprobs.view(np.uint32))
        assert x.stats.kernel_launches == b.stats.kernel_launches
    e.close()


def test_refusals(tiny_gguf, tiny128_gguf, tmp_path, monkeypatch):
    from gridllm_b200 import native as N
    from oracle import gguf_synth as S
    e = _engine(tiny_gguf)
    prompt = np.arange(10, 30)
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=2, ignore_eos=True, format="json")
    assert ei.value.code == -1
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=2, format="json", stop_ids=[int(e.tokenize("a", add_bos=False)[0])])
    assert ei.value.code == -1
    so = N.SampleOpts()
    so.num_predict, so.format = 2, 7
    import ctypes as C
    ids = np.zeros(2, np.int32)
    lps = np.zeros(2, np.float32)
    st = N.GenStats()
    p = np.ascontiguousarray(prompt, dtype=np.int32)
    assert e._lib.gl_generate(e._h, N._i32p(p), len(p), C.byref(so), N.TOKEN_CB(), None, N._i32p(ids), N._f32p(lps), C.byref(st)) == -1
    e.close()
    # a SentencePiece vocabulary without a single-byte piece for '{'
    toks = ["<unk>", "<s>", "</s>"] + ["<0x%02X>" % b for b in range(256) if b != ord("{")]
    toks += ["▁w%d" % i for i in range(512 - len(toks))]
    types = [2, 3, 3] + [6] * 255 + [1] * (512 - 258)
    path = str(tmp_path / "spm_no_brace.gguf")
    S.build_model(path, S.LlamaShape("spm-no-brace", 2, 256, 4, 2, 512, 512, 10000.0, 1e-5, 512), "q8_0", seed=3,
                  spm_vocab={"tokens": toks, "scores": [0.0] * 3 + [0.0] * 255 + [-float(i) for i in range(512 - 258)], "types": types,
                             "bos": 1, "eos": 2, "unk": 0, "chat_template": None})
    s = _engine(path)
    with pytest.raises(N.NativeError) as ei:
        s.generate(prompt, num_predict=2, format="json")
    assert ei.value.code == -4 and "0x7B" in ei.value.detail
    assert len(s.generate(prompt, num_predict=2, ignore_eos=True).ids) == 2            # other requests are unaffected
    s.close()
    # the persistent decode kernel (in use: it refuses a sampled request as well)
    monkeypatch.setenv("GL_MEGA", "1")
    m = _engine(tiny128_gguf, prefill_mode=1)
    for kw in (dict(temperature=0.8, ignore_eos=True), dict(format="json")):
        with pytest.raises(N.NativeError) as ei:
            m.generate(prompt, num_predict=2, **kw)
        assert ei.value.code == -4, kw
    m.close()


def _drain(e, want):
    out = {s: ([], [], []) for s in want}
    guard = 0
    while any(len(out[s][0]) < want[s] for s in want):
        guard += 1
        assert guard < 10000
        for slot, tok, lp, done in e.batch_step():
            if slot in out and len(out[slot][0]) < want[slot]:
                out[slot][2].append(e.seq_logits(slot))
                out[slot][0].append(int(tok))
                out[slot][1].append(float(lp))
                if done and tok < 0:
                    want[slot] = len(out[slot][0])
    return out


@pytest.mark.parametrize("mode", [1, 2])
def test_batched_json(tiny128_gguf, mode):
    e = _engine(tiny128_gguf, max_batch=8, max_ctx=1024, batch_weights=mode)
    pieces, stops = _pieces(e), _stops(e)
    rng = np.random.Generator(np.random.PCG64(41))
    pa, pb, pc = (rng.integers(0, e.info.n_vocab - 3, size=k) for k in (40, 25, 5))      # pc: below the packed-prefill threshold
    N_TOK = 14
    js = dict(num_predict=N_TOK, format="json")

    s = e.seq_open(pa, num_predict=N_TOK, ignore_eos=True)
    alone_a = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    s = e.seq_open(pb, **js)
    alone_b = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    s = e.seq_open(pc, **js)                                                                 # the single-sequence open
    alone_c = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    slots = e.seq_open_many([pa, pb], [dict(num_predict=N_TOK, ignore_eos=True), js])
    sc = e.seq_open(pc, **js)
    got = _drain(e, {slots[0]: N_TOK, slots[1]: len(alone_b[0]), sc: len(alone_c[0])})
    a, b, c = got[slots[0]], got[slots[1]], got[sc]
    assert a[0] == alone_a[0] and np.array_equal(np.float32(a[1]), np.float32(alone_a[1]))
    assert all(np.array_equal(x, y) for x, y in zip(a[2], alone_a[2]))
    for mixed, alone in ((b, alone_b), (c, alone_c)):
        assert mixed[0] == alone[0]
        assert all(np.array_equal(x, y) for x, y in zip(mixed[2], alone[2]))
    for sl in (slots[0], slots[1], sc):
        e.seq_close(sl)
    # every draw of a JSON row is the argmax of the masked logits reported, and the output is a viable prefix
    for ids, lps, lgs in (alone_b, alone_c):
        real = [t for t in ids if t >= 0]
        assert J.viable(b"".join(pieces[t] for t in real))
        for i, lg in enumerate(lgs[: len(real)]):
            assert int(np.argmax(lg)) == ids[i]
            assert np.array_equal(np.isneginf(lg), ~J.mask(pieces, stops, real[:i]))
    # the same tokens as gl_generate with the same options, up to a near-tie between the two paths' arithmetic
    for p, (ids, _lps, _lgs) in ((pb, alone_b), (pc, alone_c)):
        g = e.generate(p, want_logits=True, **js)
        for i in range(min(len(g.ids), len([t for t in ids if t >= 0]))):
            if int(g.ids[i]) != ids[i]:
                lgi = e.last_logits(i)
                srt = np.sort(lgi)
                assert srt[-1] - srt[-2] <= 2e-2 * float(np.abs(lgi[np.isfinite(lgi)]).max()), (i, srt[-1] - srt[-2])
                break
    e.close()
