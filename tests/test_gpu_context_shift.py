"""GPU, end to end: the context shift (gl_engine_opts context_shift; rule in include/gridllm_native.h) on tiny models with a
64-token context, with generations that cross the window at least twice.

Bars: greedy gl_generate against the oracle with the same shifts (tests/shift_oracle.py) within the decode bars of
tests/test_gpu_decode.py (logits 2e-3 * max|logit| of the i16 oracle, logprob 2e-2, ids equal where the margin is > 5e-2);
penalised, JSON-masked and sampled draws keep the bars of the penalty / JSON / sampler tests across a shift, with the whole
history (discarded ids included) penalised; an over-long prompt gives the bits of the explicitly cut prompt with the option off;
batch slots shift bit-identically alone and beside other rows and stay within the batched bar of the oracle (1e-2 * max|logit|
of the exact oracle); shifting sequences neither share nor index prefix pages; the prefix_cache record keeps [0, k) only;
GL_MEGA=1 refuses a shift; and requests that fit give the bits of the option off."""
import numpy as np
import pytest

import shift_oracle as SO

pytestmark = pytest.mark.gpu

W = 64


def _engine(path, **kw):
    from gridllm_b200 import native as N
    return N.Engine(path, max_ctx=W, **kw)


def _prompt(m, n, seed):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, m.n_vocab - 3, size=n)


def _compare(ref, g, e, bar, tag):
    """per-step logits / logprobs / ids of a generation against an oracle run; returns the steps compared"""
    for i in range(len(g.ids)):
        lg = e.last_logits(i) if e is not None else g.logits[i]
        ml = ref["logits"][i]
        fin = np.isfinite(ml)
        assert np.array_equal(np.isfinite(lg), fin), (tag, i)
        scale = float(np.abs(ml[fin]).max())
        err = float(np.abs(lg[fin] - ml[fin]).max())
        assert err <= bar * scale, (tag, "logits", i, err, scale)
        assert abs(float(g.logprobs[i]) - float(ref["logprobs"][i])) <= 2e-2, (tag, "logprob", i)
        if int(g.ids[i]) != int(ref["ids"][i]):
            assert ref["margins"][i] <= 5e-2, (tag, "id", i, ref["margins"][i])
            return i + 1
    return len(g.ids)


@pytest.mark.parametrize("fixture", ["tiny_gguf", "tiny128_gguf"])
@pytest.mark.parametrize("keep,n_prompt,n_pred", [(4, 50, 60), (0, 40, 64), (17, 30, 64)])
def test_greedy_generate_follows_the_oracle_across_shifts(fixture, keep, n_prompt, n_pred, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    e = _engine(path, prefill_mode=1, context_shift=True)       # every position through the decode kernels
    prompt = _prompt(m, n_prompt, 500 + keep)
    g = e.generate(prompt, num_predict=n_pred, ignore_eos=True, want_logits=True, num_keep=keep)
    assert g.stats.eval_count == n_pred and g.stats.done_reason == 1
    ref = SO.greedy_with_shifts(O.LlamaOracle(m, act="i16", kv_f16=True), prompt, n_pred, W, keep)
    assert ref["shifts"] >= 2
    assert _compare(ref, g, e, 2e-3, (fixture, keep)) >= 1
    # the same request again: bit-identical (the shift is deterministic)
    again = e.generate(prompt, num_predict=n_pred, ignore_eos=True, num_keep=keep)
    assert np.array_equal(again.ids, g.ids) and np.array_equal(again.logprobs.view(np.uint32), g.logprobs.view(np.uint32))
    e.close()


def _oracle_penalised(m, prompt, n_pred, keep, pen, pieces=None, stops=None):
    """greedy with shifts, penalties over the whole history (prompt, then every generated id) and the JSON mask"""
    from oracle import llama_oracle as O
    import json_oracle as J
    import penalty_oracle as P
    orc = O.LlamaOracle(m, act="i16", kv_f16=True)
    d = SO.discard(W, keep)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    ids, lps, margins, kept = [], [], [], []
    shifts = 0
    for i in range(n_pred):
        lg = P.penalize(logits.astype(np.float32), list(prompt) + ids, **pen).astype(np.float64)
        if pieces is not None:
            lg = J.apply_mask(lg, pieces, stops, ids)
        fin = lg[np.isfinite(lg)]
        top = int(np.argmax(lg))
        srt = np.partition(fin, -2)[-2:]
        lse = fin.max() + np.log(np.exp(fin - fin.max()).sum())
        ids.append(top)
        lps.append(float(lg[top] - lse))
        margins.append(float(srt[1] - srt[0]))
        kept.append(lg)
        if i == n_pred - 1 or (stops and top in stops):
            break
        if orc.pos == W:
            SO.shift(orc, keep, d)
            shifts += 1
        logits = orc.step(top)
    return {"ids": ids, "logprobs": lps, "margins": margins, "logits": kept, "shifts": shifts}


def test_penalised_greedy_follows_the_oracle_across_shifts(tiny_gguf):
    """the penalty history keeps the discarded ids: prompt, then every generated id"""
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    e = _engine(tiny_gguf, prefill_mode=1, context_shift=True)
    pen = dict(repeat_penalty=1.3, repeat_last_n=-1, presence_penalty=0.4, frequency_penalty=0.2)
    prompt = _prompt(m, 44, 901)
    g = e.generate(prompt, num_predict=64, ignore_eos=True, want_logits=True, num_keep=4, **pen)
    ref = _oracle_penalised(m, prompt, 64, 4, pen)
    assert ref["shifts"] >= 2
    assert _compare(ref, g, e, 2e-3, "penalised") >= 10
    e.close()


def test_sampled_and_json_draws_across_shifts(tiny_gguf):
    import json_oracle as J
    import penalty_oracle as S
    e = _engine(tiny_gguf, context_shift=True)
    n = e.info.n_vocab
    pieces = [e.token_piece(t) for t in range(n)]
    stops = [s for s in (e.info.eos_id, e.info.eot_id) if s >= 0]
    rng = np.random.Generator(np.random.PCG64(77))
    prompt = rng.integers(0, n - 3, size=40)
    # sampled with penalties and min_p: every draw inside the oracle's interval of the logits it was drawn from, replays equal
    kw = dict(num_predict=64, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.95, seed=11, min_p=0.05,
              repeat_penalty=1.3, repeat_last_n=64, frequency_penalty=0.2, num_keep=4)
    g = e.generate(prompt, want_logits=True, **kw)
    assert g.stats.eval_count == 64
    again = e.generate(prompt, **kw)
    assert list(g.ids) == list(again.ids)
    for i in range(len(g.ids)):
        assert S.interval_error(e.last_logits(i), int(g.ids[i]), 0.8, 40, 0.95, 11, i, min_p=0.05) <= 1e-4, i
    # format json, sampled: the mask continues across the shift (same automaton state), the output stays a viable document
    crossed = 0
    for seed in range(6):
        p = rng.integers(0, n - 3, size=W - 2)            # the first shift comes at the fourth draw
        gj = e.generate(p, num_predict=48, temperature=1.0, top_k=0, top_p=1.0, seed=seed, format="json", want_logits=True,
                        num_keep=4)
        ids = [int(t) for t in gj.ids]
        assert J.viable(b"".join(pieces[t] for t in ids)), seed
        for i in range(len(ids)):
            lg = e.last_logits(i)
            want = J.mask(pieces, stops, ids[:i])
            assert np.array_equal(np.isfinite(lg), want), (seed, i)
            assert S.interval_error(lg, ids[i], 1.0, 0, 1.0, seed, i) <= 1e-4, (seed, i)
        crossed += len(ids) > 3
    assert crossed >= 1
    e.close()


@pytest.mark.parametrize("fixture", ["tiny_gguf", "tiny128_gguf"])
@pytest.mark.parametrize("keep", [4, 0, -1, 20])
def test_prompt_cut_is_the_explicitly_cut_prompt(fixture, keep, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    on = _engine(path, context_shift=True)
    off = _engine(path)
    for n_prompt in (W, W + 1, 3 * W + 5):
        prompt = _prompt(m, n_prompt, 40 + n_prompt)
        k = SO.keep_count(keep, n_prompt, W)
        d = SO.discard(W, k)
        cut = SO.cut_prompt(prompt, W, k)
        assert len(cut) == W - d
        n_pred = d
        g = on.generate(prompt, num_predict=n_pred, ignore_eos=True, num_keep=keep)
        r = off.generate(cut, num_predict=n_pred, ignore_eos=True)
        assert np.array_equal(g.ids, r.ids) and np.array_equal(g.logprobs.view(np.uint32), r.logprobs.view(np.uint32)), (n_prompt, keep)
        assert g.stats.prompt_eval_count == W - d
    # requests that fit give the bits of the option off
    prompt = _prompt(m, 20, 5)
    for kw in (dict(), dict(temperature=0.9, top_k=40, seed=3), dict(repeat_penalty=1.2, repeat_last_n=64)):
        g = on.generate(prompt, num_predict=W - 20, ignore_eos=True, num_keep=keep, **kw)
        r = off.generate(prompt, num_predict=W - 20, ignore_eos=True, **kw)
        assert np.array_equal(g.ids, r.ids) and np.array_equal(g.logprobs.view(np.uint32), r.logprobs.view(np.uint32))
    on.close()
    off.close()


def test_generate_bounds_and_refusals(tiny_gguf):
    from gridllm_b200 import native as N
    e = _engine(tiny_gguf, context_shift=True)
    prompt = np.arange(10, 30, dtype=np.int32)
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=W + 1, ignore_eos=True)
    assert ei.value.code == -9
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=8, ignore_eos=True, num_keep=-2)
    assert ei.value.code == -1
    assert e.generate(prompt, num_predict=W, ignore_eos=True).stats.eval_count == W
    e.close()
    # the option off: the word is not read (garbage in num_keep changes nothing), a sequence past the context still fails
    off = _engine(tiny_gguf)
    a = off.generate(prompt, num_predict=8, ignore_eos=True, num_keep=-12345)
    b = off.generate(prompt, num_predict=8, ignore_eos=True)
    assert np.array_equal(a.ids, b.ids)
    with pytest.raises(N.NativeError) as ei:
        off.generate(prompt, num_predict=W, ignore_eos=True)
    assert ei.value.code == -9
    off.close()


def _drain(e, want, logits=None):
    out = {s: ([], []) for s in want}
    guard = 0
    while any(len(out[s][0]) < want[s] for s in want):
        guard += 1
        assert guard < 10000
        for slot, tok, lp, done in e.batch_step():
            if slot in out and len(out[slot][0]) < want[slot]:
                if logits is not None:
                    logits.setdefault(slot, []).append(e.seq_logits(slot))
                out[slot][0].append(int(tok))
                out[slot][1].append(float(lp))
    return out


@pytest.mark.parametrize("fixture", ["tiny_gguf", "tiny128_gguf"])
def test_batch_slots_shift(fixture, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    e = _engine(path, max_batch=8, context_shift=True)
    p0 = _prompt(m, 40, 1)
    # alone
    s = e.seq_open(p0, num_predict=64, ignore_eos=True, num_keep=4)
    lg = {}
    alone = _drain(e, {s: 64}, lg)[s]
    e.seq_close(s)
    ref = SO.greedy_with_shifts(O.LlamaOracle(m, act="exact", kv_f16=True), p0, 64, W, 4)
    assert ref["shifts"] >= 2

    class G:
        ids, logprobs, logits = np.array(alone[0]), np.array(alone[1], np.float32), lg[s]
    assert _compare(ref, G, None, 1e-2, (fixture, "batched")) >= 8
    # beside rows that do not shift and rows that shift in the same steps (same prompt length: same window crossings)
    others = [_prompt(m, 12, 2), _prompt(m, 40, 3), _prompt(m, 40, 4)]
    slots = e.seq_open_many([p0] + others, [dict(num_predict=64, ignore_eos=True, num_keep=4),
                                            dict(num_predict=40, ignore_eos=True, num_keep=4),
                                            dict(num_predict=64, ignore_eos=True, num_keep=4),
                                            dict(num_predict=64, ignore_eos=True, num_keep=0)])
    assert min(slots) >= 0
    got = _drain(e, {sl: (64 if i != 1 else 40) for i, sl in enumerate(slots)})
    assert got[slots[0]][0] == alone[0]
    assert np.array_equal(np.array(got[slots[0]][1], np.float32).view(np.uint32), np.array(alone[1], np.float32).view(np.uint32))
    for sl in slots:
        e.seq_close(sl)
    for i, p in enumerate(others, 1):
        o = dict(num_predict=64 if i != 1 else 40, ignore_eos=True, num_keep=0 if i == 3 else 4)
        sl = e.seq_open(p, **o)
        a = _drain(e, {sl: o["num_predict"]})[sl]
        assert a[0] == got[slots[i]][0], i
        e.seq_close(sl)
    e.close()


def test_batch_prefix_cache_skips_shifting_sequences(tiny_gguf):
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    base = _prompt(m, 40, 9)
    plain = _engine(tiny_gguf, max_batch=8, context_shift=True)
    s = plain.seq_open(base, num_predict=50, ignore_eos=True, num_keep=4)
    want = _drain(plain, {s: 50})[s]
    plain.close()
    e = _engine(tiny_gguf, max_batch=8, context_shift=True, batch_prefix_cache=True)
    # a shifting sequence: the bits of the engine without sharing, nothing shared, nothing indexed
    s = e.seq_open(base, num_predict=50, ignore_eos=True, num_keep=4)
    assert _drain(e, {s: 50})[s] == want
    e.seq_close(s)
    assert e.batch_counters()["shared_tokens"] == 0
    s2 = e.seq_open(base, num_predict=8, ignore_eos=True)        # fits: would share an indexed prefix if there were one
    _drain(e, {s2: 8})
    e.seq_close(s2)
    assert e.batch_counters()["shared_tokens"] == 0
    # a fitting sequence is indexed and shared as before, but never by a shifting one
    s3 = e.seq_open(base, num_predict=8, ignore_eos=True)
    _drain(e, {s3: 8})
    e.seq_close(s3)
    shared = e.batch_counters()["shared_tokens"]
    assert shared > 0
    s4 = e.seq_open(base, num_predict=50, ignore_eos=True, num_keep=4)
    assert _drain(e, {s4: 50})[s4] == want
    assert e.batch_counters()["shared_tokens"] == shared
    e.close()


def test_prefix_cache_record_after_a_shift(tiny_gguf):
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    e = _engine(tiny_gguf, prefix_cache=True, context_shift=True)
    prompt = _prompt(m, 40, 12)
    g = e.generate(prompt, num_predict=50, ignore_eos=True, num_keep=4)
    again = e.generate(prompt, num_predict=8, ignore_eos=True, num_keep=4)
    assert again.stats.prompt_eval_count >= len(prompt) - 4
    cold = _engine(tiny_gguf, context_shift=True).generate(prompt, num_predict=8, ignore_eos=True, num_keep=4)
    assert np.array_equal(again.ids, cold.ids)
    assert len(g.ids) == 50
    e.close()


def test_mega_refuses_a_shift(tiny128_gguf, monkeypatch):
    from gridllm_b200 import native as N
    monkeypatch.setenv("GL_MEGA", "1")
    e = _engine(tiny128_gguf, prefill_mode=1, context_shift=True)
    prompt = np.arange(10, 50, dtype=np.int32)
    with pytest.raises(N.NativeError) as ei:
        e.generate(prompt, num_predict=40, ignore_eos=True, num_keep=4)
    assert ei.value.code == -4
    with pytest.raises(N.NativeError) as ei:
        e.generate(np.arange(10, 10 + W + 3, dtype=np.int32), num_predict=4, ignore_eos=True, num_keep=4)
    assert ei.value.code == -4
    assert e.generate(prompt, num_predict=W - 40, ignore_eos=True).stats.eval_count == W - 40      # fits: runs as before
    e.close()
