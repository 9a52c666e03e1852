"""GPU: repetition / presence / frequency penalties (gridllm_b200/csrc/penalty.cu) and min_p (sampler.cu) against
the CPU restatement in tests/penalty_oracle.py, through the C ABI.

Stated bars: the penalty kernel is bit-identical to penalty_oracle.penalize (single fp32 operations, no contraction); a
penalised greedy gl_generate follows the oracle's penalised greedy loop with the decode tolerances of tests/test_gpu_decode.py
(ids equal wherever the penalised top-1/top-2 margin > 5e-2, logits within 2e-3 * max|logit| of the i16 oracle, logprob within
2e-2); sampled requests with min_p and penalties draw inside the oracle's interval to 1e-4 of the kept mass.  A request whose
penalty fields are all off replays exactly what it replayed before (same bits, same kernel launches), and unpenalised rows of a
batch are bit-identical whether or not a penalised row shares the step."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PEN = dict(repeat_penalty=1.3, repeat_last_n=64)


def _engine(path, **kw):
    from gridllm_b200 import native as N
    return N.Engine(path, **kw)


def _raw_generate(e, prompt, n, **fields):
    """gl_generate with a SampleOpts built field by field (fields not named stay zero, as a caller unaware of them sends)"""
    from gridllm_b200 import native as N
    p = np.ascontiguousarray(prompt, dtype=np.int32)
    so = N.SampleOpts()
    so.num_predict, so.ignore_eos, so.top_p = n, 1, 1.0
    for k, v in fields.items():
        setattr(so, k, v)
    ids, lps, st = np.zeros(n, np.int32), np.zeros(n, np.float32), N.GenStats()
    N._check(e._lib.gl_generate(e._h, N._i32p(p), len(p), C.byref(so), N.TOKEN_CB(), None, N._i32p(ids), N._f32p(lps), C.byref(st)))
    return ids[: st.eval_count].copy(), lps[: st.eval_count].copy(), st


def test_penalize_logits_is_bit_identical_to_the_oracle(tiny_gguf):
    import penalty_oracle as S
    e = _engine(tiny_gguf)
    n = e.info.n_vocab
    rng = np.random.Generator(np.random.PCG64(17))
    cases = 0
    for last_n in (1, 64, 1000, -1):
        for h_len, id_range in ((1, n), (50, 8), (700, n), (2500, 40)):
            hist = rng.integers(0, id_range, h_len)
            hist[:: max(1, h_len // 3)] = n - 1                    # both ends of the vocabulary, counts up to the window
            hist[1::7] = 0
            for rp, pp, fp in ((1.3, 0.0, 0.0), (0.7, 0.25, 0.5), (1.0, -0.5, 1.7), (2.0, 0.1, 0.03), (0.0, 0.0, 0.2)):
                logits = (rng.standard_normal(n) * 4).astype(np.float32)
                logits[rng.integers(0, n, 10)] = 0.0
                got = e.penalize_logits(logits, hist, rp, last_n, pp, fp)
                ref = S.penalize(logits, hist, rp, last_n, pp, fp)
                assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (last_n, h_len, rp, pp, fp)
                cases += 1
    # off: window 0, or nothing active
    logits = (rng.standard_normal(n)).astype(np.float32)
    assert np.array_equal(e.penalize_logits(logits, [1, 2, 3], 1.3, 0, 0.5, 0.5), logits)
    assert np.array_equal(e.penalize_logits(logits, [1, 2, 3], 1.0, 64, 0.0, 0.0), logits)
    # the scratch is left clean: the same call twice gives the same bits
    hist = rng.integers(0, 30, 300)
    a = e.penalize_logits(logits, hist, 1.5, -1, 0.2, 0.3)
    assert np.array_equal(a, e.penalize_logits(logits, hist, 1.5, -1, 0.2, 0.3))
    assert cases == 80
    e.close()


def test_invalid_penalty_options_are_refused(tiny_gguf):
    from gridllm_b200 import native as N
    e = _engine(tiny_gguf)
    prompt = np.arange(10, 30)
    for bad in (dict(repeat_penalty=-1.0), dict(repeat_last_n=-2), dict(min_p=1.5), dict(min_p=-0.1), dict(presence_penalty=float("nan")),
                dict(frequency_penalty=float("inf"))):
        with pytest.raises(N.NativeError) as ei:
            e.generate(prompt, num_predict=2, ignore_eos=True, **bad)
        assert ei.value.code == -1, bad
    e.close()


def _oracle_penalised(m, prompt, n, act, **pen):
    import penalty_oracle as S
    from oracle import llama_oracle as O
    orc = O.LlamaOracle(m, act=act, kv_f16=True)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    hist, out = [int(t) for t in prompt], []
    for _ in range(n):
        pl = S.penalize(logits, hist, **pen)
        tok = int(np.argmax(pl))
        srt = np.sort(pl)
        lse = float(pl.max()) + float(np.log(np.exp(pl.astype(np.float64) - pl.max()).sum()))
        out.append((tok, float(pl[tok]) - lse, float(srt[-1] - srt[-2]), pl))
        hist.append(tok)
        logits = orc.step(tok)
    return out


@pytest.mark.parametrize("prefill_mode", [1, 0])
def test_penalised_greedy_generate_follows_the_oracle(tiny_gguf, prefill_mode):
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    e = _engine(tiny_gguf, prefill_mode=prefill_mode)
    # sequential prefill: every position through the decode kernels (2e-3 of the i16 oracle); batched prefill: the tensor-core
    # prompt pass (1e-2 of exact activations), as in test_gpu_decode.py
    act, tol = ("i16", 2e-3) if prefill_mode == 1 else ("exact", 1e-2)
    compared = 0
    for seed in (1000, 1001, 1002):
        prompt = np.random.Generator(np.random.PCG64(seed)).integers(0, m.n_vocab - 3, size=24)
        g = e.generate(prompt, num_predict=16, ignore_eos=True, want_logits=True, **PEN)
        assert g.stats.eval_count == 16
        ref = _oracle_penalised(m, prompt, 16, act, **PEN)
        for i, (tok, lp, margin, pl) in enumerate(ref):
            lg = e.last_logits(i)
            assert int(np.argmax(lg)) == int(g.ids[i])             # the token is drawn from the penalised logits reported
            assert np.abs(lg - pl).max() <= tol * np.abs(pl).max(), (seed, i, np.abs(lg - pl).max())
            assert abs(float(g.logprobs[i]) - lp) <= 2e-2, (seed, i)
            compared += 1
            if int(g.ids[i]) != tok:
                assert margin <= 5e-2, (seed, i, margin)
                break
    assert compared >= 3
    e.close()


def test_first_token_is_penalised_bit_exactly(tiny_gguf):
    """step 0's logits of a penalised request = penalize(step 0's logits of the same request without penalties, prompt)"""
    import penalty_oracle as S
    for mode in (0, 1):
        e = _engine(tiny_gguf, prefill_mode=mode)
        prompt = np.random.Generator(np.random.PCG64(5)).integers(0, e.info.n_vocab - 3, size=30)
        prompt[::4] = 7
        e.generate(prompt, num_predict=1, ignore_eos=True, want_logits=True)
        u0 = e.last_logits(0)
        pen = dict(repeat_penalty=1.4, repeat_last_n=-1, presence_penalty=0.3, frequency_penalty=0.2)
        e.generate(prompt, num_predict=1, ignore_eos=True, want_logits=True, **pen)
        assert np.array_equal(e.last_logits(0), S.penalize(u0, prompt, **pen)), mode
        e.close()


def test_sampled_requests_with_min_p_and_penalties(tiny_gguf):
    import penalty_oracle as S
    e = _engine(tiny_gguf)
    n = e.info.n_vocab
    rng = np.random.Generator(np.random.PCG64(23))
    # the sampler alone: min_p cuts the candidates (both top-k kernels)
    for scale in (1.0, 3.0):
        logits = (rng.standard_normal(n) * scale).astype(np.float32)
        for t, k, p, mp in ((0.8, 40, 0.95, 0.05), (1.0, 0, 1.0, 0.1), (1.5, 64, 0.9, 0.3), (0.7, 500, 1.0, 0.02), (1.0, 10, 1.0, 1.0)):
            for seed in range(6):
                got, lp = e.sample_logits(logits, t, k, p, seed, seed, min_p=mp)
                assert S.interval_error(logits, got, t, k, p, seed, seed, min_p=mp) <= 1e-4, (t, k, p, mp, seed)
    # whole requests: penalties and min_p together, every draw inside the oracle's interval of its (penalised) logits
    prompt = rng.integers(0, n - 3, size=24)
    for top_k in (40, 0):
        kw = dict(num_predict=20, ignore_eos=True, temperature=0.8, top_k=top_k, top_p=0.95, seed=11, min_p=0.05,
                  repeat_penalty=1.3, repeat_last_n=64, frequency_penalty=0.2)
        g = e.generate(prompt, want_logits=True, **kw)
        again = e.generate(prompt, **kw)
        assert list(g.ids) == list(again.ids)
        for i in range(len(g.ids)):
            lg = e.last_logits(i)
            assert S.interval_error(lg, int(g.ids[i]), 0.8, top_k, 0.95, 11, i, min_p=0.05) <= 1e-4, (top_k, i)
    e.close()


def test_off_values_change_nothing(tiny_gguf):
    e = _engine(tiny_gguf)
    prompt = np.random.Generator(np.random.PCG64(31)).integers(0, e.info.n_vocab - 3, size=20)
    for samp in ({}, dict(temperature=0.8, top_k=40, top_p=0.9, seed=3)):
        zero_ids, zero_lps, zero_st = _raw_generate(e, prompt, 12, **samp)                  # penalty fields zeroed
        for off in (dict(repeat_penalty=1.0, repeat_last_n=64), dict(repeat_penalty=1.3, repeat_last_n=0),
                    dict(repeat_penalty=0.0, repeat_last_n=-1, presence_penalty=0.0, frequency_penalty=0.0, min_p=0.0)):
            ids, lps, st = _raw_generate(e, prompt, 12, **samp, **off)
            assert np.array_equal(ids, zero_ids) and np.array_equal(lps.view(np.uint32), zero_lps.view(np.uint32)), (samp, off)
            assert st.kernel_launches == zero_st.kernel_launches
        # a penalised request runs one kernel more per token
        ids, lps, st = _raw_generate(e, prompt, 12, **samp, repeat_penalty=1.3, repeat_last_n=64)
        assert st.kernel_launches == zero_st.kernel_launches + st.eval_count
    e.close()


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
    return out


@pytest.mark.parametrize("mode", [1, 2])
def test_batched_penalties(tiny128_gguf, mode):
    import penalty_oracle as S
    e = _engine(tiny128_gguf, max_batch=8, max_ctx=1024, batch_weights=mode)
    rng = np.random.Generator(np.random.PCG64(41))
    pa, pb, pc = (rng.integers(0, e.info.n_vocab - 3, size=k) for k in (40, 25, 5))     # pc: below the packed-prefill threshold
    pen = dict(repeat_penalty=1.3, repeat_last_n=64, presence_penalty=0.1)
    N_TOK = 14

    # unpenalised row alone, then beside penalised rows: bit-identical tokens, logprobs and logits
    s = e.seq_open(pa, num_predict=N_TOK, ignore_eos=True)
    alone_a = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    # penalised sequence alone (gl_seq_open) ...
    s = e.seq_open(pb, num_predict=N_TOK, ignore_eos=True, **pen)
    alone_b = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    s = e.seq_open(pc, num_predict=N_TOK, ignore_eos=True, **pen)                      # the single-sequence open
    alone_c = _drain(e, {s: N_TOK})[s]
    e.seq_close(s)
    # ... in one gl_seq_open_many with the unpenalised one, and in a mixed batch
    slots = e.seq_open_many([pa, pb], [dict(num_predict=N_TOK, ignore_eos=True), dict(num_predict=N_TOK, ignore_eos=True, **pen)])
    sc = e.seq_open(pc, num_predict=N_TOK, ignore_eos=True, **pen)
    got = _drain(e, {slots[0]: N_TOK, slots[1]: N_TOK, sc: N_TOK})
    a, b, c = got[slots[0]], got[slots[1]], got[sc]
    assert a[0] == alone_a[0] and np.array_equal(np.float32(a[1]), np.float32(alone_a[1]))
    assert all(np.array_equal(x, y) for x, y in zip(a[2], alone_a[2]))
    for mixed, alone in ((b, alone_b), (c, alone_c)):
        assert mixed[0] == alone[0]
        assert all(np.array_equal(x, y) for x, y in zip(mixed[2], alone[2]))
    for sl in (slots[0], slots[1], sc):
        e.seq_close(sl)
    # every draw of a penalised (greedy) row is the argmax of the penalised logits gl_seq_logits reports
    for ids, lps, lgs in (alone_b, alone_c):
        for i, lg in enumerate(lgs):
            assert int(np.argmax(lg)) == ids[i]
    # same tokens as gl_generate with the same options, up to a near-tie between the two paths' arithmetic
    for p, (ids, _lps, _lgs) in ((pb, alone_b), (pc, alone_c)):
        g = e.generate(p, num_predict=N_TOK, ignore_eos=True, want_logits=True, **pen)
        for i in range(N_TOK):
            if int(g.ids[i]) != ids[i]:
                lgi = e.last_logits(i)
                srt = np.sort(lgi)
                assert srt[-1] - srt[-2] <= 2e-2 * float(np.abs(lgi).max()), (i, srt[-1] - srt[-2])
                break
    # the first token of a penalised open is drawn from penalised logits: penalise the unpenalised open's first logits
    s = e.seq_open(pb, num_predict=2, ignore_eos=True)
    u0 = e.seq_logits(s)
    e.seq_close(s)
    s = e.seq_open(pb, num_predict=2, ignore_eos=True, **pen)
    assert np.array_equal(e.seq_logits(s), S.penalize(u0, pb, **pen))
    e.seq_close(s)
    e.close()
