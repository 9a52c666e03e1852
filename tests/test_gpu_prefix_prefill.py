"""GPU: prompt passes from any position and of any length (the PAGED prompt attention of prefill_attn.cu reading the fp16 KV
pages), and gl_generate's opt-in prefix reuse (gl_engine_opts.prefix_cache).

Stated properties: a prompt prefilled in pieces gives the bits of the same prompt in one pass (last logits and the decode steps
that read the cache pages); against the exact-activation oracle, logits within 1e-2 * max|logit|, ids equal where the oracle's
top-1/top-2 margin > 5e-2; embeddings within 5e-3."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIXTURES = ["tiny_gguf", "tiny128_gguf"]          # head dim 64 (GQA 2:1) and 128 (GQA 4:1)


def _engine(path, **kw):
    from gridllm_b200 import native as N
    return N.Engine(path, **kw)


def _toks(m, seed, n):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, m.n_vocab - 3, size=n)


# ---- an all-positions restatement of the oracle's forward (exact activations, fp16 K / V), for prompts too long to step -------
def _forward_all(m, toks):
    """final residual rows [n][n_embd], per-layer rounded K / V rows, and the RoPE tables used (the oracle's arithmetic of
    LlamaOracle.hidden_step, every position at once)"""
    from oracle import llama_oracle as O
    H, KV, hd = m.n_head, m.n_head_kv, m.head_dim
    n = len(toks)
    ff = m.w("rope_freqs.weight").reshape(-1) if m.has("rope_freqs.weight") else None
    cos, sin = O.rope_table(n + 64, hd, m.rope_base, ff, getattr(m, "rope_linear", 1.0))
    c, s = cos[:n].astype(np.float64)[:, None, :], sin[:n].astype(np.float64)[:, None, :]

    def rope(v, nh):
        v = v.reshape(n, nh, hd // 2, 2)
        out = np.empty_like(v)
        out[..., 0] = v[..., 0] * c - v[..., 1] * s
        out[..., 1] = v[..., 0] * s + v[..., 1] * c
        return out.reshape(n, nh * hd)

    def f16(a):
        return a.astype(np.float32).astype(np.float16).astype(np.float64)

    def lin(name, a):
        return a @ m.w(name).astype(np.float64).T
    x = m.w("token_embd.weight")[np.asarray(toks)].astype(np.float64)
    upper = np.triu(np.ones((n, n), dtype=bool), 1)
    ks, vs = [], []
    for il in range(m.n_layer):
        p = f"blk.{il}."
        h = O.rmsnorm(x, m.w(p + "attn_norm.weight"), m.rms_eps)
        q = rope(lin(p + "attn_q.weight", h), H)
        k = f16(rope(lin(p + "attn_k.weight", h), KV))
        v = f16(lin(p + "attn_v.weight", h))
        ks.append(k)
        vs.append(v)
        att = np.empty((n, H * hd))
        for hh in range(H):
            kvh = hh // (H // KV)
            sc = q[:, hh * hd:(hh + 1) * hd] @ k[:, kvh * hd:(kvh + 1) * hd].T / np.sqrt(hd)
            sc[upper] = -np.inf
            sc -= sc.max(axis=1, keepdims=True)
            pw = np.exp(sc)
            pw /= pw.sum(axis=1, keepdims=True)
            att[:, hh * hd:(hh + 1) * hd] = pw @ v[:, kvh * hd:(kvh + 1) * hd]
            del sc, pw
        x = x + lin(p + "attn_output.weight", att)
        h2 = O.rmsnorm(x, m.w(p + "ffn_norm.weight"), m.rms_eps)
        x = x + lin(p + "ffn_down.weight", O.silu(lin(p + "ffn_gate.weight", h2)) * lin(p + "ffn_up.weight", h2))
    return x, ks, vs, (cos, sin)


def _oracle_after(m, toks, n_gen):
    """greedy continuation of `toks` by the oracle: the prompt through _forward_all, then LlamaOracle steps on its cache"""
    from oracle import llama_oracle as O
    x, ks, vs, (cos, sin) = _forward_all(m, toks)
    orc = O.LlamaOracle(m, act="exact", kv_f16=True)
    orc.cos, orc.sin = cos, sin
    KV, hd = m.n_head_kv, m.head_dim
    for il in range(m.n_layer):
        orc.k[il] = [r for r in ks[il]]
        orc.v[il] = [r for r in vs[il]]
    orc.pos = len(toks)
    logits = orc.logits_from_hidden(x[-1])
    ids, margins, all_logits = [], [], []
    for _ in range(n_gen):
        top = int(np.argmax(logits))
        srt = np.partition(logits, -2)[-2:]
        ids.append(top)
        margins.append(float(srt[1] - srt[0]))
        all_logits.append(logits)
        logits = orc.step(top)
    return {"ids": ids, "margins": margins, "logits": all_logits, "hidden": x}


def test_all_positions_restatement_equals_the_stepping_oracle(tiny_gguf):
    """the restatement above is the oracle's forward (checked where the stepping oracle is cheap)"""
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny_gguf)
    toks = _toks(m, 11, 40)
    orc = O.LlamaOracle(m, act="exact", kv_f16=True)
    for t in toks:
        ref = orc.step(int(t))
    got = _oracle_after(m, toks, 3)
    assert np.abs(got["logits"][0] - ref).max() <= 1e-9 * np.abs(ref).max()
    assert got["ids"] == [int(t) for t in O.LlamaOracle(m, act="exact", kv_f16=True).generate(toks, 3)["ids"]]


# ---- 1 / 2: pieces equal one pass, bit for bit; and the oracle ------------------------------------------------------------
SPLITS = [(8,), (37,), (64,), (128,), (200,), (292,), (37, 150)]      # cut points of a 300-token prompt; the last is three pieces


@pytest.mark.parametrize("fixture", FIXTURES)
def test_prompt_in_pieces_equals_one_pass(fixture, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    toks = _toks(m, 8100, 300)
    ref_e = _engine(path)
    one = ref_e.prefill(toks)
    nxt = [int(np.argmax(one))]
    steps = []
    for _ in range(3):
        lg, am, _ = ref_e.decode_step(nxt[-1])
        steps.append(lg)
        nxt.append(int(am))
    ref_e.close()
    orc = O.LlamaOracle(m, act="exact", kv_f16=True)
    for t in toks:
        ref = orc.step(int(t))
    scale = np.abs(ref).max()
    e = _engine(path)
    for cuts in SPLITS:
        e.kv_reset()
        bounds = [0, *cuts, len(toks)]
        assert all(b - a >= 8 for a, b in zip(bounds, bounds[1:]))          # every piece takes the tensor-core pass
        for a, b in zip(bounds, bounds[1:]):
            last = e.prefill(toks[a:b])
        assert e.position() == len(toks)
        assert np.array_equal(last, one), (fixture, cuts, np.abs(last - one).max())
        for i in range(3):
            lg, _, _ = e.decode_step(nxt[i])
            assert np.array_equal(lg, steps[i]), (fixture, cuts, "decode step", i)
        assert np.abs(last - ref).max() <= 1e-2 * scale, (fixture, cuts, np.abs(last - ref).max(), scale)
    e.close()


# ---- 3 / 4 / 5: longer than one pass ------------------------------------------------------------------------------------
N_LONG = 4400


@pytest.mark.timeout(900)
@pytest.mark.parametrize("fixture", FIXTURES)
def test_long_prompt_generate_seq_open_and_embed(fixture, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    toks = _toks(m, 8200, N_LONG)
    ref = _oracle_after(m, toks, 8)

    e = _engine(path, max_ctx=4608, max_batch=2)
    g = e.generate(toks, num_predict=8, ignore_eos=True, want_logits=True)
    assert g.stats.prompt_eval_count == N_LONG and g.stats.eval_count == 8
    kept = [e.last_logits(i) for i in range(8)]
    for i in range(8):
        assert np.isfinite(kept[i]).all()
        scale = np.abs(ref["logits"][i]).max()
        assert np.abs(kept[i] - ref["logits"][i]).max() <= 1e-2 * scale, (fixture, i, np.abs(kept[i] - ref["logits"][i]).max(), scale)
        if int(g.ids[i]) != ref["ids"][i]:
            assert ref["margins"][i] <= 5e-2, (fixture, i)
            break

    # gl_seq_open of the same prompt (longer than a pack: the single-sequence pass into the slot's pages): the same first
    # token from the same logits; later tokens come from the batched step's own arithmetic and agree except on near-ties
    slot = e.seq_open(toks, num_predict=8, ignore_eos=True)
    ids = []
    first_logits = None
    while len(ids) < 8:
        for s, tok, _lp, _done in e.batch_step():
            if s == slot and len(ids) < 8:
                if not ids:
                    first_logits = e.seq_logits(slot)
                ids.append(int(tok))
    e.seq_close(slot)
    assert ids[0] == int(g.ids[0]) and np.array_equal(first_logits, kept[0])
    for i in range(8):
        if ids[i] != int(g.ids[i]):
            srt = np.sort(kept[i])
            assert srt[-1] - srt[-2] <= 2e-2 * float(np.abs(kept[i]).max()), (fixture, "seq_open", i)
            break

    # gl_embed of the same sequence: passes of 4 096 rows, the pooling summed over them
    out, st = e.embed([toks])
    assert st.prompt_eval_count == N_LONG
    x = ref["hidden"]
    hs = O.rmsnorm(x, m.w("output_norm.weight"), m.rms_eps).mean(axis=0)
    emb = hs / np.linalg.norm(hs)
    assert np.abs(out[0] - emb).max() <= 5e-3, (fixture, np.abs(out[0] - emb).max())
    e.close()

    # the same prompt through the decode kernels, position by position (prefill_mode=1)
    es = _engine(path, max_ctx=4608, prefill_mode=1)
    gs = es.generate(toks, num_predict=1, ignore_eos=True, want_logits=True)
    ls = es.last_logits(0)
    es.close()
    assert gs.stats.prompt_eval_count == N_LONG
    assert np.abs(kept[0] - ls).max() <= 1e-2 * np.abs(ls).max(), (fixture, np.abs(kept[0] - ls).max())


# ---- 6: prefix reuse across gl_generate calls -----------------------------------------------------------------------------
def _gen(e, prompt, n, **kw):
    g = e.generate(prompt, num_predict=n, want_logits=True, **kw)
    return g, [e.last_logits(i) for i in range(len(g.ids))]


def _close_to_cold(g, lg, gc, lgc, tag):
    """within the decode-vs-prefill tolerance of a cold call, along the cold trajectory while the ids agree"""
    for i in range(min(len(g.ids), len(gc.ids))):
        scale = np.abs(lgc[i]).max()
        assert np.abs(lg[i] - lgc[i]).max() <= 1e-2 * scale, (tag, i, np.abs(lg[i] - lgc[i]).max(), scale)
        if int(g.ids[i]) != int(gc.ids[i]):
            srt = np.sort(lgc[i])
            assert srt[-1] - srt[-2] <= 5e-2, (tag, i)
            return


@pytest.mark.parametrize("fixture", FIXTURES)
def test_prefix_reuse(fixture, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    e = _engine(path, max_ctx=4096, prefix_cache=True)
    cold = _engine(path, max_ctx=4096)
    p = _toks(m, 8300, 120)

    # a repeated request: identical ids, logprobs and kept logits; only the last prefill_min (8) prompt tokens run again
    for kw in (dict(ignore_eos=True),
               dict(temperature=0.8, top_k=40, top_p=0.9, seed=7, repeat_penalty=1.3, presence_penalty=0.5, frequency_penalty=0.2),
               dict(format="json")):
        e.kv_reset()
        g1, l1 = _gen(e, p, 16, **kw)
        assert g1.stats.prompt_eval_count == 120
        g2, l2 = _gen(e, p, 16, **kw)
        assert g2.stats.prompt_eval_count == 8, kw
        assert np.array_equal(g1.ids, g2.ids) and np.array_equal(g1.logprobs, g2.logprobs), kw
        assert all(np.array_equal(a, b) for a, b in zip(l1, l2)), kw
        gc, lc = _gen(cold, p, 16, **kw)                   # ... and the cold engine's bits
        assert gc.stats.prompt_eval_count == 120
        assert np.array_equal(gc.ids, g2.ids) and all(np.array_equal(a, b) for a, b in zip(lc, l2)), kw

    # a context round trip: the previous prompt + its output + new tokens; the reused prefix reaches into generated tokens
    e.kv_reset()
    g1, _ = _gen(e, p, 12, ignore_eos=True)
    ctx = [int(t) for t in p] + [int(t) for t in g1.ids]
    p2 = ctx + [int(t) for t in _toks(m, 8301, 40)]
    g2, l2 = _gen(e, p2, 8, ignore_eos=True)
    # every generated id but the last draw was fed: r = 120 + 11
    assert g2.stats.prompt_eval_count == len(p2) - (120 + 11)
    gc, lc = _gen(cold, p2, 8, ignore_eos=True)
    assert gc.stats.prompt_eval_count == len(p2)
    _close_to_cold(g2, l2, gc, lc, (fixture, "context"))

    # a prompt that diverges at k reuses min(k, n - 8) positions -- a prefix from a prompt pass: the bits of a cold call
    for k in (30, 117):
        e.kv_reset()
        _gen(e, p, 4, ignore_eos=True)
        q = np.array(p)
        q[k] = (q[k] + 1) % (m.n_vocab - 3)
        g, lg = _gen(e, q, 6, ignore_eos=True)
        assert g.stats.prompt_eval_count == 120 - min(k, 120 - 8), k
        gc, lc = _gen(cold, q, 6, ignore_eos=True)
        assert np.array_equal(g.ids, gc.ids) and all(np.array_equal(a, b) for a, b in zip(lg, lc)), k

    # anything else that writes the pages in between: no reuse
    for between in (lambda: e.kv_reset(), lambda: e.prefill(_toks(m, 8302, 20)), lambda: e.embed([_toks(m, 8303, 2100)]),
                    lambda: e.decode_step(5)):
        e.kv_reset()
        _gen(e, p, 4, ignore_eos=True)
        between()
        g, lg = _gen(e, p, 4, ignore_eos=True)
        assert g.stats.prompt_eval_count == 120
        gc, lc = _gen(cold, p, 4, ignore_eos=True)
        assert np.array_equal(g.ids, gc.ids) and all(np.array_equal(a, b) for a, b in zip(lg, lc))

    # a request cancelled from the callback, then continued with its context
    e.kv_reset()
    seen = []
    g1 = e.generate(p, num_predict=16, ignore_eos=True, on_token=lambda tid, lp, piece: seen.append(tid) or len(seen) >= 5)
    assert len(g1.ids) == 5 and g1.stats.done_reason == 2
    p3 = [int(t) for t in p] + [int(t) for t in g1.ids] + [int(t) for t in _toks(m, 8304, 20)]
    g3, l3 = _gen(e, p3, 8, ignore_eos=True)
    assert g3.stats.prompt_eval_count == 20                 # the five reported ids were all fed; the steps past them are not claimed
    gc, lc = _gen(cold, p3, 8, ignore_eos=True)
    _close_to_cold(g3, l3, gc, lc, (fixture, "cancelled"))

    # a default engine evaluates the whole prompt on a repeat
    gc1, _ = _gen(cold, p, 4, ignore_eos=True)
    gc2, _ = _gen(cold, p, 4, ignore_eos=True)
    assert gc1.stats.prompt_eval_count == gc2.stats.prompt_eval_count == 120
    e.close()
    cold.close()
