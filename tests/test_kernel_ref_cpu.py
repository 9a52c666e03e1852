"""CPU: the float64 kernel references (tests/kernel_ref.py) pinned against the oracle where they overlap, and evidence that
the GPU kernel checks (tests/test_gpu_kernels.py) have teeth: on the very inputs of every GPU case, each named mutant of the
reference -- the kind of bug a kernel could have -- differs from the true reference by at least four times that case's
tolerance.  A mutant is only applied where it changes the operation at all (a shifted mask needs a key past the row, or
before it; dropping the last KV tile needs a row with two tiles; h % n_kv differs from h // group only with more than one
KV head and a group above one).  Errors are measured
on a subset of the rows the GPU test compares, which can only understate a mutant's distance."""
import ctypes

import numpy as np
import pytest

import kernel_cases as KC
import kernel_ref as R

MARGIN = 4.0


def _gemm_distance(mut, ref, bound, extra=0.0, relb=R.GEMM_REL_L2):
    if not np.isfinite(mut).all():
        return np.inf
    ratio, rl2 = R.gemm_check(mut, ref, bound, extra)
    return max(ratio, rl2 / relb)


def _attn_distance(mut, ref, v, n_head, n_kv, hd):
    if not np.isfinite(mut).all():
        return np.inf
    ratio, rl2 = R.attention_check(mut, ref, v, n_head, n_kv, hd)
    return max(ratio, rl2 / R.ATTN_REL_L2)


# ---- pins against the oracle --------------------------------------------------------------------------------------------
def test_rope_pairing_matches_the_oracle():
    from oracle import llama_oracle as O
    rng = np.random.Generator(np.random.PCG64(3))
    for hd in (64, 128):
        cos_t, sin_t = O.rope_table(300, hd, 500000.0)
        x = rng.standard_normal((5, 4 * hd))
        pos = np.array([0, 1, 17, 200, 299])
        got = R.rope_rows(x, pos, cos_t, sin_t, hd)
        for i, p in enumerate(pos):
            assert np.array_equal(got[i], O.apply_rope(x[i], int(p), 4, hd, cos_t, sin_t))


def test_attention_matches_the_oracle_step():
    """one query at a time, the way llama_oracle.LlamaOracle.hidden_step attends over its cache"""
    rng = np.random.Generator(np.random.PCG64(4))
    n_head, n_kv, hd, pos0, L = 8, 2, 64, 37, 20
    q, k, v = [x.astype(np.float64) for x in KC.qkv_values(rng, pos0 + L, L, n_head, n_kv, hd, True)]
    got = R.attention(q, k, v, pos0, n_head, n_kv, hd, 1.0 / np.sqrt(hd))
    grp = n_head // n_kv
    for i in range(L):
        pos = pos0 + i
        Kc = k[:pos + 1].reshape(pos + 1, n_kv, hd)
        Vc = v[:pos + 1].reshape(pos + 1, n_kv, hd)
        qh = q[i].reshape(n_head, hd)
        for hh in range(n_head):
            s = Kc[:, hh // grp, :] @ qh[hh] / np.sqrt(hd)
            s = s - s.max()
            pw = np.exp(s)
            pw /= pw.sum()
            assert np.allclose(got[i, hh * hd:(hh + 1) * hd], pw @ Vc[:, hh // grp, :], rtol=1e-12, atol=1e-12)


def test_streamk_restatement_covers_every_unit_once():
    for n_tiles, nkb, n_sm in ((8, 1, 5), (4, 3, 13), (3, 5, 8), (32, 16, 132), (1002, 16, 132)):
        U = n_tiles * nkb
        G = R.streamk_grid(n_tiles, nkb, n_sm)
        starts = [R.q_range_start(c, U, G) for c in range(G + 1)]
        assert starts[0] == 0 and starts[-1] == U and all(a <= b for a, b in zip(starts, starts[1:]))
        for x in range(U):
            c = R.q_owner_of(x, U, G)
            assert starts[c] <= x < starts[c + 1]


# ---- GEMMs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", KC.GEMM_CASES, ids=KC.gemm_case_id)
def test_gemm_mutants_are_caught(case):
    m, n, k, epi, _kind = case
    for bf16 in (0, 1):
        _ab, a, _bb, b, old = KC.gemm_inputs(case, bf16)
        rows = np.unique(np.linspace(0, m - 1, min(m, 48)).astype(int))
        a = a[rows]
        ref, bound = R.gemm(a, b)
        nkb = (k + 63) // 64
        rel16 = R.gemm_rel_l2_bound(k, "bf16" if bf16 else "fp16")
        for j in sorted({0, nkb - 1}):
            mut, _ = R.gemm(a, b, "drop_kblock", j)
            if epi == KC.SILU:
                r, bb = R.silu_ref(ref, bound)
                d = _gemm_distance(R.silu_ref(mut, bound)[0], r, bb, R.ulp16(r, bool(bf16)), rel16)
            elif epi == KC.T16:
                d = _gemm_distance(mut, ref, bound, R.ulp16(ref, bool(bf16)), rel16)
            else:
                base = old[rows] if epi == KC.ADD else 0.0
                d = _gemm_distance(mut + base, ref + base, bound, 0.0, R.gemm_rel_l2_bound(k))
            assert d >= MARGIN, (case, bf16, "drop_kblock", j, d)
        if epi == KC.SILU:
            r, bb = R.silu_ref(ref, bound)
            d = _gemm_distance(R.silu_ref(ref, bound, "swap_gate_up")[0], r, bb, R.ulp16(r, bool(bf16)), rel16)
            assert d >= MARGIN, (case, bf16, "swap_gate_up", d)


@pytest.mark.parametrize("pos0", [0, 1, 17, 200])
def test_rope_split_mutants_are_caught(pos0):
    n_head, n_kv = KC.ROPE_HEADS
    for hd in (64, 128):
        rng = np.random.Generator(np.random.PCG64(pos0 * 7 + hd))
        x = rng.standard_normal((KC.ROPE_M, (n_head + 2 * n_kv) * hd))
        cos_t, sin_t = KC.rope_tables(hd, 512)
        segs = KC.rope_segs(pos0)
        ref = R.rope_split(x, np.abs(x), n_head, n_kv, hd, cos_t, sin_t, segs)
        for mutant in ("pos0+1", "pos0-1"):
            mut = R.rope_split(x, np.abs(x), n_head, n_kv, hd, cos_t, sin_t, segs, mutant)
            for i in (0, 1):          # q and k
                d = _gemm_distance(mut[i], ref[i], ref[3 + i], R.ulp16(ref[i]))
                assert d >= MARGIN, (pos0, hd, mutant, "qk"[i], d)


# ---- attention --------------------------------------------------------------------------------------------------------------
def _attn_mutants(n_head, n_kv, pos0, L):
    muts = ["diag"]
    if L > 1:                         # a key past the row exists for every row but the last
        muts.append("pos0+1")
    if pos0 > 0:
        muts.append("pos0-1")
    if pos0 + L > 64:                 # some row has a second KV tile
        muts.append("drop_last_kv_tile")
    if n_kv > 1 and n_head // n_kv > 1:
        muts.append("gqa_mod")
    return muts


def _attn_teeth(q, k, v, pos0, n_head, n_kv, hd, L):
    rows = R.attention_sample_rows(L)
    if len(rows) > 40:
        rows = np.unique(np.concatenate([rows[:8], rows[::max(1, len(rows) // 32)], rows[-4:]]))
    q, k, v = (x.astype(np.float64) for x in (q, k, v))
    scale = 1.0 / np.sqrt(hd)
    ref = R.attention(q, k, v, pos0, n_head, n_kv, hd, scale, rows)
    for mutant in _attn_mutants(n_head, n_kv, pos0, L):
        with np.errstate(invalid="ignore", divide="ignore"):
            mut = R.attention(q, k, v, pos0, n_head, n_kv, hd, scale, rows, mutant)
        d = _attn_distance(mut, ref, v, n_head, n_kv, hd)
        assert d >= MARGIN, (pos0, L, n_head, n_kv, hd, mutant, d)


@pytest.mark.parametrize("heads", KC.ATTN_HEADS, ids=lambda h: f"h{h[0]}kv{h[1]}")
@pytest.mark.parametrize("hd", [64, 128])
def test_flash_nonpaged_mutants_are_caught(hd, heads):
    n_head, n_kv = heads
    for L in KC.ATTN_LENS:
        for peaked in (False, True):
            rng = np.random.Generator(np.random.PCG64(L * 3 + hd + n_head + peaked))
            q, k, v = KC.qkv_values(rng, L, L, n_head, n_kv, hd, peaked)
            _attn_teeth(q, k, v, 0, n_head, n_kv, hd, L)


@pytest.mark.parametrize("heads", KC.ATTN_HEADS, ids=lambda h: f"h{h[0]}kv{h[1]}")
@pytest.mark.parametrize("hd", [64, 128])
def test_flash_paged_mutants_are_caught(hd, heads):
    n_head, n_kv = heads
    for pos0 in KC.PAGED_POS0:
        for L in KC.PAGED_LENS:
            peaked = (pos0 + L) % 2 == 1
            rng = np.random.Generator(np.random.PCG64(pos0 * 11 + L + hd + n_head))
            q, k, v = KC.qkv_values(rng, pos0 + L, L, n_head, n_kv, hd, peaked)
            _attn_teeth(q, k, v, pos0, n_head, n_kv, hd, L)


# ---- qgemm ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(KC.QG_SHAPES))
def test_qgemm_mutants_are_caught(hostcheck_lib, name):
    """dropping one qtile, dropping each kind of split-tile partial the GPU sweep produces (stream-K and cluster quarters), and
    (SiLU) swapping gate and up, each on one output tile of the shape"""
    specs, mode, k, epi, _how = KC.QG_SHAPES[name]
    srcs, mode = KC.qg_sources(name)
    act = KC.qg_act(name, k)[:64].astype(np.float64)
    n_tiles, nkb = sum(r for r, _t in specs) // 128, k // 256
    sms = (1, 2, 3, 4, 5, 8, 13, 33, 64, 132)
    parts = {p for s in sms for p in R.streamk_partials(n_tiles, nkb, s)}
    if nkb >= 4:
        parts |= {(t, lo, hi) for t in (0, n_tiles - 1) for lo, hi in R.cluster_partials(nkb)}
    tiles = sorted({0, n_tiles - 1} | {p[0] for p in parts})
    for t in tiles[:6] + tiles[-2:]:
        w = R.qtile_weights(hostcheck_lib, srcs, mode, t)
        ref, bound = act @ w.T, np.abs(act) @ np.abs(w).T
        muts = [(t, kb, kb + 1) for kb in (0, nkb - 1)] + [p for p in parts if p[0] == t]
        for _t, lo, hi in muts:
            wm = w.copy()
            wm[:, lo * 256:hi * 256] = 0.0
            mut = act @ wm.T
            for nb in (16, 32, 64):
                if epi == KC.SILU:
                    r, bb = R.silu_ref(ref[:nb], bound[:nb])
                    d = _gemm_distance(R.silu_ref(mut[:nb], bound[:nb])[0], r, bb, R.ulp16(r), R.gemm_rel_l2_bound(k, "fp16"))
                else:
                    d = _gemm_distance(mut[:nb], ref[:nb], bound[:nb], 0.0, R.gemm_rel_l2_bound(k))
                assert d >= MARGIN, (name, t, lo, hi, nb, d)
        if epi == KC.SILU:
            for nb in (16, 32, 64):
                r, bb = R.silu_ref(ref[:nb], bound[:nb])
                d = _gemm_distance(R.silu_ref(ref[:nb], bound[:nb], "swap_gate_up")[0], r, bb, R.ulp16(r), R.gemm_rel_l2_bound(k, "fp16"))
                assert d >= MARGIN, (name, t, "swap_gate_up", nb, d)


def test_folded_norm_mutant_is_caught(hostcheck_lib):
    """the consumer without its 16 / rms factor, on sums of squares of the size the producer of the GPU test writes"""
    srcs, mode = KC.qg_sources("qkv_8b")
    act = KC.qg_act("qkv_8b", 4096)[:16].astype(np.float64) / 16.0
    w = R.qtile_weights(hostcheck_lib, srcs, mode, 0)
    c, b = act @ w.T, np.abs(act) @ np.abs(w).T
    rng = np.random.Generator(np.random.PCG64(8))
    x_new = rng.standard_normal((16, 4096))
    _xg, ssq = R.norm_producer(x_new, np.ones(4096), 32)
    s = R.norm_consumer_scale(ssq, 4096, 1e-5)
    s_mut = R.norm_consumer_scale(ssq, 4096, 1e-5, "no_rms")
    d = _gemm_distance(c * s_mut[:, None], c * s[:, None], b * s[:, None], 0.0, R.gemm_rel_l2_bound(4096))
    assert d >= MARGIN, d
    assert np.allclose(ssq.sum(axis=0), (x_new ** 2).sum(axis=1))
