"""Kernel-level checks of the batch-1 decode GEMV (gemv_launch: gemv.cu, gemv_core.cuh, rowdot.h) and of the fp-weight decode
route against float64 references, one launch at a time through the launcher shim tests/gemvcheck.  Inputs, references and bounds:
tests/gemv_cases.py; tests/test_decode_gemv_cpu.py rehearses the bounds with the lane program and shows they have teeth.

Every launch runs behind a kernel that releases its dependants at once and writes x, the residual and the position only ~20 us
later: until then x and the residual are NaN and the position is an in-bounds decoy whose KV page is NaN.  Per launch: every
output within its per-element bound and finite, the sentinels around the output untouched (no padding row or row past `rows`
written), the K / V caches bit-identical except slot pos % 16 of page table[pos / 16] of each KV head (the decoy's page
included), a residual that is not aliased unchanged, and replays bit-identical.  The launch takes the ring geometry the engine
takes (gemv_geometry), unless a test overrides it.

Invariant: a row is computed by one warp in a fixed order (its lanes' K-segments in order, then warp_sum4 / warp_sum2), whatever
the grid, the warp count, the tracks, the ring depth or the prologue.  The three prologues build the same planes: each takes
fp32(x * w), the block maximum with fmaxf (order-free), the same reciprocal and rint, and integer sums; only the RMSNorm sum of
squares is reduced in a different order.  So without RMSNorm the output is bit-identical across every variant, and with it the
variants differ only through `scale`, by a few ulps.

Each family prints its worst error / bound ratio as `GEMVCHECK <family> <ratio>`."""
import ctypes

import numpy as np
import pytest

import batch_cases as B
import gemv_cases as G

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in G.cases()}
WORST = {}
EPI_NAME = {G.EPI_STORE: "store", G.EPI_ADD: "add", G.EPI_QKV: "qkv", G.EPI_SILU: "silu"}


def _note(family, r):
    WORST[family] = max(WORST.get(family, 0.0), float(r))
    print(f"GEMVCHECK {family} {WORST[family]:.4f}", flush=True)


@pytest.fixture(scope="module")
def lib():
    return G.load_shim()


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launch(lib, case, **kw):
    """run, check everything but the values; returns (out float64 [out_rows], result dict)"""
    return _checked(case, *G.run_gemv(lib, case, **kw))


def _checked(case, rc, res):
    assert rc == 0, f"{case.name}: error {rc}"
    out = res["out"]
    n = case.out_rows
    assert (out[:, :G.PAD] == G.SENT32).all() and (out[:, G.PAD + n:] == G.SENT32).all(), "write outside the output rows"
    assert (out == out[0]).all(), "replays differ"
    got = out[0, G.PAD:G.PAD + n].view(np.float32).astype(np.float64)
    assert np.isfinite(got).all(), "non-finite output"
    if case.kc is not None:
        assert (res["kc"] == res["kc"][0]).all() and (res["vc"] == res["vc"][0]).all(), "replays differ in the caches"
        assert G.check_pool(case, res["kc"][0], res["vc"][0]), "K / V written outside slot pos % 16 of page table[pos / 16]"
    if res["resid"] is not None:
        assert (res["resid"] == case.resid).all(), "the residual changed"
    return got, res


def _check_values(case, got, res):
    ref = case.reference()
    fam = EPI_NAME[case.epi]
    r = G.ratio(got, ref["out"])
    _note(fam, r)
    assert r <= 1.0, (case.name, "out", r)
    if case.epi == G.EPI_QKV:
        k = case.cache_rows(res["kc"][0])
        v = case.cache_rows(res["vc"][0])
        rk, rv = G.ratio(k, ref["k"]), G.ratio(v, ref["v"])
        _note("qkv-k", rk)
        _note("qkv-v", rv)
        assert rk <= 1.0 and rv <= 1.0, (case.name, rk, rv)


@pytest.mark.parametrize("name", list(CASES))
def test_launch_within_bound(lib, name):
    case = CASES[name]
    got, res = _launch(lib, case)
    assert res["geom"][4] == case.nks
    _check_values(case, got, res)


# no RMSNorm: bit-identical across every variant; with RMSNorm: a few ulps
INVARIANT = ["8b-ffn_down-12", "8b-attn_output", "k32768", "rows5-q4k", "gate_up-q6k-k8192", "k256-q6k", "rows4097-q6k"]
INVARIANT_NORM = ["k8192-norm", "k256-norm", "q8-gate_up"]


def _variants(case, n_sm):
    items = sum(-(-r // case.item_rows_of(m)) for m, r in enumerate(case.rows[:1] if case.pair else case.rows))
    v = [dict(n_ctas=1), dict(n_ctas=7), dict(n_ctas=items + 3), dict(nw=8), dict(nw=16), dict(pro=0), dict(pro=1), dict(pro=2),
         dict(lean=0), dict(lean=1), dict(polite=0), dict(polite=3), dict(pdl=False), dict(n_tracks=5, depth=2), dict(n_tracks=12, depth=1)]
    if case.cols <= 4096:
        v.append(dict(n_tracks=3, depth=4))
    return v


@pytest.mark.parametrize("name", INVARIANT + INVARIANT_NORM)
def test_geometry_invariant(lib, n_sm, name):
    case = CASES[name]
    base, bres = _launch(lib, case, n_ctas=n_sm, reps=1)
    pros = {bres["geom"][3]}
    for kw in _variants(case, n_sm):
        rc, res = G.run_gemv(lib, case, **dict(dict(n_ctas=n_sm, reps=2), **kw))
        if rc == -3:                          # an override the ring cannot hold at this width
            continue
        got, res = _checked(case, rc, res)
        pros.add(res["geom"][3])
        if case.norm:
            d = np.abs(got - base) / np.maximum(np.abs(base), 1e-30)
            assert float(d.max()) <= 32 * 2.0 ** -24, (name, kw, float(d.max()))
        else:
            assert (got.view(np.uint64) == base.view(np.uint64)).all(), (name, kw)
        _check_values(case, got, res)
    if case.cols <= 4096:
        assert pros == {0, 1, 2}, pros


def test_unsupported_width_is_a_clean_error(lib):
    case = G.GemvCase("k4352", [G.Q4_K], [8], 4352)     # 17 blocks: no equal cut into <= 16-block K-segments (nks = 0)
    rc, _ = G.run_gemv(lib, case)
    assert rc == -1


# ---- the fp-weight decode route --------------------------------------------------------------------------------------------------
def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("t", [G.F32, G.F16, G.BF16])
@pytest.mark.parametrize("cols", [200, 4096])
def test_fp_gemv(lib, t, cols):
    from oracle import gguf_synth as S
    from oracle import llama_oracle as O
    rng = np.random.Generator(np.random.PCG64([t, cols]))
    rows = 1000
    w = S.quantize(rng.standard_normal((rows, cols), dtype=np.float32) / np.float32(np.sqrt(cols)), t)
    x = rng.standard_normal(cols).astype(np.float32)
    y = np.zeros(rows, np.float32)
    assert lib.gc_fp_gemv(_ptr(w), t, rows, cols, _ptr(x), _ptr(y)) == 0
    w64 = O.dequantize(w, t, (rows, cols)).astype(np.float64)
    ref = w64 @ x.astype(np.float64)
    # lane order: 4 (F32) or 8 (16-bit) products per step, cols / 128 or cols / 256 steps, then five shuffle levels
    kappa = cols / 32 + 16
    bound = kappa * G.U * (np.abs(w64) @ np.abs(x.astype(np.float64)))
    r = float(np.max(np.abs(y - ref) / bound))
    _note("fp-gemv", r)
    assert r <= 1.0


@pytest.mark.parametrize("n", [256, 4096, 8192])
def test_rmsnorm(lib, n):
    from oracle import llama_oracle as O
    rng = np.random.Generator(np.random.PCG64(n))
    x = (rng.standard_normal(n) * 0.01).astype(np.float32)
    w = (1 + 0.25 * rng.standard_normal(n)).astype(np.float32)
    y = np.zeros(n, np.float32)
    assert lib.gc_rmsnorm(_ptr(x), _ptr(w), n, ctypes.c_float(1e-5), _ptr(y)) == 0
    ref = O.rmsnorm(x, w, 1e-5)
    bound = (((n / 256 + 13) / 2 + 3) + 2) * G.U * np.abs(ref) + 1e-30
    r = float(np.max(np.abs(y - ref) / bound))
    _note("rmsnorm", r)
    assert r <= 1.0


@pytest.mark.parametrize("hd,n_head,n_kv,pos", [(128, 32, 8, 575), (64, 8, 2, 17), (128, 8, 1, 0), (64, 4, 1, 2047)])
def test_rope_kv(lib, hd, n_head, n_kv, pos):
    case = G.GemvCase("rope", [G.Q4_K] * 3, [n_head * hd, n_kv * hd, n_kv * hd], 256, G.EPI_QKV, head_dim=hd, n_kv=n_kv, pos=pos)
    rng = np.random.Generator(np.random.PCG64([hd, pos]))
    q = rng.standard_normal(n_head * hd).astype(np.float32)
    k = rng.standard_normal(n_kv * hd).astype(np.float32)
    v = rng.standard_normal(n_kv * hd).astype(np.float32)
    qo, kc, vc = q.copy(), case.kc.copy(), case.vc.copy()
    rc = lib.gc_rope_kv(_ptr(qo), _ptr(k), _ptr(v), n_head, n_kv, hd, _ptr(case.cos), _ptr(case.sin), ctypes.c_size_t(case.cos.size), pos,
                        _ptr(case.table), case.n_table, _ptr(kc), _ptr(vc), ctypes.c_size_t(kc.nbytes))
    assert rc == 0
    assert G.check_pool(case, kc, vc)
    zq, zk = np.zeros(q.size), np.zeros(k.size)
    qr, qb = case._rope(q.astype(np.float64), zq, pos, None)
    kr, kb = case._rope(k.astype(np.float64), zk, pos, None)
    r = max(G.ratio(qo, (qr, qb + 1e-30)), G.ratio(case.cache_rows(kc), (kr, kb + G.ulp16(kr))))
    _note("rope_kv", r)
    assert r <= 1.0
    assert (case.cache_rows(vc) == v.astype(np.float16).astype(np.float64)).all()


def test_silu_mul_and_add(lib):
    rng = np.random.Generator(np.random.PCG64(5))
    n = 14336
    a = (4 * rng.standard_normal(n)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    out = np.zeros(n, np.float32)
    assert lib.gc_eltwise(0, _ptr(a), _ptr(b), n, _ptr(out)) == 0
    a64 = a.astype(np.float64)
    ref = a64 / (1 + np.exp(-a64)) * b
    r = float(np.max(np.abs(out - ref) / (8 * G.U * np.abs(ref) + 1e-38)))
    _note("silu_mul", r)
    assert r <= 1.0
    assert lib.gc_eltwise(1, _ptr(a), _ptr(b), n, _ptr(out)) == 0
    assert (out == a + b).all()


@pytest.mark.parametrize("t", [G.Q4_K, G.Q6_K, G.Q8_0, G.F16, G.F32, G.BF16])
def test_embed(lib, t):
    from oracle import gguf_synth as S
    from oracle import llama_oracle as O
    rng = np.random.Generator(np.random.PCG64(t))
    n_vocab, cols = 300, 4096
    w = S.random_blocks(rng, t, n_vocab, cols)
    ids = rng.permutation(n_vocab)[:64].astype(np.int32)
    # (pos, n_prompt, out_idx, token) -> the row embed_launch must gather: the prompt's token while pos < n_prompt and nothing
    # was drawn; the drawn token otherwise, also at a position below n_prompt after a context shift
    for pos, n_prompt, out_idx, token, want in ((5, 64, 0, 7, ids[5]), (63, 64, 0, 7, ids[63]), (64, 64, 0, 9, 9), (20, 64, 3, 11, 11),
                                                (0, 64, 0, 299, ids[0])):
        st = np.zeros(1, B.STEP_STATE)
        st["pos"], st["n_prompt"], st["out_idx"], st["token"] = pos, n_prompt, out_idx, token
        x = np.zeros(cols, np.float32)
        assert lib.gc_embed(_ptr(w), t, n_vocab, cols, _ptr(st), _ptr(ids), ids.size, _ptr(x)) == 0
        assert int(st["token"][0]) == int(want)
        if t in (G.Q4_K, G.Q6_K, G.Q8_0):
            ref, a = G.dequant_parts(w[int(want):int(want) + 1], t, cols)
            r = float(np.max(np.abs(x - ref[0]) / (3 * G.U * a[0] + 1e-38)))
            _note("embed", r)
            assert r <= 1.0
        else:
            assert (x == O.dequantize(w[int(want):int(want) + 1], t, (1, cols))[0]).all()
