"""Kernel-level checks of the batched decode step's per-row kernels (batch.cu, and the embedding gather of prefill.cu) against
float64 references, one launch at a time through the launcher shim tests/batchcheck.  Inputs, references and bounds:
tests/batch_cases.py; tests/test_batch_kernels_cpu.py rehearses the bounds on these very cases and shows they have teeth.

Attention launches run in both modes -- fused (the kernel rotates q and appends the step's K / V rows) and unfused
(batch_rope_kv_launch, then the kernel on q) -- behind a kernel that releases its dependants at once and writes the QKV rows only
~20 us later (a read before griddepcontrol.wait sees NaN).  Unowned pages and table entries past a row's pages are NaN; the row's
own last page holds stale data past its position.  Per launch: the error of every live row within the bound, replays
bit-identical, the counters zero afterwards, nothing written outside the live rows of the output, the K / V pool byte-identical
except each live row's newest slot, and that slot within the RoPE bound (K) and bit-exact (V).

Each family prints its worst error / bound ratio as `BATCHCHECK <family> <ratio>`."""
import ctypes
import os

import numpy as np
import pytest

import batch_cases as B
import kernel_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAD = 256                          # sentinel halves / floats around outputs
SENT32 = np.uint32(0x7FC0BAD5)
WORST = {}


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), float(ratio))
    print(f"BATCHCHECK {family} {WORST[family]:.4f}", flush=True)


@pytest.fixture(scope="module")
def lib():
    from gridllm_b200 import native
    native.load_library()
    path = os.path.join(ROOT, "tests", "batchcheck", "libbatchcheck.so")
    assert os.path.exists(path), "tests/batchcheck/libbatchcheck.so is missing (run __graft_entry__.build())"
    l = ctypes.CDLL(path)
    for f in ("bc_attn", "bc_sample_greedy", "bc_sample_single", "bc_rmsnorm", "bc_embed_rows"):
        getattr(l, f).restype = ctypes.c_int
    assert l.bc_state_bytes() == B.STEP_STATE.itemsize and l.bc_ctl_bytes() == B.BATCH_CTL.itemsize
    return l


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _attn(lib, case, fused, reps=2):
    """run the launch; returns (out16 [reps][bucket][n_head * hd] float64, kc_all, vc_all, counters, q_out)"""
    n_out = case.bucket * case.qd
    out16 = np.full(n_out + 2 * PAD, B.SENT16, np.uint16)
    out_all = np.zeros((reps, out16.size), np.uint16)
    kc_all = np.zeros((reps,) + case.kc.shape, np.uint16)
    vc_all = np.zeros_like(kc_all)
    ctr = np.full((reps, case.bucket * case.n_kv), 0xFFFFFFFF, np.uint32)
    q_all = np.zeros((reps, case.bucket * case.qd), np.float32)
    Z, I, U, F = ctypes.c_size_t, ctypes.c_int, ctypes.c_uint, ctypes.c_float
    rc = lib.bc_attn(I(int(fused)), I(reps), U(20000), _p(case.qkv), I(case.ld), _p(case.ctl), _p(case.st), _p(case.tables),
                     I(case.stride), _p(case.cos), _p(case.sin), Z(case.cos.size), _p(case.kc), _p(case.vc), Z(case.kc.nbytes),
                     I(case.bucket), I(case.n_head), I(case.n_kv), I(case.hd), I(case.S), F(float(case.scale)), _p(out16), Z(out16.size),
                     Z(PAD), _p(out_all), _p(kc_all), _p(vc_all), _p(ctr), _p(q_all))
    assert rc == 0, f"CUDA error {rc}"
    assert (out_all[:, :PAD] == B.SENT16).all() and (out_all[:, -PAD:] == B.SENT16).all(), "write outside out16"
    assert (out_all[:, PAD + case.n_rows * case.qd:-PAD] == B.SENT16).all(), "a padded row was written"
    assert (out_all == out_all[0]).all(), "replays differ"
    assert (kc_all == kc_all[0]).all() and (vc_all == vc_all[0]).all(), "replays differ in the caches"
    assert (ctr == 0).all(), "ticket counters not back at zero"
    got = out_all[0, PAD:PAD + case.n_rows * case.qd].view(np.float16).astype(np.float64).reshape(case.n_rows, case.qd)
    return got, kc_all[0], vc_all[0], q_all[0].reshape(case.bucket, case.qd)


def _check_pool(case, kc, vc):
    """byte-identical except each live row's newest slot; K there within the RoPE bound, V bit-exact"""
    keep = ~case.newest[:, None, :, None] & np.ones(kc.shape, bool)
    assert (kc[keep] == case.kc[keep]).all() and (vc[keep] == case.vc[keep]).all(), "K / V written outside the newest slots"
    worst = 0.0
    bound = B.rope_bound(case.k_raw, case.hd) + R.ulp16(case.k_ref)
    for r in range(case.n_rows):
        ph, t = case.slot_of(r)
        assert (vc[ph, :, t] == case.vc_after[ph, :, t]).all(), ("V row not float32 -> float16", r)
        k = kc[ph, :, t].view(np.float16).astype(np.float64).reshape(-1)
        worst = max(worst, float((np.abs(k - case.k_ref[r]) / bound[r]).max()))
    assert worst <= 1.0, worst
    _note("rope_kv", worst)


def _check_attn(case, got, fused):
    worst = 0.0
    for r in range(case.n_rows):
        ref, v = case.reference(r)
        d = B.attn_distance(got[r], ref, v, case.n_head, case.n_kv, case.hd)
        assert d <= 1.0, (r, int(case.pos[r]), "fused" if fused else "unfused", d)
        worst = max(worst, d)
    _note("attention", worst)


CASES = B.attn_cases()


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_batch_attention(lib, name, kw, fused):
    case = B.AttnCase(**kw)
    got, kc, vc, q = _attn(lib, case, fused)
    _check_pool(case, kc, vc)
    _check_attn(case, got, fused)
    if not fused:       # q_out: the float64 rotation within 2^-22 (|x0| + |x1|); padded rows untouched (NaN)
        qb = B.rope_bound(case.qkv[:case.n_rows, :case.qd].astype(np.float64), case.hd)
        assert (np.abs(q[:case.n_rows] - case.q_ref) <= qb).all()
        assert np.isnan(q[case.n_rows:]).all()


def test_shared_prefix_matches_private_pages(lib):
    """two rows whose tables share their first pages give the bits of the same bytes held in private pages"""
    kw = B.layout_kwargs()
    a = B.AttnCase(**kw)
    b = B.AttnCase(**B.private_copy_kwargs(kw))
    # the private case draws other values: give its rows the shared case's logical rows
    for r in range(a.n_rows):
        for j in range(int(a.n_pages[r])):
            b.kc[b.tables[b.slots[r], j]] = a.kc[a.tables[a.slots[r], j]]
            b.vc[b.tables[b.slots[r], j]] = a.vc[a.tables[a.slots[r], j]]
    b.qkv = a.qkv
    for fused in (True, False):
        ga = _attn(lib, a, fused, reps=1)[0]
        gb = _attn(lib, b, fused, reps=1)[0]
        assert (ga.view(np.uint64) == gb.view(np.uint64)).all(), fused


# ---- greedy draw -----------------------------------------------------------------------------------------------------------
VOCABS = [9, 4097, 32000, 128256, 151936]


@pytest.mark.parametrize("n_vocab", VOCABS)
def test_batch_greedy(lib, n_vocab):
    bucket, n_rows, max_out = 128, 12, 4
    lg = np.zeros((bucket, n_vocab), np.float32)
    lg[:n_rows] = B.greedy_logits(n_vocab, n_rows, 1)
    lg[n_rows:] = np.float32(np.nan)                       # padded rows are never read
    rng = np.random.Generator(np.random.PCG64(n_vocab))
    slots = rng.permutation(B.MAX_BATCH)[:n_rows]
    ctl = np.zeros(1, B.BATCH_CTL)
    ctl["n_rows"] = n_rows
    ctl["row_slot"][0, :n_rows] = slots
    st = np.zeros(B.MAX_BATCH, B.STEP_STATE)
    st["pos"] = rng.integers(0, 1000, B.MAX_BATCH)
    st["token"] = -5
    st["out_idx"] = 1
    st["n_stop"] = 2
    st["stop_ids"][:, 0] = n_vocab + 3
    st["stop_ids"][:, 1] = n_vocab + 4
    ids_ref, lp_ref = B.greedy_ref(lg[:n_rows])
    # state branches on rows 5 .. 10 (their logits stay ordinary rows)
    s = slots
    st["temperature"][s[5]] = 0.7                          # sampled row: left alone
    st["done"][s[6]] = 1                                   # finished: left alone
    st["stop_ids"][s[7], 1] = ids_ref[7]                   # stop id hit
    st["stop_ids"][s[8], 0] = ids_ref[8]                   # stop id hit, but ignore_eos
    st["ignore_eos"][s[8]] = 1
    st["out_idx"][s[9]] = max_out                          # output buffer full: the state advances, nothing is written
    st["out_idx"][s[10]] = max_out + 3
    out_len = B.MAX_BATCH * max_out + PAD
    out_ids = np.full(out_len, -77, np.int32)
    out_lps = np.full(out_len, SENT32, np.uint32).view(np.float32)
    bout = np.zeros(B.MAX_BATCH, B.BATCH_OUT)
    bout["token"] = -99
    scratch = np.zeros(B.MAX_BATCH * B.SAMPLE_ROW_FLOATS, np.float32)
    st_in, out_ids_in, out_lps_in = st.copy(), out_ids.copy(), out_lps.copy()
    st_all = np.zeros((2, B.MAX_BATCH), B.STEP_STATE)
    bout_all = np.zeros((2, B.MAX_BATCH), B.BATCH_OUT)
    rc = lib.bc_sample_greedy(2, _p(lg), n_vocab, bucket, _p(ctl), _p(st), _p(out_ids), _p(out_lps), ctypes.c_size_t(out_len), max_out,
                              _p(bout), _p(scratch), _p(st_all), _p(bout_all))
    assert rc == 0, rc
    assert st_all[0].tobytes() == st_all[1].tobytes() and bout_all[0].tobytes() == bout_all[1].tobytes(), "second launch differs"
    tickets = scratch.view(np.uint32).reshape(B.MAX_BATCH, B.SAMPLE_ROW_FLOATS)[:, 3 * B.SAMPLE_PARTS]
    assert (tickets == 0).all(), "ticket counters not back at zero"
    bound = B.greedy_lp_bound(n_vocab)
    worst = 0.0
    other = np.setdiff1d(np.arange(B.MAX_BATCH), slots)
    assert st[other].tobytes() == st_in[other].tobytes(), "a slot outside the batch changed"
    written = np.zeros(out_len, bool)
    for r in range(n_rows):
        sl = int(s[r])
        a, b = st_in[sl], st[sl]
        if r in (5, 6):
            assert a.tobytes() == b.tobytes(), r
        else:
            assert b["token"] == ids_ref[r], (r, int(b["token"]), int(ids_ref[r]))
            assert b["pos"] == a["pos"] + 1 and b["out_idx"] == a["out_idx"] + 1
            assert b["done"] == (1 if r == 7 else 0), r
            k = int(a["out_idx"])
            if k < max_out:
                assert out_ids[sl * max_out + k] == ids_ref[r]
                err = abs(float(out_lps[sl * max_out + k]) - lp_ref[r])
                assert err <= bound, (r, err, bound)
                worst = max(worst, err / bound)
                written[sl * max_out + k] = True
        # batch_collect: {token, logprob, done, pos} of the row
        o = bout[r]
        assert o["token"] == b["token"] and o["done"] == b["done"] and o["pos"] == b["pos"]
        k = int(b["out_idx"]) - 1
        exp_lp = np.float32(out_lps[sl * max_out + k]) if 0 <= k < max_out else np.float32(0.0)
        assert o["logprob"].tobytes() == exp_lp.tobytes(), r
    assert (out_ids[~written] == out_ids_in[~written]).all() and (out_lps.view(np.uint32)[~written] == out_lps_in.view(np.uint32)[~written]).all()
    assert (bout[n_rows:bucket]["token"] == 0).all() and (bout[n_rows:bucket]["logprob"] == 0).all()
    assert (bout[n_rows:bucket]["done"] == 0).all() and (bout[n_rows:bucket]["pos"] == 0).all()
    _note("greedy_logprob", worst)
    # the single-sequence sampler draws the same ids
    for r in range(n_rows):
        one = np.zeros(1, B.STEP_STATE)
        oi = np.full(2, -1, np.int32)
        ol = np.zeros(2, np.float32)
        row = np.ascontiguousarray(lg[r])
        assert lib.bc_sample_single(_p(row), n_vocab, _p(one), _p(oi), _p(ol), 2) == 0
        assert oi[0] == ids_ref[r] and one["token"][0] == ids_ref[r], r
        assert abs(float(ol[0]) - lp_ref[r]) <= 2e-5 + bound, r


# ---- RMSNorm ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [64, 256, 4096, 5120, 8192])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_batch_rmsnorm(lib, n, eps):
    x, w = B.rmsnorm_rows(n)
    rows = x.shape[0]
    y = np.full((rows + 3) * n + PAD, B.SENT16, np.uint16)
    rc = lib.bc_rmsnorm(_p(x), _p(w), rows, n, ctypes.c_float(eps), _p(y), ctypes.c_size_t(y.size))
    assert rc == 0, rc
    assert (y[rows * n:] == B.SENT16).all(), "rows past `rows` written"
    got = y[:rows * n].view(np.float16).astype(np.float64).reshape(rows, n)
    ref = B.rmsnorm_ref(x, w, eps)
    d = B.rmsnorm_distance(got, ref)
    assert d <= 1.0, d
    assert (got[3] == 0).all(), "an all-zero row must come out as 0 (-0 where w < 0)"
    _note("rmsnorm", d)


# ---- embedding gather ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["Q4_K", "Q6_K", "Q8_0", "F16", "F32"])
def test_batch_embed_rows(lib, typ):
    from oracle import gguf_synth as S, llama_oracle as O
    t = getattr(S, typ)
    n_vocab, cols, bucket = 300, 512, 16
    rng = np.random.Generator(np.random.PCG64(len(typ) + t))
    blocks = np.ascontiguousarray(S.random_blocks(rng, t, n_vocab, cols))
    ref = O.dequantize(blocks, t, (n_vocab, cols)).astype(np.float64)
    bound = B.embed_bound(blocks, t, n_vocab, cols)
    toks = [0, n_vocab - 1, 7, 7, 123, 0, n_vocab - 1]
    n_rows = len(toks)
    slots = rng.permutation(B.MAX_BATCH)[:n_rows]
    ctl = np.zeros(1, B.BATCH_CTL)
    ctl["n_rows"] = n_rows
    ctl["row_slot"][0, :n_rows] = slots
    st = np.zeros(B.MAX_BATCH, B.STEP_STATE)
    st["token"] = 5
    st["token"][slots] = toks
    x = np.full((bucket + 2) * cols, SENT32, np.uint32).view(np.float32)
    ids = np.full(B.MAX_BATCH, -3, np.int32)
    rb = S.row_bytes(t, cols)
    rc = lib.bc_embed_rows(_p(blocks), ctypes.c_size_t(blocks.nbytes), t, cols, rb, _p(ctl), _p(st), bucket, _p(x), ctypes.c_size_t(x.size), _p(ids))
    assert rc == 0, rc
    assert (ids[:bucket] == np.array(toks + [0] * (bucket - n_rows))).all() and (ids[bucket:] == -3).all()
    assert (x.view(np.uint32)[bucket * cols:] == SENT32).all(), "rows past the bucket written"
    got = x[:bucket * cols].astype(np.float64).reshape(bucket, cols)
    want = ref[ids[:bucket]]
    err = np.abs(got - want)
    if t in (S.F16, S.F32):
        assert (err == 0).all()
        _note("embed", 0.0)
    else:
        b = bound[ids[:bucket]]
        assert (err <= b).all(), float((err / np.maximum(b, 1e-300)).max())
        _note("embed", float((err / np.maximum(b, 1e-300)).max()))
