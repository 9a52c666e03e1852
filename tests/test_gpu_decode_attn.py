"""Kernel-level check of the batch-1 decode attention (attention.cu, attn_decode_launch) against a float64 reference, through
the launcher shim tests/attncheck.

Every launch runs behind a small upstream kernel (programmatic dependent launch, as behind the QKV GEMV) that appends the
pending K / V rows only ~20 us after the attention kernel may have started, and only then publishes the position: a row read
before griddepcontrol.wait is a NaN, and so is every unused page slot of the shuffled page table and every row past the
position.  Sentinels around the output must come back untouched, and replays must be bit-identical.  The CPU test at the end
shows that the tolerance has teeth: dropping a split's pages, a stale newest row or an off-by-one page lands at least 4x the
tolerance away on the same inputs."""
import ctypes
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN16 = np.uint16(0x7E5A)            # poison / sentinel bits: a quiet NaN no kernel writes
NAN32 = np.uint32(0x7FC0BAD5)
MAX_CTX = 2048
PAD = 64                             # sentinel floats on each side of the output
MARGIN = 4.0

POSITIONS = [0, 1, 14, 15, 16, 17, 575, 576, MAX_CTX - 1]
SHAPES = [(64, 1), (64, 4), (64, 8), (128, 1), (128, 4), (128, 8)]      # (head_dim, GQA group); 2 KV heads


# ---- float64 reference ------------------------------------------------------------------------------------------------------
TOL = 1e-4          # |O - O_ref| <= TOL * max|V| of the head's KV head (fp32 math on fp16 K / V)


def decode_attention(q, k, v, pos, n_head, n_kv, hd, scale, n_splits=16, mutant=None):
    """softmax(q k^T scale) v of the token at position `pos` over keys 0 .. pos.  q [n_head, hd], k / v [>= pos + 1, n_kv, hd]
    (logical rows).  Returns [n_head, hd].  Mutants: 'drop_split' (the pages of split 1 -- pages p with p % n_splits == 1 --
    never visited), 'stale_newest' (row pos still holds zeros: read before the QKV epilogue appended it), 'page_off_by_one' (the
    newest page's rows read from the page before it)."""
    n = pos + 1
    kk = np.array(k[:n], dtype=np.float64)
    vv = np.array(v[:n], dtype=np.float64)
    keep = np.ones(n, dtype=bool)
    last = pos // 16 * 16
    if mutant == "drop_split":
        keep = (np.arange(n) // 16) % n_splits != 1
    elif mutant == "stale_newest":
        kk[pos] = 0.0
        vv[pos] = 0.0
    elif mutant == "page_off_by_one":
        kk[last:n] = np.asarray(k[last - 16:last - 16 + n - last], dtype=np.float64)
        vv[last:n] = np.asarray(v[last - 16:last - 16 + n - last], dtype=np.float64)
    grp = n_head // n_kv
    out = np.zeros((n_head, hd))
    for h in range(n_head):
        s = (kk[:, h // grp] @ np.asarray(q[h], dtype=np.float64)) * scale
        s = np.where(keep, s, -np.inf)
        e = np.exp(s - s.max())
        out[h] = (e @ vv[:, h // grp]) / e.sum()
    return out


def decode_attention_check(got, ref, v, pos, n_head, n_kv):
    """worst error / bound ratio of O against O_ref"""
    grp = n_head // n_kv
    worst = 0.0
    for h in range(n_head):
        vmax = max(float(np.abs(np.asarray(v[:pos + 1, h // grp], dtype=np.float64)).max()), 1e-30)
        worst = max(worst, float(np.abs(got[h] - ref[h]).max() / (TOL * vmax)))
    return worst


def _case(hd, grp, pos, n_kv=2, peaked=False, seed=0):
    """q, logical K / V rows [pos + 1][n_kv][hd] (fp16 values), the shuffled page table and the poisoned caches"""
    rng = np.random.Generator(np.random.PCG64(1000 * hd + 100 * grp + pos + (7 if peaked else 0) + seed))
    n_head = n_kv * grp
    n = pos + 1
    k = rng.standard_normal((n, n_kv, hd)).astype(np.float16)
    v = rng.standard_normal((n, n_kv, hd)).astype(np.float16)
    q = rng.standard_normal((n_head, hd)).astype(np.float32)
    if peaked:      # even heads peak on the newest row, odd heads on a row of page 1 (split 1): one split dominates
        for h in range(n_head):
            r = pos if h % 2 == 0 else min(pos, 21)
            q[h] = 2.0 * k[r, h // grp].astype(np.float32)
    n_table = MAX_CTX // 16
    n_phys = n_table + 4
    table = rng.permutation(n_phys)[:n_table].astype(np.int32)
    return q, k, v, table, n_phys


def _caches(k, v, table, n_phys, row0):
    """[page][kv head][16][hd] fp16 caches holding the rows below row0; everything else NaN"""
    n_kv, hd = k.shape[1], k.shape[2]
    kc = np.full((n_phys, n_kv, 16, hd), NAN16, dtype=np.uint16)
    vc = kc.copy()
    for r in range(row0):
        kc[table[r // 16], :, r % 16] = k[r].view(np.uint16)
        vc[table[r // 16], :, r % 16] = v[r].view(np.uint16)
    return kc, vc


@pytest.fixture(scope="module")
def kc():
    out = os.path.join(ROOT, "tests", "attncheck", "libattncheck.so")
    assert os.path.exists(out), "tests/attncheck/libattncheck.so is missing (run __graft_entry__.build())"
    lib = ctypes.CDLL(out)
    P, Z, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.ac_attn_decode.argtypes = [P, Z, P, P, Z, P, I, P, P, Z, I, I, I, I, I, I, ctypes.c_float, P, Z, Z, I, ctypes.c_uint, P]
    return lib


def _run(kc, q, k, v, table, n_phys, pos, row0, n_splits, reps=1):
    n_head, hd = q.shape
    n_kv = k.shape[1]
    kcache, vcache = _caches(k, v, table, n_phys, row0)
    krows = np.ascontiguousarray(k[row0:pos + 1])
    vrows = np.ascontiguousarray(v[row0:pos + 1])
    n_out = n_head * hd + 2 * PAD
    out = np.full(n_out, NAN32, dtype=np.uint32)
    out_all = np.zeros((reps, n_out), dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = kc.ac_attn_decode(p(q), q.nbytes, p(kcache), p(vcache), kcache.nbytes, p(table), len(table), p(krows), p(vrows), krows.nbytes,
                           row0, pos, n_head, n_kv, hd, n_splits, 1.0 / np.sqrt(hd), p(out), n_out, PAD, reps, 20000, p(out_all))
    assert rc == 0, rc
    assert (out_all[:, :PAD] == NAN32).all() and (out_all[:, -PAD:] == NAN32).all(), "write outside attn_"
    return out_all[:, PAD:-PAD].view(np.float32).reshape(reps, n_head, hd)


@pytest.mark.gpu
@pytest.mark.parametrize("pos", POSITIONS)
@pytest.mark.parametrize("hd,grp", SHAPES)
def test_decode_attention_matches_reference(kc, hd, grp, pos):
    """16 splits (the default), only the newest row pending; replays bit-identical"""
    q, k, v, table, n_phys = _case(hd, grp, pos)
    got = _run(kc, q, k, v, table, n_phys, pos, pos, 16, reps=3)
    assert np.isfinite(got).all()
    assert (got.view(np.uint32) == got[0].view(np.uint32)).all(), "replays differ"
    ref = decode_attention(q, k, v, pos, q.shape[0], k.shape[1], hd, 1.0 / np.sqrt(hd))
    assert decode_attention_check(got[0], ref, v, pos, q.shape[0], k.shape[1]) <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("pos", [1, 17, 576, MAX_CTX - 1])
@pytest.mark.parametrize("n_splits", [8, 16])
@pytest.mark.parametrize("hd,grp", [(64, 8), (128, 4)])
def test_decode_attention_stale_position_and_peaks(kc, hd, grp, pos, n_splits):
    """8 and 16 splits (2047 at 8 splits: a second staging tile per split), peaked scores, and a position read before the
    wait that is behind by up to 20 rows (rows >= it fetched again after the wait)"""
    q, k, v, table, n_phys = _case(hd, grp, pos, peaked=True)
    ref = decode_attention(q, k, v, pos, q.shape[0], k.shape[1], hd, 1.0 / np.sqrt(hd))
    for row0 in sorted({pos, max(0, pos - 1), max(0, pos - 20)}):
        got = _run(kc, q, k, v, table, n_phys, pos, row0, n_splits)[0]
        assert np.isfinite(got).all(), row0
        assert decode_attention_check(got, ref, v, pos, q.shape[0], k.shape[1]) <= 1.0, row0


@pytest.mark.gpu
def test_decode_attention_8b_shape(kc):
    """Llama-3-8B's layout: 8 KV heads, group 4, head dim 128, at the benchmarked context"""
    q, k, v, table, n_phys = _case(128, 4, 576, n_kv=8, peaked=True)
    got = _run(kc, q, k, v, table, n_phys, 576, 576, 16, reps=2)
    assert (got.view(np.uint32) == got[0].view(np.uint32)).all()
    ref = decode_attention(q, k, v, 576, 32, 8, 128, 1.0 / np.sqrt(128))
    assert decode_attention_check(got[0], ref, v, 576, 32, 8) <= 1.0


@pytest.mark.parametrize("pos", [17, 576, MAX_CTX - 1])
@pytest.mark.parametrize("hd,grp", [(64, 8), (128, 4)])
def test_decode_attention_mutants_are_caught(hd, grp, pos):
    """on the peaked inputs of the GPU test, every mutant lands >= 4x the tolerance from the reference"""
    q, k, v, _, _ = _case(hd, grp, pos, peaked=True)
    args = (q, k, v, pos, q.shape[0], k.shape[1], hd, 1.0 / np.sqrt(hd))
    ref = decode_attention(*args)
    for n_splits in (8, 16):
        for mutant in ("drop_split", "stale_newest", "page_off_by_one"):
            d = decode_attention_check(decode_attention(*args, n_splits=n_splits, mutant=mutant), ref, v, pos, q.shape[0], k.shape[1])
            assert d >= MARGIN, (mutant, n_splits, d)
