"""Kernel-level check of the context shift of the paged KV cache (kv_shift.cu, kv_shift_launch) through the launcher shim
tests/shiftcheck.

Every case runs on a shuffled page table over a pool whose unused page slots are NaN-poisoned, with sentinels around both
caches and around the step states.  Each moved K element must be within one fp16 ulp of float64 R(-d) K computed with the same
fp32 cos / sin table; V must move bit for bit; rows [0, k), the pages of sequences not in the launch and every sentinel must come
back bit-unchanged; pos must drop by d; two launches on the same inputs must be bit-identical.  A discard smaller than the moved
range takes the chunked launches (rows in blocks of at most d, in increasing order)."""
import ctypes
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN16 = np.uint16(0x7E5A)
SENT32 = np.int32(0x5EAD5EAD)
PAD = 4096                 # sentinel bytes before and after each cache
N_LAYER = 2
N_CTX = 256                # rows of the cos / sin table and of each sequence's logical context


def _lib():
    from gridllm_b200 import native
    native.load_library()
    path = os.path.join(ROOT, "tests", "shiftcheck", "libshiftcheck.so")
    if not os.path.exists(path):
        pytest.fail("tests/shiftcheck/libshiftcheck.so missing: __graft_entry__.build() builds it")
    lib = ctypes.CDLL(path)
    lib.sc_kv_shift.restype = ctypes.c_int
    return lib


def _run(hd, n_kv, seqs, other_seq=True, reps=2, seed=0):
    """seqs: list of (W, keep, discard).  Returns a dict of every check's inputs / outputs."""
    from oracle import llama_oracle as O
    lib = _lib()
    rng = np.random.Generator(np.random.PCG64(10_000 + 100 * hd + 10 * n_kv + len(seqs) + seed))
    cos, sin = O.rope_table(N_CTX, hd, 10000.0)
    pages_per_seq = N_CTX // 16
    n_seq_all = len(seqs) + (1 if other_seq else 0)
    pool = n_seq_all * pages_per_seq + 5                  # a few pages nobody owns (poisoned)
    perm = rng.permutation(pool)
    tables = perm[: n_seq_all * pages_per_seq].reshape(n_seq_all, pages_per_seq).astype(np.int32)
    layer_elems = pool * n_kv * 16 * hd
    nbytes = N_LAYER * layer_elems * 2
    kbuf = np.full(nbytes // 2 + 2 * PAD // 2, NAN16, dtype=np.uint16)
    vbuf = kbuf.copy()
    k = kbuf[PAD // 2: PAD // 2 + nbytes // 2].view(np.float16).reshape(N_LAYER, pool, n_kv, 16, hd)
    v = vbuf[PAD // 2: PAD // 2 + nbytes // 2].view(np.float16).reshape(N_LAYER, pool, n_kv, 16, hd)
    for s in range(n_seq_all):                             # every owned page gets values (unused pages stay NaN)
        for pg in tables[s]:
            k[:, pg] = rng.standard_normal((N_LAYER, n_kv, 16, hd)).astype(np.float16)
            v[:, pg] = rng.standard_normal((N_LAYER, n_kv, 16, hd)).astype(np.float16)
    sb = lib.sc_state_bytes()
    st_words = (sb // 4) * len(seqs) + 64
    st_buf = np.full(st_words, SENT32, dtype=np.int32)
    st_off = np.zeros(len(seqs), dtype=np.int64)
    for i, (W, _, _) in enumerate(seqs):
        off = 32 + i * (sb // 4)
        st_buf[off: off + sb // 4] = 0
        st_buf[off] = W                                    # StepState.pos
        st_off[i] = off * 4
    keep = np.array([s[1] for s in seqs], dtype=np.int32)
    disc = np.array([s[2] for s in seqs], dtype=np.int32)
    rows = np.array([s[0] - s[1] - s[2] for s in seqs], dtype=np.int32)
    kout = np.zeros((reps,) + kbuf.shape, dtype=np.uint16)
    vout = np.zeros_like(kout)
    sout = np.zeros((reps,) + st_buf.shape, dtype=np.int32)
    P = ctypes.c_void_p
    rc = lib.sc_kv_shift(P(kbuf.ctypes.data), P(vbuf.ctypes.data), ctypes.c_size_t(kbuf.nbytes), ctypes.c_size_t(PAD),
                         ctypes.c_size_t(layer_elems), N_LAYER, n_kv, hd, P(cos.ctypes.data), P(sin.ctypes.data),
                         ctypes.c_size_t(cos.size), P(tables.ctypes.data), pages_per_seq, P(keep.ctypes.data), P(disc.ctypes.data),
                         P(rows.ctypes.data), len(seqs), P(st_buf.ctypes.data), ctypes.c_size_t(st_buf.nbytes),
                         P(st_off.ctypes.data), reps, P(kout.ctypes.data), P(vout.ctypes.data), P(sout.ctypes.data))
    assert rc == 0, f"cudaError {rc}"
    return dict(kbuf=kbuf, vbuf=vbuf, kout=kout, vout=vout, st_buf=st_buf, sout=sout, st_off=st_off, tables=tables, cos=cos,
                sin=sin, pool=pool, n_kv=n_kv, hd=hd, seqs=seqs, layer_elems=layer_elems)


def _logical(buf, r, s):
    """[layer][row][kv][hd] of sequence s's logical rows 0 .. N_CTX - 1 in the cache buffer"""
    nbytes = N_LAYER * r["layer_elems"] * 2
    c = buf[PAD // 2: PAD // 2 + nbytes // 2].reshape(N_LAYER, r["pool"], r["n_kv"], 16, r["hd"])
    t = r["tables"][s]
    return c[:, t].transpose(0, 1, 3, 2, 4).reshape(N_LAYER, N_CTX, r["n_kv"], r["hd"])


def _check(r):
    from shift_oracle import rotate_back
    assert np.array_equal(r["kout"][0], r["kout"][1]) and np.array_equal(r["vout"][0], r["vout"][1]), "replays differ"
    assert np.array_equal(r["sout"][0], r["sout"][1])
    ko, vo = r["kout"][0], r["vout"][0]
    for buf_in, buf_out in ((r["kbuf"], ko), (r["vbuf"], vo)):      # sentinels
        assert np.array_equal(buf_in[: PAD // 2], buf_out[: PAD // 2]) and np.array_equal(buf_in[-PAD // 2:], buf_out[-PAD // 2:])
    touched = np.zeros(r["pool"], dtype=bool)
    for s, (W, keep, d) in enumerate(r["seqs"]):
        touched[r["tables"][s]] = True
        kin, vin = _logical(r["kbuf"], r, s), _logical(r["vbuf"], r, s)
        kgot, vgot = _logical(ko, r, s), _logical(vo, r, s)
        n = W - keep - d
        assert np.array_equal(kgot[:, :keep], kin[:, :keep]) and np.array_equal(vgot[:, :keep], vin[:, :keep]), "rows [0, k) changed"
        assert np.array_equal(vgot[:, keep: keep + n], vin[:, keep + d: W]), "V rows not moved bit for bit"
        assert np.array_equal(kgot[:, keep + n:], kin[:, keep + n:]) and np.array_equal(vgot[:, keep + n:], vin[:, keep + n:])
        if n > 0:
            src = kin[:, keep + d: W].view(np.float16).astype(np.float64)
            ref = rotate_back(src, d, r["cos"], r["sin"])
            got = kgot[:, keep: keep + n].view(np.float16).astype(np.float64)
            ulp = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float64)
            assert np.all(np.abs(got - ref) <= ulp), ("K", float(np.max(np.abs(got - ref) / ulp)))
        off = int(r["st_off"][s]) // 4
        assert r["sout"][0][off] == W - d, "pos not lowered by d"
        words = r["sout"][0][off + 1: off + lib_state_words()]
        assert np.array_equal(words, r["st_buf"][off + 1: off + lib_state_words()]), "other StepState fields changed"
    # step-state sentinels, and pages of sequences outside the launch (the last table when other_seq) / unowned pages
    mask = np.ones(r["st_buf"].shape, dtype=bool)
    for s in range(len(r["seqs"])):
        mask[int(r["st_off"][s]) // 4] = False
    assert np.array_equal(r["sout"][0][mask], r["st_buf"][mask])
    nbytes = N_LAYER * r["layer_elems"] * 2
    for buf_in, buf_out in ((r["kbuf"], ko), (r["vbuf"], vo)):
        a = buf_in[PAD // 2: PAD // 2 + nbytes // 2].reshape(N_LAYER, r["pool"], -1)
        b = buf_out[PAD // 2: PAD // 2 + nbytes // 2].reshape(N_LAYER, r["pool"], -1)
        assert np.array_equal(a[:, ~touched], b[:, ~touched]), "pages outside the launch changed"


def lib_state_words():
    return _lib().sc_state_bytes() // 4


@pytest.mark.parametrize("hd,n_kv", [(64, 1), (64, 4), (64, 8), (128, 1), (128, 4), (128, 8)])
@pytest.mark.parametrize("keep", [0, 1, 15, 16, 17])
def test_kv_shift_rule_discard(hd, n_kv, keep):
    """the rule's own discard (one launch: source and destination do not overlap)"""
    W = 160
    d = (W - keep + 1) // 2
    _check(_run(hd, n_kv, [(W, keep, d)]))


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("keep,d", [(0, 5), (1, 16), (17, 3), (15, 40)])
def test_kv_shift_chunked(hd, keep, d):
    """a discard smaller than the moved range: launches of at most d rows, in increasing order"""
    W = N_CTX
    assert d < W - keep - d
    _check(_run(hd, 4, [(W, keep, d)]))


@pytest.mark.parametrize("hd", [64, 128])
def test_kv_shift_several_sequences(hd):
    """several sequences of one launch, each with its own window, keep and discard (one of them chunked)"""
    seqs = [(N_CTX, 4, (N_CTX - 4 + 1) // 2), (96, 0, 48), (128, 17, 7), (64, 63, 1)]
    _check(_run(hd, 2, seqs))
