"""float64 references of the tensor-core kernels, for tests/test_gpu_kernels.py (one kernel at a time) and
tests/test_kernel_ref_cpu.py (which pins these references and shows the GPU checks have teeth).

Every reference works on the exact 16-bit values the kernel reads and accumulates in float64.  Each one takes an optional
`mutant`: a named, deliberately wrong variant of the same operation (a kernel bug the GPU check must not let through).
The per-element bounds are the ones DESIGN.md section 2 states:
  * 16-bit-input GEMMs and qgemm: |C - C_ref| <= 1e-4 (|A| |B|^T)_mn (+ one ulp of a 16-bit output), rel-L2 <= 1e-5;
  * prompt attention: |O - O_ref| <= 2^-9 max|V| per head, rel-L2 <= 1e-3."""
import ctypes

import numpy as np

GEMM_EPI_F32, GEMM_EPI_ADD_F32, GEMM_EPI_T16, GEMM_EPI_SILU, GEMM_EPI_ROPE_SPLIT = 0, 1, 2, 3, 4
KV_PAGE = 16
GEMM_ELEM_TOL, GEMM_REL_L2 = 1e-4, 1e-5
ATTN_ELEM_TOL, ATTN_REL_L2 = 2.0 ** -9, 1e-3


# ---- 16-bit formats -------------------------------------------------------------------------------------------------
def to_bf16_bits(x):
    """float32 -> bf16 bits (round to nearest even)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return u.astype(np.uint16)


def bf16_bits_to_f64(b):
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def ulp16(x, bf16=False):
    """one ulp of the 16-bit output format at |x| (subnormal floor included)"""
    ax = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** (-126 if bf16 else -14))
    return 2.0 ** (np.floor(np.log2(ax)) - (7 if bf16 else 10))


def rel_l2(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# ---- GEMM: C = A B^T ------------------------------------------------------------------------------------------------
def gemm(a, b, mutant=None, drop_kblock=0):
    """a [m, k], b [n, k] (float64 copies of the 16-bit inputs) -> (C, |A||B|^T).
    mutant 'drop_kblock': K columns [64 j, 64 j + 64) left out (a lost K-step of the pipeline)."""
    if mutant == "drop_kblock":
        a = a.copy()
        a[:, 64 * drop_kblock:64 * drop_kblock + 64] = 0.0
    elif mutant is not None:
        raise ValueError(mutant)
    return a @ b.T, np.abs(a) @ np.abs(b).T


def silu_ref(c, bound, mutant=None):
    """C columns interleaved [8 gate | 8 up] -> hidden [m, n / 2] = silu(gate) * up, and its error bound from the bound of C.
    mutant 'swap_gate_up': silu(up) * gate."""
    m, n = c.shape
    g = c.reshape(m, n // 16, 2, 8)[:, :, 0, :].reshape(m, n // 2)
    u = c.reshape(m, n // 16, 2, 8)[:, :, 1, :].reshape(m, n // 2)
    bg = bound.reshape(m, n // 16, 2, 8)[:, :, 0, :].reshape(m, n // 2)
    bu = bound.reshape(m, n // 16, 2, 8)[:, :, 1, :].reshape(m, n // 2)
    if mutant == "swap_gate_up":
        g, u = u, g
    elif mutant is not None:
        raise ValueError(mutant)
    sg = g / (1.0 + np.exp(-g))
    # |d silu / dg| <= 1.1: propagate the per-element accumulation bound of both operands
    return sg * u, 1.1 * bg * np.abs(u) + np.abs(sg) * bu


def rope_rows(x, pos, cos_t, sin_t, hd):
    """adjacent pairs (x[2i], x[2i+1]) of every head of rows x [rows, heads * hd] rotated by the fp32 tables at positions pos"""
    rows = x.shape[0]
    v = x.reshape(rows, -1, hd // 2, 2)
    c = cos_t[pos].astype(np.float64)[:, None, :]
    s = sin_t[pos].astype(np.float64)[:, None, :]
    out = np.empty_like(v)
    out[..., 0] = v[..., 0] * c - v[..., 1] * s
    out[..., 1] = v[..., 0] * s + v[..., 1] * c
    return out.reshape(rows, -1)


def seg_positions(m, segs, mutant=None):
    """absolute position of every row of a pack (-1: padding) and its segment (-1: none).  segs: (start, len, pos0) triples.
    mutant 'pos0+1' / 'pos0-1': every segment's pos0 off by one."""
    d = {"pos0+1": 1, "pos0-1": -1}.get(mutant, 0)
    pos = np.full(m, -1, np.int64)
    seg = np.full(m, -1, np.int64)
    for i, (s0, ln, p0) in enumerate(segs):
        lp = (ln + 127) // 128 * 128
        seg[s0:s0 + lp] = i
        pos[s0:s0 + ln] = max(p0 + d, 0) + np.arange(ln)
    return pos, seg


def rope_split(c, bound, n_head, n_kv, hd, cos_t, sin_t, segs, mutant=None):
    """GEMM_EPI_ROPE_SPLIT / rope_split_segs: the QKV accumulator [m, (n_head + 2 n_kv) hd] -> (q, k, v, their bounds, pos).
    Padding rows are zero."""
    qd, kvd = n_head * hd, n_kv * hd
    pos, _ = seg_positions(c.shape[0], segs, mutant)
    live = pos >= 0
    pz = np.where(live, pos, 0)
    q = np.where(live[:, None], rope_rows(c[:, :qd], pz, cos_t, sin_t, hd), 0.0)
    k = np.where(live[:, None], rope_rows(c[:, qd:qd + kvd], pz, cos_t, sin_t, hd), 0.0)
    v = np.where(live[:, None], c[:, qd + kvd:], 0.0)

    def pair_bound(b):      # a rotation mixes the two members of a pair: |err| <= err0 + err1
        r = b.reshape(b.shape[0], -1, 2)
        return np.repeat(r.sum(axis=2), 2, axis=1)
    return q, k, v, pair_bound(bound[:, :qd]), pair_bound(bound[:, qd:qd + kvd]), bound[:, qd + kvd:], pos


# ---- prompt attention -----------------------------------------------------------------------------------------------
def attention(q, k, v, pos0, n_head, n_kv, hd, scale, rows=None, mutant=None):
    """causal softmax(q k^T scale) v.  q [len, n_head * hd] at absolute positions pos0 .. pos0 + len - 1 (the query rows of one
    segment), k / v [kv_len, n_kv * hd] for positions 0 .. kv_len - 1; rows: the query rows to compute (None: all).
    Returns [len(rows), n_head * hd].  Mutants: 'diag' (col >= row masked: a query misses its own key), 'pos0+1' / 'pos0-1'
    (the mask of a shifted position), 'drop_last_kv_tile' (the last 64-key tile of every row never visited), 'gqa_mod'
    (KV head h % n_kv instead of h // group)."""
    ln = q.shape[0]
    rows = np.arange(ln) if rows is None else np.asarray(rows)
    grp = n_head // n_kv
    p = pos0 + rows
    if mutant == "pos0+1":
        p = p + 1
    elif mutant == "pos0-1":
        p = p - 1
    kv_len = k.shape[0]
    col = np.arange(kv_len)
    allowed = col[None, :] < p[:, None] if mutant == "diag" else col[None, :] <= p[:, None]
    if mutant == "drop_last_kv_tile":        # (rows whose diagonal lies in the first tile have no other tile: left alone)
        last = (pos0 + rows) // 64 * 64
        allowed &= (col[None, :] < last[:, None]) | (last[:, None] == 0)
    out = np.zeros((len(rows), n_head * hd))
    for h in range(n_head):
        kvh = h % n_kv if mutant == "gqa_mod" else h // grp
        qh = q[rows, h * hd:(h + 1) * hd]
        s = (qh @ k[:, kvh * hd:(kvh + 1) * hd].T) * scale
        s = np.where(allowed, s, -np.inf)
        s -= s.max(axis=1, keepdims=True)
        e = np.exp(s)
        e /= e.sum(axis=1, keepdims=True)
        out[:, h * hd:(h + 1) * hd] = e @ v[:, kvh * hd:(kvh + 1) * hd]
    return out


def attention_sample_rows(ln):
    """query rows of a long segment that the reference computes: the first and last row of every 128-row tile, both sides
    of every warp boundary (32 rows), the middle of every warp and the last rows; all rows up to 300"""
    if ln <= 300:
        return np.arange(ln)
    s = set()
    for b in range(0, ln, 32):
        s.update((b, b + 1, b + 31, b + 15, b + 16))
    s.update(range(max(0, ln - 3), ln))
    return np.array(sorted(x for x in s if 0 <= x < ln))


def attention_check(got, ref, v, n_head, n_kv, hd):
    """worst error / bound ratio of O against O_ref (bound 2^-9 max|V| of the head's KV head) and rel-L2"""
    worst = 0.0
    grp = n_head // n_kv
    for h in range(n_head):
        sl = slice(h * hd, (h + 1) * hd)
        kvh = h // grp
        vmax = max(float(np.abs(v[:, kvh * hd:(kvh + 1) * hd]).max()), 1e-30)
        worst = max(worst, float(np.abs(got[:, sl] - ref[:, sl]).max() / (ATTN_ELEM_TOL * vmax)))
    return worst, rel_l2(got, ref)


# ---- qgemm: the exact fp16 weights of the kernel's own unpack program ------------------------------------------------
Q4_K, Q6_K = 12, 14
BLOCK_BYTES = {Q4_K: 144, Q6_K: 210}


def packed_rows(srcs, mode):
    """(source index, source row) of every packed row.  srcs: [(blocks [rows, nkb, bb], type)].  mode 0: concatenation;
    mode 1: [8 gate | 8 up] interleave of two sources."""
    if mode == 1:
        n = 2 * srcs[0][0].shape[0]
        r = np.arange(n)
        return (r & 15) >> 3, (r >> 4) * 8 + (r & 7)
    si = np.concatenate([np.full(b.shape[0], i) for i, (b, _t) in enumerate(srcs)])
    sr = np.concatenate([np.arange(b.shape[0]) for b, _t in srcs])
    return si, sr


def qtile_weights(hc, srcs, mode, tile):
    """float64 [128, k] weights of packed tile `tile`, qtile by qtile from hc_qg_dequant (tests/hostcheck)"""
    si, sr = packed_rows(srcs, mode)
    rows = slice(tile * 128, tile * 128 + 128)
    tsrc = si[rows]
    assert (tsrc == tsrc[0]).all() or mode == 1
    typ = srcs[int(tsrc[0])][1]
    nkb = srcs[0][0].shape[1]
    w = np.empty((128, nkb * 256), np.float64)
    out = np.empty((128, 256), np.uint16)
    nbytes = ctypes.c_int(0)
    trow = sr[rows]
    for kb in range(nkb):
        blk = np.empty((128, BLOCK_BYTES[typ]), np.uint8)
        for s in np.unique(tsrc):
            sel = tsrc == s
            blk[sel] = srcs[int(s)][0][trow[sel], kb]
        rc = hc.hc_qg_dequant(typ, blk.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(nbytes))
        assert rc == 0
        w[:, kb * 256:(kb + 1) * 256] = out.view(np.float16)
    return w


def qgemm(hc, srcs, mode, act, mutant=None, drop=None):
    """C [nb, n] = act W^T and |act| |W|^T, one 128-row tile at a time.  act: float64 [nb, k].
    mutant 'drop_qtile' (drop = (tile, kb)): one 256-column qtile of one tile left out;
    'drop_partial' (drop = (tile, kb_lo, kb_hi)): one CTA's share [kb_lo, kb_hi) of a split tile left out."""
    n = sum(b.shape[0] for b, _t in srcs)
    c = np.empty((act.shape[0], n))
    bound = np.empty_like(c)
    aa = np.abs(act)
    for t in range(n // 128):
        w = qtile_weights(hc, srcs, mode, t)
        if mutant == "drop_qtile" and drop[0] == t:
            w[:, drop[1] * 256:(drop[1] + 1) * 256] = 0.0
        elif mutant == "drop_partial" and drop[0] == t:
            w[:, drop[1] * 256:drop[2] * 256] = 0.0
        elif mutant is not None and mutant not in ("drop_qtile", "drop_partial"):
            raise ValueError(mutant)
        c[:, t * 128:(t + 1) * 128] = act @ w.T
        bound[:, t * 128:(t + 1) * 128] = aa @ np.abs(w).T
    return c, bound


def norm_producer(x_new, gamma, n_tiles):
    """folded RMSNorm, producer side: xg = x_new gamma / 16 and the sums of squares per (tile, 32-row slice, token)
    ([n_tiles * 4, nb])"""
    nb = x_new.shape[0]
    xg = x_new * gamma[None, :] / 16.0
    ssq = (x_new * x_new).reshape(nb, n_tiles * 4, 32).sum(axis=2).T
    return xg, ssq


def norm_consumer_scale(ssq_parts, n_norm, eps, mutant=None):
    """per token: 16 / sqrt(sum of the parts / n + eps).  mutant 'no_rms': the factor left out"""
    if mutant == "no_rms":
        return np.ones(ssq_parts.shape[1])
    return 16.0 / np.sqrt(ssq_parts.sum(axis=0) / n_norm + eps)


# ---- how qgemm deals its qtiles to the CTAs (restated from qgemm.cu, used to assert what a test reaches) ---------------
def q_range_start(c, U, G):
    return c * U // G


def q_owner_of(x, U, G):
    return ((x + 1) * G + U - 1) // U - 1


def streamk_grid(n_tiles, nkb, n_sm):
    return min(n_sm, 132, n_tiles * nkb)


def streamk_patterns(n_tiles, nkb, n_sm):
    """sharing patterns of a stream-K launch: 'whole' (some CTA owns a tile's whole K range), 'shared3' (a tile shared by >= 3
    CTAs), 'span3' (a CTA's range touches >= 3 tiles)"""
    U = n_tiles * nkb
    G = streamk_grid(n_tiles, nkb, n_sm)
    pats = set()
    for c in range(G):
        u0, u1 = q_range_start(c, U, G), q_range_start(c + 1, U, G)
        if u1 > u0 and (u1 - 1) // nkb - u0 // nkb + 1 >= 3:
            pats.add("span3")
    for t in range(n_tiles):
        a, b = q_owner_of(t * nkb, U, G), q_owner_of(t * nkb + nkb - 1, U, G)
        if a == b:
            pats.add("whole")
        if b - a + 1 >= 3:
            pats.add("shared3")
    return pats


def streamk_partials(n_tiles, nkb, n_sm):
    """(tile, kb_lo, kb_hi) of every part of a split tile that a CTA other than its finisher computes"""
    U = n_tiles * nkb
    G = streamk_grid(n_tiles, nkb, n_sm)
    out = []
    for t in range(n_tiles):
        a, b = q_owner_of(t * nkb, U, G), q_owner_of(t * nkb + nkb - 1, U, G)
        for c in range(a + 1, b + 1):
            lo, hi = max(q_range_start(c, U, G), t * nkb), min(q_range_start(c + 1, U, G), t * nkb + nkb)
            if hi > lo:
                out.append((t, lo - t * nkb, hi - t * nkb))
    return out


def cluster_partials(nkb):
    """K-block quarters of a tile in cluster mode: rank r owns [r nkb / 4, (r + 1) nkb / 4)"""
    return [(r * nkb // 4, (r + 1) * nkb // 4) for r in range(4)]


def gemm_rel_l2_bound(k, out16=None):
    """rel-L2 bound of a K-deep 16-bit-input GEMM.  The tensor cores add in fp32 with truncation (up to 2^-23 per addition); on
    a random-sign sum the partial sums grow like sqrt(j), so the expected error relative to |C| is 2^-23 sqrt(K / 2) (1.0e-5
    at K = 14336, measured 1.2e-5 on an H100).  Bound: twice that, and never below 1e-5.  16-bit outputs add their own
    rounding: half an ulp relative, 2^-11 (fp16) or 2^-8 (bf16)."""
    b = max(GEMM_REL_L2, 2.0 ** -22 * np.sqrt(k / 2.0))
    return b + {None: 0.0, "fp16": 2.0 ** -11, "bf16": 2.0 ** -8}[out16]


def gemm_check(got, ref, bound, extra=0.0):
    """worst |got - ref| / (1e-4 bound + extra) and rel-L2"""
    tol = GEMM_ELEM_TOL * bound + extra + 1e-300
    return float((np.abs(np.asarray(got, np.float64) - ref) / tol).max()), rel_l2(got, ref)
