"""Inputs, float64 references and per-element bounds of the batch-1 decode GEMV (gemv.cu / gemv_core.cuh / rowdot.h) and of the
fp-weight decode route, shared by tests/test_gpu_decode_gemv.py (one launch at a time through tests/gemvcheck) and
tests/test_decode_gemv_cpu.py (the bounds rehearsed with the lane program on the CPU, and shown to have teeth).

Reference of one launch, in float64 (DESIGN.md section 2):
  x_hat = snap(fp32(x * norm_w)) per 32-column block, exactly as the prologue builds it (oracle snap_i16 / snap_q8);
  y_ref = rstd64 * W64 x_hat with W the dequantised GGUF values and rstd64 = 1 / sqrt(mean(x^2) + eps) (1 without a norm);
  then the epilogue in float64: residual add, silu(g) u, RoPE with the kernel's fp32 cos / sin rows, fp16 rounding of K and V.

Bound, per element: |y - y_ref| <= kappa 2^-24 rstd A_r + c_r |y_ref|.  Every 32-column block term of the lane program is an fp32
expression of exact dp4a integers and fp32 scales; A_r sums the magnitudes of the parts that are rounded separately (Q4_K: d sc q
and dmin m, which can cancel; Q6_K: d sc (q + 32), the q.v and 32.s16 parts; Q8_0: |d q|) against |x_hat|.  kappa counts the
roundings on the longest path: int -> float, x sx, x sc, the in-unit sums, x d, the Q4_K subtraction, one per K-segment in the
lane, five levels of warp_sum4 / warp_sum2, and x scale.  c_r is the fp32 rstd: the sum of squares (per thread, warp tree,
across warps), the square root and the division."""
import ctypes
import os

import numpy as np

from oracle import gguf_synth as S
from oracle import llama_oracle as O

Q4_K, Q6_K, Q8_0, F32, F16, BF16 = S.Q4_K, S.Q6_K, S.Q8_0, S.F32, S.F16, S.BF16
EPI_STORE, EPI_ADD, EPI_QKV, EPI_SILU = 0, 1, 2, 3
PAGE = 16
PAD = 64
U = 2.0 ** -24
ROPE_BASE = 500000.0
SENT32 = np.uint32(0x7FC0BAD5)         # sentinel bits around every output: a NaN no kernel writes
NAN16 = np.uint16(0x7E5A)
BIG = 64 << 20                         # elements: cases above this skip the CPU lane-program rehearsal
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def item_rows(t):
    return 4 if t == Q4_K else 2


def ksplit(cols):
    """rowdot.h ksplit(): (K-segments, 256-column blocks per segment); (0, 0) outside the envelope"""
    if cols <= 0 or cols % 256:
        return 0, 0
    nb = cols // 256
    nks = (nb + 15) // 16
    while nks <= 8 and nb % nks:
        nks += 1
    return (0, 0) if nks > 8 else (nks, nb // nks)


# ---- float64 dequantisation, with the magnitudes of the separately rounded parts ----------------------------------------------
_E = np.arange(256)
_Q6_QL = (_E >> 7) * 64 + (_E & 63)
_Q6_QLS = 4 * ((_E & 127) >> 6)
_Q6_QH = 128 + (_E >> 7) * 32 + (_E & 31)
_Q6_QHS = 2 * ((_E & 127) >> 5)


def _f16(b):
    return np.ascontiguousarray(b).view(np.float16)[..., 0].astype(np.float64)


def dequant_parts(blocks, t, cols):
    """GGUF rows [n][row bytes] -> (W, A) float64 [n][cols]: the values and the magnitudes the bound sums (module docstring)"""
    n = blocks.shape[0]
    if t == Q4_K:
        b = blocks.reshape(n, cols // 256, 144)
        d, dmin = _f16(b[..., 0:2]), _f16(b[..., 2:4])
        sc = b[..., 4:16].astype(np.int64)
        s = np.empty(sc.shape[:-1] + (8,), np.int64)
        m = np.empty_like(s)
        s[..., :4] = sc[..., 0:4] & 63
        m[..., :4] = sc[..., 4:8] & 63
        s[..., 4:] = (sc[..., 8:12] & 0xF) | ((sc[..., 0:4] >> 6) << 4)
        m[..., 4:] = (sc[..., 8:12] >> 4) | ((sc[..., 4:8] >> 6) << 4)
        qs = b[..., 16:].reshape(n, cols // 256, 4, 32).astype(np.int64)
        q = np.stack([qs & 0xF, qs >> 4], axis=3).reshape(n, cols // 256, 8, 32)
        main = d[..., None, None] * s[..., None] * q
        mn = (dmin[..., None] * m)[..., None] * np.ones(32)
        return (main - mn).reshape(n, cols), (np.abs(main) + np.abs(mn)).reshape(n, cols)
    if t == Q6_K:
        b = blocks.reshape(n, cols // 256, 210)
        d = _f16(b[..., 208:210])
        sc = b[..., 192:208].view(np.int8).astype(np.float64)
        qu = ((b[..., _Q6_QL] >> _Q6_QLS) & 0xF).astype(np.int64) | (((b[..., _Q6_QH] >> _Q6_QHS) & 3).astype(np.int64) << 4)
        ds = d[..., None] * sc[..., _E >> 4]
        return (ds * (qu - 32)).reshape(n, cols), (np.abs(ds) * (qu + 32)).reshape(n, cols)
    if t == Q8_0:
        b = blocks.reshape(n, cols // 32, 34)
        w = _f16(b[..., 0:2])[..., None] * b[..., 2:].view(np.int8).astype(np.float64)
        return w.reshape(n, cols), np.abs(w).reshape(n, cols)
    raise ValueError(t)


def snap(x, abits, block=32):
    """the prologue's activation fixed point (x fp32; block 256 only for the amax mutant)"""
    if block == 32:
        return O.snap_i16(x) if abits == 16 else O.snap_q8(x)
    rng = 16256.0 if abits == 16 else 127.0
    x32 = np.asarray(x, np.float32).reshape(-1, block)
    amax = np.abs(x32).max(axis=1, keepdims=True)
    sx = (amax / np.float32(rng)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(amax > 0, np.float32(rng) / amax, np.float32(0)).astype(np.float32)
    return (np.rint(x32 * inv).astype(np.float64) * sx).reshape(np.shape(x))


def drop_lo(x, abits):
    """the lo plane dropped: the 15-bit value keeps only 128 hi"""
    x32 = np.asarray(x, np.float32).reshape(-1, 32)
    amax = np.abs(x32).max(axis=1, keepdims=True)
    sx = (amax / np.float32(16256.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(amax > 0, np.float32(16256.0) / amax, np.float32(0)).astype(np.float32)
    v = np.rint(x32 * inv)
    return (128.0 * np.floor((v + 64) / 128) * sx).reshape(np.shape(x))


def kappa(nks):
    return 17 + nks


def rstd_rel(cols):
    """relative bound of the fp32 rstd: the longest sum-of-squares path over the 8 / 16 consumer-warp variants, halved by the
    square root, plus the sqrt, the mean and the division"""
    n_ss = max(cols / 256 + 13, cols / 512 + 21)
    return (n_ss / 2 + 3) * U


# ---- one launch ---------------------------------------------------------------------------------------------------------------
class GemvCase:
    """One decode GEMV launch.  types / rows: the 1-3 matrices (QKV: q, k, v; pair: gate, up).  x: 'normal', 'edges' (an all-zero
    block, a block with one outlier 10^4 x the rest, a block whose x inv lands on k + 1/2), 'outlier' (one value 10^4 x the rest of
    its 256 columns) or 'small' (mean(x^2) ~ 10 eps, so the
    norm's eps matters)."""

    def __init__(self, name, types, rows, cols, epi=EPI_STORE, pair=False, norm=False, abits=16, head_dim=128, n_kv=8, pos=0,
                 alias=False, polite=0, x="normal", seed=0):
        self.name, self.types, self.rows, self.cols = name, list(types), list(rows), cols
        self.epi, self.pair, self.norm, self.abits = epi, pair, norm, abits
        self.hd, self.n_kv, self.pos, self.alias, self.polite = head_dim, n_kv, pos, alias, polite
        self.eps = 1e-5
        self.x_kind = x
        self.nks = ksplit(cols)[0]
        rng = np.random.Generator(np.random.PCG64([seed, cols, sum(rows), epi, abits, pos, len(name)]))
        self.blocks = []
        for t, r in zip(self.types, self.rows):
            if r * cols > (1 << 22):
                self.blocks.append(S.random_blocks(rng, t, r, cols))
            else:
                self.blocks.append(S.quantize(rng.standard_normal((r, cols), dtype=np.float32) / np.float32(np.sqrt(cols)), t))
        xv = rng.standard_normal(cols).astype(np.float32)
        if x == "small":
            xv *= np.float32(1e-2)
        elif x == "outlier":
            xv[64 + 7] *= np.float32(1e4)                             # one block 10^4 x the rest of its 256 columns
        elif x == "edges":
            rng_top = 16256.0 if abits == 16 else 127.0
            xv[32:64] = 0.0                                           # all-zero block: inv = 0
            xv[64:96] *= np.float32(1e-4)
            xv[64 + 7] = np.float32(3.0)                              # outlier 10^4 x the rest of its block
            k = rng.integers(-int(rng_top) + 1, int(rng_top) - 1, size=31)
            xv[96] = np.float32(rng_top)                              # amax = RANGE: inv = 1 exactly, x inv = k + 1/2
            xv[97:128] = (k + 0.5).astype(np.float32)
            xv[128:160] = -xv[96:128]
        self.x = xv
        self.norm_w = (1.0 + 0.25 * rng.standard_normal(cols)).astype(np.float32) if norm else None
        self.resid = rng.standard_normal(self.rows[0]).astype(np.float32) if epi == EPI_ADD else None
        self.out_rows = self.rows[0]
        if epi == EPI_QKV:
            self.n_table = pos // PAGE + 3
            n_phys = self.n_table + 2
            perm = rng.permutation(n_phys).astype(np.int32)
            self.table = perm[:self.n_table].copy()
            self.decoy_pos = (pos // PAGE + 1) * PAGE + 5                   # in bounds; its page is NaN
            shape = (n_phys, n_kv, PAGE, head_dim)
            self.kc = np.full(shape, NAN16, np.uint16)
            self.vc = self.kc.copy()
            for lp in range(pos // PAGE + 1):                                # history (and a previous owner's row at pos)
                ph = self.table[lp]
                self.kc[ph] = rng.standard_normal(shape[1:]).astype(np.float16).view(np.uint16)
                self.vc[ph] = rng.standard_normal(shape[1:]).astype(np.float16).view(np.uint16)
            self.cos, self.sin = O.rope_table(self.decoy_pos + 2, head_dim, ROPE_BASE)
        else:
            self.table = self.kc = self.vc = self.cos = self.sin = None
            self.n_table, self.decoy_pos = 0, pos
        self._ref = None

    @property
    def elems(self):
        return sum(self.rows) * self.cols

    def gemv_ref(self, m, mutant=None):
        """(y, bound) of matrix m, float64, in row chunks of ~8 M elements"""
        chunk = max(64, (8 << 20) // self.cols)
        x = self.x
        xw = (x * self.norm_w).astype(np.float32) if self.norm else x
        if mutant == "lo_plane":
            xh = drop_lo(xw, self.abits)
        elif mutant == "amax256":
            xh = snap(xw, self.abits, 256)
        else:
            xh = snap(xw, self.abits)
        rstd = 1.0
        if self.norm:
            x64 = x.astype(np.float64)
            ms = (x64 * x64).sum() / (self.cols - 1 if mutant == "mean_k-1" else self.cols)
            rstd = 1.0 / np.sqrt(ms + (0.0 if mutant == "no_eps" else self.eps))
        t, rows, cols = self.types[m], self.rows[m], self.cols
        y, a = np.empty(rows), np.empty(rows)
        ax = np.abs(xh)
        drop = None
        if mutant == "drop_kseg":
            seg = cols // self.nks
            drop = slice((self.nks - 1) * seg, cols)
        for r0 in range(0, rows, chunk):
            w, aw = dequant_parts(self.blocks[m][r0:r0 + chunk], t, cols)
            if drop is not None and r0 == 0:
                w[:self.item_rows_of(m), drop] = 0.0                      # one K-segment of the first item
            y[r0:r0 + chunk] = w @ xh
            a[r0:r0 + chunk] = aw @ ax
        y *= rstd
        if mutant == "swap_rows":
            y[[0, 1]] = y[[1, 0]]
        if mutant == "drop_ragged":
            ir = self.item_rows_of(m)
            if rows % ir:
                y[rows - rows % ir:] = 0.0
        bound = kappa(self.nks) * U * rstd * a + (rstd_rel(cols) if self.norm else 0.0) * np.abs(y)
        return y, bound

    def item_rows_of(self, m):
        ir = item_rows(self.types[m])
        return ir // 2 if self.pair else ir

    def reference(self, mutant=None):
        """dict of float64 outputs and their bounds: 'out' (+ 'k', 'v' for QKV) -> (value, bound)"""
        if mutant is None and self._ref is not None:
            return self._ref
        ys = [self.gemv_ref(m, mutant) for m in range(len(self.types))]
        y, b = ys[0]
        res = {}
        if self.epi == EPI_STORE:
            res["out"] = (y, b)
        elif self.epi == EPI_ADD:
            r = self.resid.astype(np.float64) if mutant != "no_resid" else 0.0
            o = r + y
            res["out"] = (o, b + U * np.abs(o))
        elif self.epi == EPI_SILU:
            g, bg = ys[0]
            u, bu = ys[1]
            if mutant == "swap_gate_up":
                g, u = u, g
            sg = g / (1.0 + np.exp(-g))
            o = sg * u
            res["out"] = (o, 1.1 * bg * np.abs(u) + np.abs(sg) * bu + 1.1 * bg * bu + 8 * U * np.abs(o))
        else:
            pos = self.pos + {"pos+1": 1, "pos-1": -1}.get(mutant, 0)
            q, bq = ys[0]
            k, bk = ys[1]
            v, bv = ys[2]
            qr, qb = self._rope(q, bq, pos, mutant)
            kr, kb = self._rope(k, bk, pos, mutant)
            k16 = kr.astype(np.float16).astype(np.float64)
            v16 = v.astype(np.float16).astype(np.float64)
            res["out"] = (qr, qb)
            res["k"] = (kr, kb + ulp16(kr))
            res["v"] = (v, bv + ulp16(v))
            res["k16"], res["v16"] = k16, v16
        if mutant is None:
            self._ref = res
        return res

    def _rope(self, y, b, pos, mutant):
        """adjacent pairs (2i, 2i + 1) of every head rotated by the fp32 table row pos; the bound of a member is the sum of both
        members' bounds (|cos|, |sin| <= 1) plus the three roundings of the rotation.  mutant 'neox': pairs (i, i + hd / 2)."""
        hd = self.hd
        c = self.cos[pos].astype(np.float64)
        s = self.sin[pos].astype(np.float64)
        if mutant == "sin_sign":
            s = -s
        if mutant == "neox":
            v = y.reshape(-1, 2, hd // 2).transpose(0, 2, 1)
            bb = b.reshape(-1, 2, hd // 2).transpose(0, 2, 1)
        else:
            v = y.reshape(-1, hd // 2, 2)
            bb = b.reshape(-1, hd // 2, 2)
        o = np.empty_like(v)
        o[..., 0] = v[..., 0] * c - v[..., 1] * s
        o[..., 1] = v[..., 0] * s + v[..., 1] * c
        pb = bb[..., 0] + bb[..., 1] + 3 * U * (np.abs(v[..., 0]) + np.abs(v[..., 1]))
        pb = np.repeat(pb[..., None], 2, axis=-1)
        if mutant == "neox":
            o, pb = o.transpose(0, 2, 1), pb.transpose(0, 2, 1)
        return o.reshape(-1), pb.reshape(-1)

    def slot(self, kvh):
        """(physical page, slot) the launch writes for KV head kvh"""
        return int(self.table[self.pos // PAGE]), self.pos % PAGE

    def cache_rows(self, cache):
        """the rows at pos of every KV head from a cache [page][kv][16][hd] (uint16) -> float64 [n_kv hd]"""
        ph, t = self.slot(0)
        return cache[ph, :, t, :].view(np.float16).astype(np.float64).reshape(-1)


def ulp16(x):
    ax = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(ax)) - 10)


def ratio(got, ref_bound):
    ref, bound = ref_bound
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / bound))


def check_pool(case, kc, vc):
    """True when the K / V caches differ from the inputs only in slot pos % 16 of page table[pos / 16], for each KV head"""
    keep = np.ones(case.kc.shape, bool)
    ph, t = case.slot(0)
    keep[ph, :, t, :] = False
    return bool((kc[keep] == case.kc[keep]).all() and (vc[keep] == case.vc[keep]).all())


# ---- the case matrix ----------------------------------------------------------------------------------------------------------
def cases():
    C = []
    add = lambda *a, **k: C.append(GemvCase(*a, **k))
    # Llama-3-8B
    for tv in (Q4_K, Q6_K):
        add(f"8b-qkv-v{tv}", [Q4_K, Q4_K, tv], [4096, 1024, 1024], 4096, EPI_QKV, norm=True, x="small", pos=575)
    add("8b-attn_output", [Q4_K], [4096], 4096, EPI_ADD, alias=True, polite=3)
    add("8b-gate_up", [Q4_K, Q4_K], [14336, 14336], 4096, EPI_SILU, pair=True, norm=True)
    for t in (Q6_K, Q4_K):
        add(f"8b-ffn_down-{t}", [t], [4096], 14336, EPI_ADD)
    add("8b-lm_head", [Q6_K], [128256], 4096, norm=True)
    # Llama-3-70B
    add("70b-qkv", [Q4_K, Q4_K, Q6_K], [8192, 1024, 1024], 8192, EPI_QKV, norm=True, pos=2047)
    add("70b-attn_output", [Q4_K], [8192], 8192, EPI_ADD, alias=True, polite=3)
    add("70b-gate_up", [Q4_K, Q4_K], [28672, 28672], 8192, EPI_SILU, pair=True, norm=True)
    add("70b-ffn_down", [Q6_K], [8192], 28672, EPI_ADD)
    add("70b-lm_head", [Q6_K], [128256], 8192, norm=True)
    # Q8_0
    add("q8-qkv", [Q8_0, Q8_0, Q8_0], [4096, 1024, 1024], 4096, EPI_QKV, norm=True, pos=17)
    add("q8-gate_up", [Q8_0, Q8_0], [14336, 14336], 4096, EPI_SILU, pair=True, norm=True)
    # edges
    for r in (1, 2, 3, 5, 4097):
        add(f"rows{r}-q4k", [Q4_K], [r], 4096, x="edges")
        add(f"rows{r}-q6k", [Q6_K], [r], 4096)
    add("outlier-q4k", [Q4_K], [256], 4096, x="outlier")
    add("k256-norm", [Q4_K], [512], 256, norm=True, x="small")
    add("k256-q6k", [Q6_K], [512], 256, x="edges")
    add("k8192-norm", [Q6_K], [1024], 8192, norm=True)
    add("k32768", [Q4_K], [1024], 32768, x="edges")
    add("k32768-q6k", [Q6_K], [512], 32768, EPI_ADD)
    for hd, nkv, pos in ((64, 1, 0), (64, 2, 15), (128, 2, 16), (128, 1, 17), (64, 8, 2047)):
        add(f"qkv-hd{hd}-kv{nkv}-p{pos}", [Q4_K, Q4_K, Q6_K], [nkv * hd * 4, nkv * hd, nkv * hd], 2048, EPI_QKV, norm=True,
            head_dim=hd, n_kv=nkv, pos=pos)
    add("qkv-a8", [Q4_K, Q4_K, Q6_K], [4096, 1024, 1024], 4096, EPI_QKV, norm=True, abits=8, pos=16)
    add("lm_head-a8", [Q6_K], [32768], 4096, norm=True, abits=8)
    add("edges-a8", [Q4_K], [256], 4096, abits=8, x="edges")
    add("gate_up-ragged", [Q4_K, Q4_K], [1030, 1030], 4096, EPI_SILU, pair=True, norm=True)
    add("gate_up-q6k-k8192", [Q6_K, Q6_K], [2050, 2050], 8192, EPI_SILU, pair=True)
    return C


MUTANTS = ("drop_kseg", "swap_rows", "drop_ragged", "lo_plane", "amax256", "no_eps", "mean_k-1", "pos+1", "pos-1", "sin_sign",
           "neox", "swap_gate_up", "no_resid")


def mutant_applies(case, mutant):
    if mutant == "drop_kseg":
        return case.nks > 1
    if mutant == "drop_ragged":
        return case.rows[0] % case.item_rows_of(0) != 0
    if mutant == "swap_rows":
        return case.rows[0] >= 2 and case.epi in (EPI_STORE, EPI_ADD)
    if mutant == "lo_plane":        # a 2^-8 relative change per block: seen on the worst of a few dozen rows
        return case.abits == 16 and case.rows[0] >= 16
    if mutant == "amax256":          # visible where a block's scale matters: next to an outlier, or at 8 bits
        return case.x_kind == "outlier" or (case.abits == 8 and case.x_kind != "edges")
    if mutant == "no_eps":
        return case.norm and float(np.mean(case.x.astype(np.float64) ** 2)) < 100 * case.eps
    if mutant == "mean_k-1":
        return case.norm and case.cols <= 256
    if mutant in ("pos+1", "pos-1", "sin_sign", "neox"):
        return case.epi == EPI_QKV and (case.pos > 0 or mutant == "pos+1")        # position 0 does not rotate
    if mutant == "swap_gate_up":
        return case.epi == EPI_SILU
    if mutant == "no_resid":
        return case.epi == EPI_ADD
    raise ValueError(mutant)


def mutant_distance(case, mutant):
    """the largest |mutant - ref| / bound over the outputs the mutant changes"""
    ref = case.reference()
    mut = case.reference(mutant)
    d = 0.0
    for key in ("out", "k", "v"):
        if key not in ref:
            continue
        r, b = ref[key]
        m = mut[key][0]
        d = max(d, float(np.max(np.abs(m - r) / b)))
    return d


# ---- the shim's entry points (tests/gemvcheck/gemvcheck.cu) -------------------------------------------------------------------
GC_GEMV_ARGS = ("w0", "w1", "w2", "types", "rows", "nmat", "pair", "cols", "epi", "norm_w", "eps", "x", "resid", "alias", "rope_cos",
                "rope_sin", "rope_floats", "head_dim", "n_kv", "table", "n_table", "kc", "vc", "cache_bytes", "pos", "decoy_pos",
                "abits", "nw", "n_ctas", "pdl", "geom_in", "reps", "delay_ns", "out_init", "out_floats", "pad", "out_all", "kc_all",
                "vc_all", "resid_all", "geom_out")
STEP_STATE_BYTES = 108


def load_shim():
    from gridllm_b200 import native
    native.load_library()
    path = os.path.join(ROOT, "tests", "gemvcheck", "libgemvcheck.so")
    assert os.path.exists(path), "tests/gemvcheck/libgemvcheck.so is missing (run __graft_entry__.build())"
    lib = ctypes.CDLL(path)
    assert lib.gc_state_bytes() == STEP_STATE_BYTES
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def run_gemv(lib, case, nw=12, n_ctas=132, pdl=True, n_tracks=-1, depth=-1, polite=None, pro=-1, lean=-1, reps=2, delay_ns=20000):
    """one launch configuration of a case, reps times.  Returns (rc, result dict): 'out' [reps][out_rows + 2 PAD] uint32 bits,
    'kc' / 'vc' [reps] caches, 'resid' [reps][rows] or None, 'geom' (n_tracks, depth, slot_bytes, prologue, nks)."""
    Z, I, F = ctypes.c_size_t, ctypes.c_int, ctypes.c_float
    n_out = case.out_rows
    out_init = np.full(n_out + 2 * PAD, SENT32, np.uint32)
    if case.alias:
        out_init[PAD:PAD + n_out] = np.float32(np.nan).view(np.uint32)
    out_all = np.zeros((reps, out_init.size), np.uint32)
    kc_all = vc_all = None
    cache_bytes = 0
    if case.kc is not None:
        kc_all = np.zeros((reps,) + case.kc.shape, np.uint16)
        vc_all = np.zeros_like(kc_all)
        cache_bytes = case.kc.nbytes
    resid_all = np.zeros((reps, case.rows[0]), np.float32) if (case.resid is not None and not case.alias) else None
    geom_in = np.array([n_tracks, depth, case.polite if polite is None else polite, pro, lean], np.int32)
    geom_out = np.zeros(5, np.int32)
    ws = [np.ascontiguousarray(b) for b in case.blocks] + [None] * (3 - len(case.blocks))
    types = np.array(case.types + [0] * (3 - len(case.types)), np.int32)
    rows = np.array(case.rows + [0] * (3 - len(case.rows)), np.int32)
    args = dict(w0=_p(ws[0]), w1=_p(ws[1]), w2=_p(ws[2]), types=_p(types), rows=_p(rows), nmat=I(len(case.types)), pair=I(int(case.pair)),
                cols=I(case.cols), epi=I(case.epi), norm_w=_p(case.norm_w), eps=F(case.eps), x=_p(case.x), resid=_p(case.resid),
                alias=I(int(case.alias)), rope_cos=_p(case.cos), rope_sin=_p(case.sin), rope_floats=Z(0 if case.cos is None else case.cos.size),
                head_dim=I(case.hd), n_kv=I(case.n_kv), table=_p(case.table), n_table=I(case.n_table), kc=_p(case.kc), vc=_p(case.vc),
                cache_bytes=Z(cache_bytes), pos=I(case.pos), decoy_pos=I(case.decoy_pos), abits=I(case.abits), nw=I(nw),
                n_ctas=I(n_ctas), pdl=I(int(pdl)), geom_in=_p(geom_in), reps=I(reps), delay_ns=ctypes.c_uint(delay_ns),
                out_init=_p(out_init), out_floats=Z(n_out), pad=Z(PAD), out_all=_p(out_all), kc_all=_p(kc_all), vc_all=_p(vc_all),
                resid_all=_p(resid_all), geom_out=_p(geom_out))
    rc = lib.gc_gemv(*[args[a] for a in GC_GEMV_ARGS])
    return rc, dict(out=out_all, kc=kc_all, vc=vc_all, resid=resid_all, geom=tuple(int(g) for g in geom_out))
