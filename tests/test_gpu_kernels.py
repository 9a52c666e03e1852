"""Kernel-level checks of the tensor-core GEMMs (gemm_tc5, gemm_tn), the GEMM on quantised weights (qgemm) and the prompt
attention kernel (flash_prefill, both instantiations) against the float64 references of tests/kernel_ref.py, through the
launcher shim tests/kernelcheck (host buffers in, every buffer the kernel may touch back out, sentinels included).

Tolerances (DESIGN.md section 2): GEMMs |C - C_ref| <= 1e-4 (|A||B|^T) per element (+ one ulp of a 16-bit output),
rel-L2 <= 1e-5; attention |O - O_ref| <= 2^-9 max|V| per head, rel-L2 <= 1e-3.  The worst error / bound ratio of every
family is printed (pytest -s) as `KERNELCHECK <family> <ratio>`."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import kernel_cases as KC
import kernel_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN16 = np.uint16(0x7E5A)            # sentinel / poison bits: a quiet NaN no kernel writes
NAN32 = np.uint32(0x7FC0BAD5)
WORST = {}


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"KERNELCHECK {k} {WORST[k]:.4f}")


@pytest.fixture(scope="module")
def kc():
    """the launcher shim, rebuilt when stale and nvcc is there; a missing library is a failure"""
    d = os.path.join(ROOT, "tests", "kernelcheck")
    out = os.path.join(d, "libkernelcheck.so")
    deps = [os.path.join(d, "kernelcheck.cu"), os.path.join(ROOT, "gridllm_b200", "csrc", "prefill.h"),
            os.path.join(ROOT, "gridllm_b200", "csrc", "qgemm.h"), os.path.join(ROOT, "gridllm_b200", "libgridllm_native.so")]
    stale = not os.path.exists(out) or any(os.path.exists(p) and os.path.getmtime(p) > os.path.getmtime(out) for p in deps)
    if stale and os.path.exists("/usr/local/cuda/bin/nvcc"):
        subprocess.check_call(["make", "-C", d, "-B"])
    assert os.path.exists(out), "tests/kernelcheck/libkernelcheck.so is missing (run __graft_entry__.build())"
    lib = ctypes.CDLL(out)
    lib.kc_flash_prefill.argtypes = [ctypes.c_void_p, ctypes.c_size_t] * 4 + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + \
        [ctypes.c_int] * 4 + [ctypes.c_float] + [ctypes.c_int] + [ctypes.c_void_p] * 5 + [ctypes.c_size_t]
    lib.kc_qgemm.argtypes = None
    return lib


def _p(x):
    return None if x is None else x.ctypes.data_as(ctypes.c_void_p)


def _nb(x):
    return 0 if x is None else x.nbytes


def _segs_args(segs, tabs):
    """(nseg, start, len, pos0, tab_off, flat table) for the shim"""
    st = np.array([s[0] for s in segs], np.int32)
    ln = np.array([s[1] for s in segs], np.int32)
    p0 = np.array([s[2] for s in segs], np.int32)
    offs, flat, o = [], [], 0
    for t in tabs:
        if t is None:
            offs.append(-1)
        else:
            offs.append(o)
            flat.append(t)
            o += len(t)
    flat = np.concatenate(flat).astype(np.int32) if flat else None
    return len(segs), st, ln, p0, np.array(offs, np.int32), flat


# =============================================================================================================================
# GEMMs
# =============================================================================================================================
def _run_gemm(kc, which, bf16, epi, a_bits, a_rows_alloc, b_bits, m, n, k, ldc, cbuf, c_off):
    rc = kc.kc_gemm(ctypes.c_int(which), ctypes.c_int(bf16), ctypes.c_int(epi), _p(a_bits), ctypes.c_size_t(a_bits.nbytes), _p(b_bits),
                    ctypes.c_size_t(b_bits.nbytes), _p(cbuf), ctypes.c_size_t(cbuf.nbytes), ctypes.c_size_t(c_off), m, n, k, k, k, ldc,
                    a_rows_alloc, 1, ctypes.c_longlong(0), ctypes.c_longlong(0), ctypes.c_longlong(0), 1)
    assert rc == 0, ("kc_gemm", which, rc)


def _c_buffer(m, ldc, epi, old):
    """C with 64 bytes of sentinel in front and one sentinel row behind; returns (buffer, byte offset of C, view of C)"""
    if epi in (KC.T16, KC.SILU):
        pre = 32
        buf = np.full(pre + (m + 1) * ldc, NAN16, np.uint16)
    else:
        pre = 16
        buf = np.full(pre + (m + 1) * ldc, NAN32, np.uint32)
        if old is not None:
            view = buf[pre:pre + m * ldc].view(np.float32).reshape(m, ldc)
            view[:, :old.shape[1]] = old
    return buf, pre * buf.itemsize, buf[pre:pre + m * ldc].reshape(m, ldc)


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", KC.GEMM_CASES, ids=KC.gemm_case_id)
def test_gemm_matches_float64(kc, case, bf16):
    m, n, k, epi, kind = case
    a_bits, a, b_bits, b, old = KC.gemm_inputs(case, bf16)
    ref, bound = R.gemm(a, b)
    if epi == KC.SILU:
        ref, bound = R.silu_ref(ref, bound)
    elif epi == KC.ADD:
        ref = ref + old
    w = ref.shape[1]
    ldc = KC.ldc_of(n, epi, kind)
    # rows [m, a_rows_alloc) of A are NaN: no row below m may see them
    a_rows_alloc = m + 5
    a_full = np.full((a_rows_alloc, k), NAN16 if not bf16 else np.uint16(0x7FC1), np.uint16)
    a_full[:m] = a_bits
    for which in (0, 1):
        if which == 0:
            sup = kc.kc_gemm_tc5_supported(epi, m, n, k, k, k, ldc, ctypes.c_ulonglong(1 << 20), ctypes.c_ulonglong(1 << 21),
                                           ctypes.c_ulonglong(1 << 22))
            assert sup == 1, case
        buf, off, cview = _c_buffer(m, ldc, epi, old)
        before = buf.copy()
        _run_gemm(kc, which, bf16, epi, a_full if which == 0 else a_bits, a_rows_alloc if which == 0 else m, b_bits, m, n, k, ldc, buf, off)
        if epi in (KC.T16, KC.SILU):
            got = (R.bf16_bits_to_f64(cview[:, :w]) if (bf16 and epi == KC.T16) or (bf16 and epi == KC.SILU) else
                   cview[:, :w].view(np.float16).astype(np.float64))
            extra = R.ulp16(ref, bool(bf16))
        else:
            got = cview[:, :w].view(np.float32).astype(np.float64)
            extra = 2.0 ** -23 * np.abs(ref) if epi == KC.ADD else 0.0
        ratio, rl2 = R.gemm_check(got, ref, bound, extra)
        fam = f"gemm_{'tc5' if which == 0 else 'tn'}"
        relb = R.gemm_rel_l2_bound(k, ("bf16" if bf16 else "fp16") if epi in (KC.T16, KC.SILU) else None)
        _note(fam, ratio)
        _note(fam + "_relL2/bound", rl2 / relb)
        assert np.isfinite(got).all(), (fam, case)
        assert ratio <= 1.0, (fam, case, ratio)
        assert rl2 <= relb, (fam, case, rl2)
        # every byte outside rows < m, columns < n (the documented output) is unchanged
        mask = np.ones(buf.shape, bool)
        pre = off // buf.itemsize
        for r in range(m):
            mask[pre + r * ldc:pre + r * ldc + w] = False
        assert np.array_equal(buf[mask], before[mask]), (fam, case, "wrote outside C")


def test_gemm_slice_is_bit_identical(kc):
    """the rows of one 128-row slice computed alone equal the same rows of the full GEMM, for both kernels"""
    case = (2048, 1000, 200, KC.T16, "scalar")
    m, n, k, epi, kind = case
    a_bits, _a, b_bits, _b, _old = KC.gemm_inputs(case, 0)
    ldc = KC.ldc_of(n, epi, kind)
    for which in (0, 1):
        full, off, cv = _c_buffer(m, ldc, epi, None)
        _run_gemm(kc, which, 0, epi, a_bits, m, b_bits, m, n, k, ldc, full, off)
        part, off2, cv2 = _c_buffer(128, ldc, epi, None)
        sl = np.ascontiguousarray(a_bits[384:512])
        _run_gemm(kc, which, 0, epi, sl, 128, b_bits, 128, n, k, ldc, part, off2)
        assert np.array_equal(cv2[:, :n], cv[384:512, :n]), which


def test_gemm_tn_batched_gqa(kc):
    """gemm_tn with batch > 1 and b_batch_div = 2 (two query heads share one KV head), both input types"""
    batch, div, m, n, k = 4, 2, 200, 96, 128
    for bf16 in (0, 1):
        rng = np.random.Generator(np.random.PCG64(31 + bf16))
        a_bits, a = KC.operand(rng, batch * m, k, bf16)
        b_bits, b = KC.operand(rng, (batch // div) * n, k, bf16, 0.1)
        ldc = n + 4
        c = np.full(batch * m * ldc + 16, NAN32, np.uint32)
        rc = kc.kc_gemm(1, bf16, KC.F32, _p(a_bits), ctypes.c_size_t(a_bits.nbytes), _p(b_bits), ctypes.c_size_t(b_bits.nbytes), _p(c),
                        ctypes.c_size_t(c.nbytes), ctypes.c_size_t(0), m, n, k, k, k, ldc, m, batch, ctypes.c_longlong(m * k),
                        ctypes.c_longlong(n * k), ctypes.c_longlong(m * ldc), div)
        assert rc == 0
        for z in range(batch):
            ref, bound = R.gemm(a[z * m:(z + 1) * m], b[(z // div) * n:(z // div + 1) * n])
            got = c[z * m * ldc:(z + 1) * m * ldc].view(np.float32).reshape(m, ldc)[:, :n].astype(np.float64)
            ratio, rl2 = R.gemm_check(got, ref, bound)
            _note("gemm_tn", ratio)
            assert ratio <= 1.0 and rl2 <= R.gemm_rel_l2_bound(k), (bf16, z, ratio, rl2)
            assert (c[z * m * ldc:(z + 1) * m * ldc].reshape(m, ldc)[:, n:] == NAN32).all()
        assert (c[batch * m * ldc:] == NAN32).all()


def test_gemm_tc5_supported_refuses_what_the_epilogue_cannot_store(kc):
    """SiLU stores 16 bytes at c + row ldc: refused unless ldc % 8 == 0; any C base not 16-byte aligned is refused (the engine
    then runs gemm_tn).  No launch."""
    A, B, C = 1 << 20, 1 << 21, 1 << 22
    assert kc.kc_gemm_tc5_supported(KC.SILU, 128, 256, 256, 256, 256, 128, ctypes.c_ulonglong(A), ctypes.c_ulonglong(B), ctypes.c_ulonglong(C)) == 1
    assert kc.kc_gemm_tc5_supported(KC.SILU, 128, 256, 256, 256, 256, 132, ctypes.c_ulonglong(A), ctypes.c_ulonglong(B), ctypes.c_ulonglong(C)) == 0
    for epi in (KC.F32, KC.ADD, KC.T16, KC.SILU):
        assert kc.kc_gemm_tc5_supported(epi, 128, 256, 256, 256, 256, 128, ctypes.c_ulonglong(A), ctypes.c_ulonglong(B), ctypes.c_ulonglong(C + 8)) == 0
        assert kc.kc_gemm_tc5_supported(epi, 128, 256, 256, 256, 256, 128, ctypes.c_ulonglong(A), ctypes.c_ulonglong(B), ctypes.c_ulonglong(C)) == 1


# ---- RoPE / split: the QKV epilogue and the stand-alone kernel -----------------------------------------------------------------
def _rope_buffers(m, n_head, n_kv, hd, n_pages):
    qd, kvd = n_head * hd, n_kv * hd
    vt_ld = m + 8
    q = np.full((m + 1) * qd, NAN16, np.uint16)
    kk = np.full((m + 1) * kvd, NAN16, np.uint16)
    vt = np.full(kvd * vt_ld, NAN16, np.uint16)
    kc_ = np.full(n_pages * n_kv * 16 * hd, NAN16, np.uint16)
    vc_ = np.full(n_pages * n_kv * 16 * hd, NAN16, np.uint16)
    return q, kk, vt, kc_, vc_, vt_ld


def _check_rope_outputs(tag, bufs, before, ref, segs, tabs, m, n_head, n_kv, hd, tol_scale):
    q, kk, vt, kcache, vcache, vt_ld = bufs
    qr, kr, vr, bq, bk, bv, pos = ref
    qd, kvd = n_head * hd, n_kv * hd
    f16 = lambda x: x.view(np.float16).astype(np.float64)   # noqa: E731

    def chk(name, got, want, b):
        tol = tol_scale(b) + R.ulp16(want)
        ratio = float((np.abs(got - want) / tol).max())
        _note(tag, ratio)
        assert ratio <= 1.0, (tag, name, ratio)
    chk("q", f16(q[:m * qd]).reshape(m, qd), qr, bq)
    chk("k", f16(kk[:m * kvd]).reshape(m, kvd), kr, bk)
    chk("vt", f16(vt).reshape(kvd, vt_ld)[:, :m].T, vr, bv)
    assert (q[m * qd:] == NAN16).all() and (kk[m * kvd:] == NAN16).all() and (vt.reshape(kvd, vt_ld)[:, m:] == NAN16).all(), tag
    # cache: exactly the slots of the live rows, at table[pos // 16], slot pos % 16
    _, seg = R.seg_positions(m, segs)
    kc4 = kcache.reshape(-1, n_kv, 16, hd)
    vc4 = vcache.reshape(-1, n_kv, 16, hd)
    written = np.zeros(kc4.shape[:3], bool)
    for r in np.nonzero(pos >= 0)[0]:
        t = tabs[seg[r]]
        pg, sl = int(t[pos[r] // 16]), int(pos[r] % 16)
        written[pg, :, sl] = True
        for h in range(n_kv):
            assert np.array_equal(kc4[pg, h, sl], kk[r * kvd + h * hd:r * kvd + (h + 1) * hd]), (tag, "k cache", r)
            want = vr[r, h * hd:(h + 1) * hd]
            got = f16(vc4[pg, h, sl])
            assert (np.abs(got - want) <= tol_scale(bv[r, h * hd:(h + 1) * hd]) + R.ulp16(want)).all(), (tag, "v cache", r)
    assert np.array_equal(kcache.reshape(kc4.shape)[~written], before[3].reshape(kc4.shape)[~written]), tag
    assert np.array_equal(vcache.reshape(vc4.shape)[~written], before[4].reshape(vc4.shape)[~written]), tag


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("pos0", [0, 1, 17, 200])
def test_rope_split_epilogue_and_kernel(kc, pos0, hd):
    n_head, n_kv = KC.ROPE_HEADS
    m, k = KC.ROPE_M, 512
    n = (n_head + 2 * n_kv) * hd
    segs = KC.rope_segs(pos0)
    rng = np.random.Generator(np.random.PCG64(pos0 * 7 + hd))
    n_pages = 64
    tabs = KC.page_tables(rng, segs, n_pages)
    cos_t, sin_t = KC.rope_tables(hd, 512)
    nseg, st, ln, p0, toff, flat = _segs_args(segs, tabs)
    for bf16 in (0, 1):
        a_bits, a = KC.operand(rng, m, k, bf16)
        b_bits, b = KC.operand(rng, n, k, bf16, 1.0 / np.sqrt(k))
        c, bound = R.gemm(a, b)
        ref = R.rope_split(c, bound, n_head, n_kv, hd, cos_t, sin_t, segs)
        bufs = _rope_buffers(m, n_head, n_kv, hd, n_pages)
        before = [x.copy() for x in bufs[:5]]
        q, kk, vt, kcache, vcache, vt_ld = bufs
        rc = kc.kc_gemm_rope(bf16, _p(a_bits), ctypes.c_size_t(a_bits.nbytes), _p(b_bits), ctypes.c_size_t(b_bits.nbytes), m, n, k, k, k, m,
                             _p(cos_t), _p(sin_t), ctypes.c_size_t(cos_t.nbytes), _p(q), ctypes.c_size_t(q.nbytes), _p(kk), ctypes.c_size_t(kk.nbytes),
                             _p(vt), ctypes.c_size_t(vt.nbytes), _p(kcache), _p(vcache), ctypes.c_size_t(kcache.nbytes), n_head, n_kv, hd, vt_ld,
                             nseg, _p(st), _p(ln), _p(p0), _p(toff), _p(flat), ctypes.c_size_t(_nb(flat)))
        assert rc == 0
        _check_rope_outputs("rope_split_epilogue", bufs, before, ref, segs, tabs, m, n_head, n_kv, hd, lambda bb: R.GEMM_ELEM_TOL * bb)
    # the stand-alone kernel on fp32 QKV rows
    qkv = rng.standard_normal((m, n)).astype(np.float32)
    x = qkv.astype(np.float64)
    ref = R.rope_split(x, np.abs(x), n_head, n_kv, hd, cos_t, sin_t, segs)
    bufs = _rope_buffers(m, n_head, n_kv, hd, n_pages)
    before = [y.copy() for y in bufs[:5]]
    q, kk, vt, kcache, vcache, vt_ld = bufs
    rc = kc.kc_rope_split_segs(_p(qkv), ctypes.c_size_t(qkv.nbytes), m, n_head, n_kv, hd, _p(cos_t), _p(sin_t), ctypes.c_size_t(cos_t.nbytes),
                               _p(q), ctypes.c_size_t(q.nbytes), _p(kk), ctypes.c_size_t(kk.nbytes), _p(vt), ctypes.c_size_t(vt.nbytes),
                               _p(kcache), _p(vcache), ctypes.c_size_t(kcache.nbytes), vt_ld, nseg, _p(st), _p(ln), _p(p0), _p(toff), _p(flat),
                               ctypes.c_size_t(_nb(flat)))
    assert rc == 0
    _check_rope_outputs("rope_split_segs", bufs, before, ref, segs, tabs, m, n_head, n_kv, hd, lambda bb: 2.0 ** -22 * bb)


# =============================================================================================================================
# prompt attention
# =============================================================================================================================
def _flash(kc, q, k, vt, out, kcache, vcache, n_head, n_kv, hd, vt_ld, segs, tabs):
    nseg, st, ln, p0, toff, flat = _segs_args(segs, tabs)
    rc = kc.kc_flash_prefill(_p(q), _nb(q), _p(k), _nb(k), _p(vt), _nb(vt), _p(out), _nb(out), _p(kcache), _p(vcache), _nb(kcache),
                             n_head, n_kv, hd, vt_ld, 1.0 / np.sqrt(hd), nseg, _p(st), _p(ln), _p(p0), _p(toff), _p(flat), _nb(flat))
    assert rc == 0, rc


def _nonpaged_pack(qs, ks, vs, n_head, n_kv, hd):
    """pack several sequences (q/k/v lists) at 128-row starts: q/k rows, V^T columns [len, roundup(len, 64)) zero, everything
    past that and every padding row of q / k NaN (never read)"""
    qd, kvd = n_head * hd, n_kv * hd
    starts, o = [], 0
    for q in qs:
        starts.append(o)
        o += (len(q) + 127) // 128 * 128
    rows = o
    vt_ld = rows + 8
    Q = np.full((rows, qd), NAN16, np.uint16)
    K = np.full((rows, kvd), NAN16, np.uint16)
    VT = np.full((kvd, vt_ld), NAN16, np.uint16)
    for s0, q, k, v in zip(starts, qs, ks, vs):
        L = len(q)
        Q[s0:s0 + L] = q.view(np.uint16)
        K[s0:s0 + L] = k.view(np.uint16)
        VT[:, s0:s0 + L] = v.view(np.uint16).T
        VT[:, s0 + L:s0 + (L + 63) // 64 * 64] = 0
    return Q, K, VT, vt_ld, starts


def _check_attn(tag, got, q, k, v, pos0, n_head, n_kv, hd, rows):
    ref = R.attention(q.astype(np.float64), k.astype(np.float64), v.astype(np.float64), pos0, n_head, n_kv, hd, 1.0 / np.sqrt(hd), rows)
    ratio, rl2 = R.attention_check(got[rows].astype(np.float64), ref, v.astype(np.float64), n_head, n_kv, hd)
    _note("flash_" + tag, ratio)
    _note("flash_" + tag + "_relL2/1e-3", rl2 / R.ATTN_REL_L2)
    assert ratio <= 1.0 and rl2 <= R.ATTN_REL_L2, (tag, pos0, len(q), ratio, rl2)


@pytest.mark.parametrize("heads", KC.ATTN_HEADS, ids=lambda h: f"h{h[0]}kv{h[1]}")
@pytest.mark.parametrize("hd", [64, 128])
def test_flash_nonpaged(kc, hd, heads):
    n_head, n_kv = heads
    qd = n_head * hd
    for L in KC.ATTN_LENS:
        for peaked in (False, True):
            rng = np.random.Generator(np.random.PCG64(L * 3 + hd + n_head + peaked))
            q, k, v = KC.qkv_values(rng, L, L, n_head, n_kv, hd, peaked)
            Q, K, VT, vt_ld, _ = _nonpaged_pack([q], [k], [v], n_head, n_kv, hd)
            rows = Q.shape[0]
            out = np.full((rows + 1, qd), NAN16, np.uint16)
            _flash(kc, Q, K, VT, out, None, None, n_head, n_kv, hd, vt_ld, [(0, L, 0)], [None])
            o = out.view(np.float16)
            assert (o[L:rows] == 0).all() and (out[rows] == NAN16).all(), L     # padding rows zero, nothing past them written
            _check_attn("nonpaged" + ("_peaked" if peaked else ""), o, q, k, v, 0, n_head, n_kv, hd, R.attention_sample_rows(L))


def _paged_cache(rng, k, v, n_kv, hd, n_pool, spare=3):
    """K / V of positions 0 .. kv_len - 1 in shuffled pages of a pool; the table has `spare` extra entries that point at valid
    pages, and every unused slot and unmapped page is NaN"""
    kv_len = k.shape[0]
    need = (kv_len + 15) // 16
    assert need + spare <= n_pool
    tab = rng.permutation(n_pool)[:need + spare].astype(np.int32)
    kc4 = np.full((n_pool, n_kv, 16, hd), NAN16, np.uint16)
    vc4 = np.full((n_pool, n_kv, 16, hd), NAN16, np.uint16)
    for p in range(kv_len):
        kc4[tab[p // 16], :, p % 16] = k[p].view(np.uint16).reshape(n_kv, hd)
        vc4[tab[p // 16], :, p % 16] = v[p].view(np.uint16).reshape(n_kv, hd)
    return kc4.reshape(-1), vc4.reshape(-1), tab


@pytest.mark.parametrize("heads", KC.ATTN_HEADS, ids=lambda h: f"h{h[0]}kv{h[1]}")
@pytest.mark.parametrize("hd", [64, 128])
def test_flash_paged(kc, hd, heads):
    n_head, n_kv = heads
    qd = n_head * hd
    for pos0 in KC.PAGED_POS0:
        for L in KC.PAGED_LENS:
            peaked = (pos0 + L) % 2 == 1
            rng = np.random.Generator(np.random.PCG64(pos0 * 11 + L + hd + n_head))
            kv_len = pos0 + L
            q, k, v = KC.qkv_values(rng, kv_len, L, n_head, n_kv, hd, peaked)
            kcache, vcache, tab = _paged_cache(rng, k, v, n_kv, hd, (kv_len + 15) // 16 + 5)
            rows = (L + 127) // 128 * 128
            Q = np.full((rows, qd), NAN16, np.uint16)
            Q[:L] = q.view(np.uint16)
            out = np.full((rows + 1, qd), NAN16, np.uint16)
            _flash(kc, Q, None, None, out, kcache, vcache, n_head, n_kv, hd, 8, [(0, L, pos0)], [tab])
            o = out.view(np.float16)
            assert (o[L:rows] == 0).all() and (out[rows] == NAN16).all(), (pos0, L)
            _check_attn("paged" + ("_peaked" if peaked else ""), o, q, k, v, pos0, n_head, n_kv, hd, R.attention_sample_rows(L))


@pytest.mark.parametrize("hd", [64, 128])
def test_flash_packs_and_bit_identity(kc, hd):
    n_head, n_kv = 8, 2
    qd = n_head * hd
    rng = np.random.Generator(np.random.PCG64(500 + hd))
    # --- non-paged pack of three sequences: each equals its own launch, bit for bit
    lens = [300, 65, 1]
    seqs = [KC.qkv_values(rng, L, L, n_head, n_kv, hd, True) for L in lens]
    Q, K, VT, vt_ld, starts = _nonpaged_pack([s[0] for s in seqs], [s[1] for s in seqs], [s[2] for s in seqs], n_head, n_kv, hd)
    out = np.full((Q.shape[0], qd), NAN16, np.uint16)
    _flash(kc, Q, K, VT, out, None, None, n_head, n_kv, hd, vt_ld, [(s0, L, 0) for s0, L in zip(starts, lens)], [None] * 3)
    for s0, L, (q, k, v) in zip(starts, lens, seqs):
        Q1, K1, VT1, vt1, _ = _nonpaged_pack([q], [k], [v], n_head, n_kv, hd)
        o1 = np.full((Q1.shape[0], qd), NAN16, np.uint16)
        _flash(kc, Q1, K1, VT1, o1, None, None, n_head, n_kv, hd, vt1, [(0, L, 0)], [None])
        assert np.array_equal(out[s0:s0 + L], o1[:L]), ("pack", L)
        _check_attn("pack", out.view(np.float16)[s0:s0 + L], q, k, v, 0, n_head, n_kv, hd, R.attention_sample_rows(L))
    # --- a paged chunk at pos0 = p equals rows p.. of one non-paged pass over the whole sequence
    for p, L in ((100, 129), (17, 64), (128, 300)):
        T = p + L
        q, k, v = KC.qkv_values(rng, T, T, n_head, n_kv, hd, True)
        Qw, Kw, VTw, vtw, _ = _nonpaged_pack([q], [k], [v], n_head, n_kv, hd)
        ow = np.full((Qw.shape[0], qd), NAN16, np.uint16)
        _flash(kc, Qw, Kw, VTw, ow, None, None, n_head, n_kv, hd, vtw, [(0, T, 0)], [None])
        kcache, vcache, tab = _paged_cache(rng, k, v, n_kv, hd, (T + 15) // 16 + 4)
        rows = (L + 127) // 128 * 128
        Qp = np.full((rows, qd), NAN16, np.uint16)
        Qp[:L] = q[p:].view(np.uint16)
        op = np.full((rows, qd), NAN16, np.uint16)
        _flash(kc, Qp, None, None, op, kcache, vcache, n_head, n_kv, hd, 8, [(0, L, p)], [tab])
        assert np.array_equal(op[:L], ow[p:T]), ("chunk", p, L)
    # --- a paged pack mixing pos0 = 0 and pos0 > 0 (each segment its own pages in one pool)
    specs = [(129, 0), (64, 100), (7, 4096)]
    pool = sum((p0 + L + 15) // 16 for L, p0 in specs) + 6
    perm = rng.permutation(pool).astype(np.int32)
    kc4 = np.full((pool, n_kv, 16, hd), NAN16, np.uint16)
    vc4 = np.full((pool, n_kv, 16, hd), NAN16, np.uint16)
    segs, tabs, data, used, o = [], [], [], 0, 0
    for L, p0 in specs:
        T = p0 + L
        q, k, v = KC.qkv_values(rng, T, L, n_head, n_kv, hd, False)
        need = (T + 15) // 16
        tab = perm[used:used + need]
        used += need
        for pp in range(T):
            kc4[tab[pp // 16], :, pp % 16] = k[pp].view(np.uint16).reshape(n_kv, hd)
            vc4[tab[pp // 16], :, pp % 16] = v[pp].view(np.uint16).reshape(n_kv, hd)
        segs.append((o, L, p0))
        tabs.append(tab)
        data.append((q, k, v))
        o += (L + 127) // 128 * 128
    Q = np.full((o, qd), NAN16, np.uint16)
    for (s0, L, _p0), (q, _k, _v) in zip(segs, data):
        Q[s0:s0 + L] = q.view(np.uint16)
    out = np.full((o, qd), NAN16, np.uint16)
    _flash(kc, Q, None, None, out, kc4.reshape(-1), vc4.reshape(-1), n_head, n_kv, hd, 8, segs, tabs)
    for (s0, L, p0), (q, k, v) in zip(segs, data):
        _check_attn("paged_pack", out.view(np.float16)[s0:s0 + L], q, k, v, p0, n_head, n_kv, hd, R.attention_sample_rows(L))


# =============================================================================================================================
# qgemm
# =============================================================================================================================
_QG_REF = {}


def _qg_ref(hc, name):
    """float64 C and |act||W|^T of a shape for all 64 batch rows (NB = 16 / 32 use the first rows)"""
    if name not in _QG_REF:
        specs, mode, k, _epi, _how = KC.QG_SHAPES[name]
        srcs, mode = KC.qg_sources(name)
        act = KC.qg_act(name, k)
        c, b = R.qgemm(hc, srcs, mode, act[:64].astype(np.float64))
        _QG_REF[name] = (srcs, mode, act, c, b)
    return _QG_REF[name]


def _run_qgemm(kc, srcs, mode, k, act, nb, c, ldc, epi, n_sm, reps=2, norm=None):
    """returns (C of every rep, info, counters of every rep, xg of every rep, ssq of every rep)"""
    nsrc = len(srcs)
    n_rows = sum(b.shape[0] for b, _t in srcs)
    n_tiles = n_rows // 128
    blk = [np.ascontiguousarray(b) for b, _t in srcs]
    src_p = (ctypes.c_void_p * 3)(*[b.ctypes.data for b in blk] + [None] * (3 - nsrc))
    src_b = (ctypes.c_size_t * 3)(*[b.nbytes for b in blk] + [0] * (3 - nsrc))
    types = (ctypes.c_int * 3)(*[t for _b, t in srcs] + [0] * (3 - nsrc))
    rows = (ctypes.c_int * 3)(*[b.shape[0] for b in blk] + [0] * (3 - nsrc))
    toff = np.zeros(n_tiles, np.uint64)
    ttype = np.zeros(n_tiles, np.uint8)
    info = np.zeros(4, np.int32)
    c_out = np.empty((reps,) + c.shape, c.dtype)
    cnt = np.full((reps, n_tiles), 0xFFFFFFFF, np.uint32)
    nm = norm or {}
    gamma, xg, ssq_out, ssq_in = nm.get("gamma"), nm.get("xg"), nm.get("ssq_out"), nm.get("ssq_in")
    xg_all = np.empty((reps,) + xg.shape, xg.dtype) if xg is not None else None
    ssq_all = np.empty((reps,) + ssq_out.shape, ssq_out.dtype) if ssq_out is not None else None
    rc = kc.kc_qgemm(ctypes.c_int(nsrc), ctypes.c_int(mode), ctypes.c_int(k), src_p, src_b, types, rows, _p(toff), _p(ttype), _p(info),
                     _p(act), ctypes.c_size_t(act.nbytes), ctypes.c_int(act.shape[0]), ctypes.c_int(nb), _p(c), ctypes.c_size_t(c.nbytes),
                     ctypes.c_int(ldc), ctypes.c_int(epi), ctypes.c_int(n_sm), ctypes.c_int(reps), _p(c_out), _p(cnt),
                     _p(gamma), ctypes.c_size_t(_nb(gamma)), _p(xg), ctypes.c_size_t(_nb(xg)), ctypes.c_int(nm.get("ldxg", 0)),
                     _p(ssq_out), ctypes.c_size_t(_nb(ssq_out)), _p(ssq_in), ctypes.c_size_t(_nb(ssq_in)), ctypes.c_int(nm.get("parts", 0)),
                     ctypes.c_int(nm.get("n_norm", 0)), ctypes.c_float(nm.get("eps", 0.0)), _p(xg_all), _p(ssq_all))
    assert rc == 0, rc
    assert (cnt == 0).all(), "split-tile counters must be zero after every launch"
    for r in range(1, reps):
        assert np.array_equal(c_out[r].view(np.uint8), c_out[0].view(np.uint8)), "the same launch twice must give the same bits"
        if xg_all is not None:
            assert np.array_equal(xg_all[r], xg_all[0]) and np.array_equal(ssq_all[r].view(np.uint32), ssq_all[0].view(np.uint32))
    return c_out[0], info, xg_all[0] if xg_all is not None else None, ssq_all[0] if ssq_all is not None else None


def _qg_check(name, got_buf, ref, bound, old, epi, nb, ldc, n):
    """C region against the reference; every other element of the buffer unchanged"""
    w = n // 2 if epi == KC.SILU else n
    relb = R.gemm_rel_l2_bound(KC.QG_SHAPES[name][2], "fp16" if epi == KC.SILU else None)
    if epi == KC.SILU:
        r, b = R.silu_ref(ref[:nb], bound[:nb])
        got = got_buf.view(np.float16)[:nb * ldc].reshape(nb, ldc)[:, :w].astype(np.float64)
        ratio, rl2 = R.gemm_check(got, r, b, R.ulp16(r))
        rest_ok = (got_buf[:nb * ldc].reshape(nb, ldc)[:, w:] == NAN16).all() and (got_buf[nb * ldc:] == NAN16).all()
    else:
        r = ref[:nb] + (old[:nb] if epi == KC.ADD else 0.0)
        got = got_buf.view(np.float32)[:nb * ldc].reshape(nb, ldc)[:, :w].astype(np.float64)
        ratio, rl2 = R.gemm_check(got, r, bound[:nb], 2.0 ** -23 * np.abs(r) if epi == KC.ADD else 0.0)
        rest_ok = (got_buf[:nb * ldc].reshape(nb, ldc)[:, w:] == NAN32).all() and (got_buf[nb * ldc:] == NAN32).all()
    _note("qgemm", ratio)
    _note("qgemm_relL2/bound", rl2 / relb)
    assert ratio <= 1.0 and rl2 <= relb, (name, nb, ratio, rl2)
    assert rest_ok, (name, nb, "wrote outside C")


def _qg_buffers(name, nb, n, epi, rng):
    w = n // 2 if epi == KC.SILU else n
    ldc = w + (8 if epi != KC.F32 else 4)
    if epi == KC.SILU:
        return np.full(nb * ldc + 64, NAN16, np.uint16), ldc, None
    c = np.full(nb * ldc + 64, NAN32, np.uint32)
    old = None
    if epi == KC.ADD:
        old = rng.standard_normal((nb, n)).astype(np.float32)
        c[:nb * ldc].view(np.float32).reshape(nb, ldc)[:, :n] = old
        old = np.vstack([old.astype(np.float64), np.zeros((64 - nb, n))])
    return c, ldc, old


def _qg_act_nan(act, nb):
    a = act.copy()
    a[nb:] = np.float16(np.nan)          # rows at and beyond the batch are read by nobody's result
    return a


QG_SWEEP = ["nkb1", "nkb3", "nkb5", "three_src", "silu_small", "o_8b"]


def test_qgemm_partition_sweep(kc, hostcheck_lib):
    """every NB over n_sm in {1, 2, 3, 4, 5, 8, 13, 33, 64, device}: stream-K partitions the model tests never produce, and the
    cluster mode.  Asserts the sweep reached, for every NB: cluster mode, a whole tile under stream-K, a tile shared by >= 3
    CTAs and a CTA whose range spans >= 3 tiles."""
    dev = kc.kc_device_sms()
    assert dev > 0
    sms = sorted({s for s in (1, 2, 3, 4, 5, 8, 13, 33, 64, dev) if s <= dev})
    reached = {nb: set() for nb in (16, 32, 64)}
    rng = np.random.Generator(np.random.PCG64(77))
    for name in QG_SWEEP:
        srcs, mode, act, ref, bound = _qg_ref(hostcheck_lib, name)
        _specs, _mode, k, epi, _how = KC.QG_SHAPES[name]
        n = ref.shape[1]
        n_tiles, nkb = n // 128, k // 256
        for nb in (16, 32, 64):
            for n_sm in sms:
                c, ldc, old = _qg_buffers(name, nb, n, epi, rng)
                got, info, _, _ = _run_qgemm(kc, srcs, mode, k, _qg_act_nan(act, nb), nb, c, ldc, epi, n_sm)
                assert info[1] == (0 if name == "three_src" else 1), (name, "tile tables")
                _qg_check(name, got, ref, bound, old, epi, nb, ldc, n)
                if info[0]:
                    reached[nb].add("cluster")
                else:
                    reached[nb] |= R.streamk_patterns(n_tiles, nkb, n_sm)
    for nb, pats in reached.items():
        assert {"cluster", "whole", "shared3", "span3"} <= pats, (nb, pats)
    print("KERNELCHECK qgemm coverage " + " ".join(f"NB{nb}:{','.join(sorted(p))}" for nb, p in reached.items()))


@pytest.mark.parametrize("name", ["qkv_8b", "gate_up_8b", "down_8b", "lm_head_8b"])
def test_qgemm_8b_shapes(kc, hostcheck_lib, name):
    dev = kc.kc_device_sms()
    srcs, mode, act, ref, bound = _qg_ref(hostcheck_lib, name)
    _specs, _mode, k, epi, _how = KC.QG_SHAPES[name]
    n = ref.shape[1]
    rng = np.random.Generator(np.random.PCG64(5))
    for nb in ((16,) if name == "lm_head_8b" else (16, 32, 64)):
        for n_sm in ((dev,) if name == "lm_head_8b" else (dev, 13)):
            c, ldc, old = _qg_buffers(name, nb, n, epi, rng)
            got, info, _, _ = _run_qgemm(kc, srcs, mode, k, _qg_act_nan(act, nb), nb, c, ldc, epi, n_sm)
            assert info[1] == 1
            _qg_check(name, got, ref, bound, old, epi, nb, ldc, n)


@pytest.mark.parametrize("nb", [16, 32, 64])
def test_qgemm_folded_norm_pair(kc, hostcheck_lib, nb):
    """attn_output (residual add, producer: xg = fp16(x_new gamma / 16) and per-slice sums of squares, cluster mode) -> QKV
    (consumer: (W xg) 16 / sqrt(sum of parts / n + eps)), each against float64 on its own inputs"""
    dev = kc.kc_device_sms()
    name = "o_8b"
    srcs, mode, act, ref, bound = _qg_ref(hostcheck_lib, name)
    k = KC.QG_SHAPES[name][2]
    n = ref.shape[1]
    n_tiles = n // 128
    cand = [s for s in (dev, 64, 33, 16) if s <= dev and kc.kc_qgemm_uses_cluster(n_tiles, k // 256, nb, KC.ADD, s) == 1]
    assert cand, "no n_sm puts the attn_output shape in cluster mode"
    rng = np.random.Generator(np.random.PCG64(99 + nb))
    gamma = (1.0 + 0.5 * rng.standard_normal(n)).astype(np.float32)
    xg = np.zeros((128, n), np.float16)
    ssq = np.full((n_tiles * 4, 64), np.nan, np.float32)
    c, ldc, old = _qg_buffers(name, nb, n, KC.ADD, rng)
    got, info, xg_got, ssq_got = _run_qgemm(kc, srcs, mode, k, _qg_act_nan(act, nb), nb, c, ldc, KC.ADD, cand[0],
                                            norm={"gamma": gamma, "xg": xg, "ldxg": n, "ssq_out": ssq})
    assert info[0] == 1
    _qg_check(name, got, ref, bound, old, KC.ADD, nb, ldc, n)
    x_new = ref[:nb] + old[:nb]
    xb = bound[:nb] * R.GEMM_ELEM_TOL + 2.0 ** -23 * np.abs(x_new)          # bound of x_new as the kernel holds it
    xg_ref, ssq_ref = R.norm_producer(x_new, gamma.astype(np.float64), n_tiles)
    g16 = np.abs(gamma.astype(np.float64)) / 16.0
    ratio = float((np.abs(xg_got[:nb].astype(np.float64) - xg_ref) / (xb * g16 + R.ulp16(xg_ref))).max())
    _note("qgemm_norm_producer_xg", ratio)
    assert ratio <= 1.0, ratio
    assert (xg_got[nb:] == 0).all()
    ssq_b = (2.0 * np.abs(x_new) * xb + 32 * 2.0 ** -23 * x_new * x_new).reshape(nb, n_tiles * 4, 32).sum(axis=2).T
    ratio = float((np.abs(ssq_got[:, :nb].astype(np.float64) - ssq_ref) / ssq_b).max())
    _note("qgemm_norm_producer_ssq", ratio)
    assert ratio <= 1.0, ratio
    # consumer: the QKV projection on the producer's xg and sums of squares
    cname = "qkv_8b"
    csrcs, cmode, _cact, _cref, _cb = _qg_ref(hostcheck_lib, cname)
    eps = 1e-5
    xg_act = xg_got.copy()
    xg_act[nb:] = np.float16(np.nan)
    cr, cbnd = R.qgemm(hostcheck_lib, csrcs, cmode, xg_act[:nb].astype(np.float64))
    scale = R.norm_consumer_scale(ssq_got[:, :nb].astype(np.float64), n, eps)
    cn = cr.shape[1]
    c2, ldc2, _ = _qg_buffers(cname, nb, cn, KC.F32, rng)
    got2, _info2, _, _ = _run_qgemm(kc, csrcs, cmode, k, xg_act, nb, c2, ldc2, KC.F32, dev,
                                    norm={"ssq_in": np.ascontiguousarray(ssq_got), "parts": n_tiles * 4, "n_norm": n, "eps": eps})
    want = cr * scale[:, None]
    g = got2.view(np.float32)[:nb * ldc2].reshape(nb, ldc2)[:, :cn].astype(np.float64)
    # + the per-token scale: fp32 sum of the parts (parts 2^-24 worst case, halved by the square root), rsqrtf and the multiply
    srel = n_tiles * 4 * 2.0 ** -25 + 2.0 ** -21
    tol = R.GEMM_ELEM_TOL * cbnd * scale[:, None] + srel * np.abs(want)
    ratio = float((np.abs(g - want) / tol).max())
    _note("qgemm_norm_consumer", ratio)
    assert ratio <= 1.0 and R.rel_l2(g, want) <= R.gemm_rel_l2_bound(k) + srel, (ratio, R.rel_l2(g, want))
