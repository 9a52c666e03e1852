"""CPU: the bounds of tests/test_gpu_decode_gemv.py rehearsed and shown to have teeth, on the very inputs of its GPU cases.

* The GEMV lane program of rowdot.h, run on the host by tests/hostcheck (fp32, the kernel's own per-lane code; its sum over
  lanes is a plain loop rather than the warp tree), stays within half of the bound on every case that is not huge.  The orders
  differ, so this is evidence that the bound holds, not a bit-exact check.
* Every named mutant of the reference -- a bug the kernel could have -- lands at least 4x the bound away on the outputs it
  changes, so a check at the bound cannot let it through.
* The Python wrapper passes the shim's arguments in the order gemvcheck.cu declares them."""
import ctypes
import os
import re

import numpy as np
import pytest

import gemv_cases as G

MARGIN = 4.0
CASES = {c.name: c for c in G.cases()}
SMALL = [n for n, c in CASES.items() if c.elems <= G.BIG]


def _lane_program(hc, case, m):
    """rstd32 * (lane program over fp32(x * norm_w)), as float64"""
    xw = (case.x * case.norm_w).astype(np.float32) if case.norm else case.x
    y = np.zeros(case.rows[m], np.float32)
    b = np.ascontiguousarray(case.blocks[m])
    rc = hc.hc_gemv_r(case.types[m], b.ctypes.data_as(ctypes.c_void_p), case.rows[m], case.cols, xw.ctypes.data_as(ctypes.c_void_p),
                      y.ctypes.data_as(ctypes.c_void_p), case.abits, 0)
    assert rc == 0
    if case.norm:
        ss = np.float32((case.x * case.x).sum(dtype=np.float32))
        rstd = np.float32(1.0) / np.sqrt(ss / np.float32(case.cols) + np.float32(case.eps))
        y = y * rstd
    return y.astype(np.float64)


@pytest.mark.parametrize("name", SMALL)
def test_lane_program_within_half_the_bound(hostcheck_lib, name):
    case = CASES[name]
    for m in range(len(case.types)):
        y, bound = case.gemv_ref(m)
        got = _lane_program(hostcheck_lib, case, m)
        assert np.isfinite(got).all()
        r = float(np.max(np.abs(got - y) / bound))
        assert r <= 0.5, (name, m, r)


@pytest.mark.parametrize("name", SMALL)
def test_mutants_are_caught(name):
    case = CASES[name]
    for mutant in G.MUTANTS:
        if G.mutant_applies(case, mutant):
            d = G.mutant_distance(case, mutant)
            assert d >= MARGIN, (name, mutant, d)


def test_every_mutant_is_exercised():
    seen = {m for n in SMALL for m in G.MUTANTS if G.mutant_applies(CASES[n], m)}
    assert seen == set(G.MUTANTS), set(G.MUTANTS) - seen


def test_v_in_the_decoy_slot_is_caught():
    """a V row written to the decoy position's slot (or unrounded anywhere else) changes bytes the pool check keeps"""
    case = CASES["qkv-hd64-kv2-p15"]
    kc, vc = case.kc.copy(), case.vc.copy()
    ref = case.reference()
    ph, t = case.slot(0)
    kc[ph, :, t, :] = ref["k16"].astype(np.float16).view(np.uint16).reshape(case.n_kv, case.hd)
    vc[ph, :, t, :] = ref["v16"].astype(np.float16).view(np.uint16).reshape(case.n_kv, case.hd)
    assert G.check_pool(case, kc, vc)
    dp = int(case.table[case.decoy_pos // G.PAGE])
    assert dp != ph
    vc[dp, :, case.decoy_pos % G.PAGE, :] = vc[ph, :, t, :]
    assert not G.check_pool(case, kc, vc)


def test_edge_activations_hit_their_edges():
    """the 'edges' input has an all-zero block, an outlier block and a block whose x inv lands on k + 1/2 (ties to even)"""
    case = CASES["rows1-q4k"]
    x = case.x
    assert (x[32:64] == 0).all()
    blk = np.abs(x[64:96])
    assert blk.max() >= 1e3 * np.sort(blk)[-2]
    inv = np.float32(16256.0) / np.float32(np.abs(x[96:128]).max())
    assert inv == 1.0 and (np.modf(np.abs(x[97:128] * inv))[0] == 0.5).all()


def test_ksplit_matches_rowdot(hostcheck_lib):
    for cols in (256, 4096, 4352, 8192, 14336, 28672, 32768):
        nks, nb = ctypes.c_int(), ctypes.c_int()
        rc = hostcheck_lib.hc_ksplit(cols, ctypes.byref(nks), ctypes.byref(nb))
        assert (nks.value if rc == 0 else 0, nb.value if rc == 0 else 0) == G.ksplit(cols), cols
    assert G.ksplit(14336) == (4, 14) and G.ksplit(28672) == (7, 16) and G.ksplit(32768) == (8, 16) and G.ksplit(4352) == (0, 0)


def test_shim_argument_order_matches_the_wrapper():
    src = open(os.path.join(G.ROOT, "tests", "gemvcheck", "gemvcheck.cu")).read()
    sig = re.search(r"int gc_gemv\((.*?)\)\s*\{", src, re.S).group(1)
    names = [re.split(r"[\s*]+", a.strip())[-1] for a in sig.split(",")]
    assert tuple(names) == G.GC_GEMV_ARGS
    assert "StepState" in src and G.STEP_STATE_BYTES == 108
