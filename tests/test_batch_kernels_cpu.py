"""CPU: the bounds of tests/test_gpu_batch_kernels.py rehearsed and shown to have teeth, on the very inputs of its GPU cases.

* A numpy restatement of the tensor-core batched attention's roundings (batch_cases.attn_model: fp16 q * scale, fp16 P against
  each warp's running maximum, the warp and split merges, fp16 output) stays within half of the attention bound on every case.
* Every named mutant of the attention reference -- a bug the kernel could have -- lands at least 4x the bound away on every row
  it applies to; so do the RoPE and RMSNorm mutants.  The greedy draw's checks are exact and need no mutants."""
import numpy as np
import pytest

import batch_cases as B
import kernel_ref as R

MARGIN = 4.0
CASES = B.attn_cases()


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_attention_model_within_half_the_bound(name, kw):
    case = B.AttnCase(**kw)
    worst = 0.0
    for r in range(case.n_rows):
        ref, v = case.reference(r)
        d = B.attn_distance(B.attn_model(case, r), ref, v, case.n_head, case.n_kv, case.hd)
        worst = max(worst, d)
    assert worst <= 0.5, (name, worst)


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_attention_mutants_are_caught(name, kw):
    case = B.AttnCase(**kw)
    seen = set()
    for r in range(case.n_rows):
        ref, v = case.reference(r)
        for mutant in B.ATTN_MUTANTS:
            if not case.applies(r, mutant):
                continue
            seen.add(mutant)
            mut, _ = case.reference(r, mutant)
            d = B.attn_distance(mut, ref, v, case.n_head, case.n_kv, case.hd)
            assert d >= MARGIN, (name, r, int(case.pos[r]), mutant, d)
    assert {"stale_newest", "neighbour_table"} <= seen
    if name.startswith("long-S1"):
        assert "broken_reload" in seen


def test_attention_cases_reach_the_edges():
    """what the launches cover: every split count the engine picks, fewer pages than splits, a fifth page per split, the table
    reload, padded rows, a slot permutation and shared pages"""
    cov = set()
    for name, kw in CASES:
        S = kw["S"]
        npg = np.asarray(kw["positions"]) // 16 + 1
        cov.add(("S", S))
        if (npg < S).any():
            cov.add("fewer pages than splits")
        if ((npg == 4 * S) .any() and (npg == 4 * S + 1).any()):
            cov.add("4S / 4S + 1")
        if (npg > 32 * 4 * S).any():
            cov.add("reload")
        if kw.get("bucket", len(npg)) > len(npg):
            cov.add("padded rows")
        if kw.get("share"):
            cov.add("shared pages")
    for n_kv in (2, 8, 16):
        for _b, s in B.engine_splits(n_kv):
            assert ("S", s) in cov
    for s in B.ATTN_SPLITS:
        assert ("S", s) in cov
    assert {"fewer pages than splits", "4S / 4S + 1", "reload", "padded rows", "shared pages"} <= cov


def test_broken_reload_map_moves_pages_past_32():
    m = B.broken_reload_map(512, 1)
    assert (m[:128] == np.arange(128)).all() and m[128] == 0 and m[129] == 1 and m[511] == 511 - 384
    assert (B.broken_reload_map(100, 2) == np.arange(100)).all()


@pytest.mark.parametrize("hd", [64, 128])
def test_rope_mutants_are_caught(hd):
    case = B.AttnCase(hd, 4 * (hd // 64), 2, 2, [1, 16, 17, 300, 4000])
    bound = B.rope_bound(case.k_raw, hd) + R.ulp16(case.k_ref)
    for mutant in ("pos-1", "pos+1", "neox"):
        mut = B.rope_mutant(case.k_raw, case.pos, case.cos, case.sin, hd, mutant)
        assert (np.abs(mut - case.k_ref) / bound).max() >= MARGIN, mutant


@pytest.mark.parametrize("n", [64, 256, 4096, 5120, 8192])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_rmsnorm_mutants_are_caught(n, eps):
    """eps dropped matters on the small row only; mean over n - 1 moves every output by 1 / (2 n) relative, which one fp16 ulp
    resolves 4x over only at n = 64 (at n >= 256 it is below 2^-9: a one-ulp check cannot see it, and no kernel computes it)"""
    x, w = B.rmsnorm_rows(n)
    ref = B.rmsnorm_ref(x, w, eps)
    live = [0, 1, 2, 4]
    assert B.rmsnorm_distance(B.rmsnorm_ref(x, w, eps, "no_eps")[[1]], ref[[1]]) >= MARGIN
    assert B.rmsnorm_distance(B.rmsnorm_ref(x, w, eps, "w_shift")[live], ref[live]) >= MARGIN
    if n == 64:
        assert B.rmsnorm_distance(B.rmsnorm_ref(x, w, eps, "mean_n-1")[live], ref[live]) >= MARGIN


def test_rmsnorm_fp32_restatement_within_one_ulp():
    """the kernel's fp32 arithmetic (sum of squares, rstd, x rstd w) rounded to fp16 stays within one ulp of the float64 value"""
    for n in (64, 5120):
        x, w = B.rmsnorm_rows(n)
        ref = B.rmsnorm_ref(x, w, 1e-5)
        ss = (x * x).sum(axis=1, dtype=np.float32)
        rstd = np.float32(1.0) / np.sqrt(ss / np.float32(n) + np.float32(1e-5))
        got = ((x * rstd[:, None]) * w[None, :]).astype(np.float16).astype(np.float64)
        assert B.rmsnorm_distance(got, ref) <= 1.0
        assert (got[3] == 0).all()


def test_greedy_reference_tie_rule_and_bound():
    lg = B.greedy_logits(4097, 5, 0)
    ids, lp = B.greedy_ref(lg)
    per = -(-4097 // 8)
    assert ids[0] == per * ((4097 - 1) // per) - 1 or ids[0] == per * 7 - 1
    assert ids[1] == 5 and ids[2] == 4096 and ids[3] == 4096 and ids[4] == 0
    assert abs(lp[3]) == 0.0 and abs(lp[4] + np.log(4097)) < 1e-12
    assert B.greedy_lp_bound(151936) < 3e-5


def test_state_layouts_match_the_shim():
    """the numpy records have the sizes of the C structs they are copied into"""
    assert B.STEP_STATE.itemsize == 108 and B.BATCH_CTL.itemsize == 4 * 129 and B.BATCH_OUT.itemsize == 16
