"""GPU parity AT THE BENCHMARKED SHAPE: the synthetic Llama-3-8B q4_K_M GGUF bench.py times (32 layers, d = 4096, 128 256-entry
vocabulary, K = 14336 rows cut into four K-segments, GQA 4:1, Q4_K + Q6_K mix) against the C restatement in EXACT mode
(oracle/c/llama_cpu.c act_mode 0: dequantised fp32 weights x fp32 activations) on the same tokens.

The small-model suites (tests/test_gpu_decode.py, tests/test_gpu_batch.py) cover every kernel variant against the numpy oracle;
this file checks that the COMBINATION the benchmark runs -- never exercised as a whole by 2-layer models -- computes the same
function: the single-sequence decode step, the batched tensor-core prefill, and the batched decode step (continuous batching).
Tolerances are those of the small-model tests: logits within 1e-2 * max|logit| of exact arithmetic, logprob within 2e-2, greedy
ids equal wherever the oracle's top-1/top-2 margin exceeds 5e-2.  The model file is the bench's (built once per box, ~1 min)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bench_model():
    sys.path.insert(0, ROOT)
    import bench
    return bench.build_model_once("llama3_8b_q4km", 0, lambda: None)


@pytest.fixture(scope="module")
def oracle_8b(bench_model):
    so = os.path.join(ROOT, "oracle", "_ref", "liboracle_cpu.so")
    lib = C.CDLL(so)
    lib.oc_load.restype = C.c_void_p
    lib.oc_load.argtypes = [C.c_char_p, C.c_int]
    lib.oc_step.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.oc_reset.argtypes = [C.c_void_p]
    lib.oc_free.argtypes = [C.c_void_p]
    lib.oc_set_threads.argtypes = [C.c_int]
    lib.oc_set_threads(min(32, os.cpu_count() or 8))                # not every logical CPU: exact mode is memory-bound
    h = lib.oc_load(bench_model.encode(), 64)
    assert h
    yield lib, h
    lib.oc_free(h)


@pytest.fixture(scope="module")
def engine_8b(bench_model):
    from gridllm_b200 import native as N
    e = N.Engine(bench_model, max_ctx=256, max_batch=4)
    yield e
    e.close()


def _oracle_run(oracle, toks, n_gen):
    """exact-mode logits for every token fed: prompt tokens, then the oracle's own greedy continuation"""
    lib, h = oracle
    lib.oc_reset(h)
    lg = np.zeros(128256, np.float32)
    out = []
    tok = None
    for i in range(len(toks) + n_gen - 1):
        t = int(toks[i]) if i < len(toks) else tok
        assert lib.oc_step(h, t, 0, lg.ctypes.data_as(C.c_void_p), None) == 0
        out.append(lg.copy())
        tok = int(np.argmax(lg))
    return out


def _margin(lg):
    s = np.sort(lg)
    return float(s[-1] - s[-2])


def test_decode_step_at_the_benchmarked_shape(engine_8b, bench_model):
    import bench
    pre = bench.preflight_8b_parity(engine_8b, bench_model)           # the same check bench.py runs before it times anything
    assert pre["tokens_compared"] == 8 and pre["worst_logit_err_over_scale"] <= 1e-2


def test_batched_prefill_at_the_benchmarked_shape(engine_8b, oracle_8b):
    toks = np.random.Generator(np.random.PCG64(31337)).integers(0, 128000, size=16)
    ref = _oracle_run(oracle_8b, toks, 1)[-1]
    engine_8b.kv_reset()
    lg = engine_8b.prefill(toks)                                       # wgmma GEMMs on the resident 16-bit weights
    scale = float(np.abs(ref).max())
    assert np.isfinite(lg).all() and float(np.abs(lg - ref).max()) <= 1e-2 * scale
    if _margin(ref) > 5e-2:
        assert int(np.argmax(lg)) == int(np.argmax(ref))
    # and the decode kernels continue on the KV pages the prefill wrote
    nxt = int(np.argmax(ref))
    lib, h = oracle_8b
    r2 = np.zeros(128256, np.float32)
    lib.oc_step(h, nxt, 0, r2.ctypes.data_as(C.c_void_p), None)
    l2, _am, _lp = engine_8b.decode_step(nxt)
    assert float(np.abs(l2 - r2).max()) <= 1e-2 * float(np.abs(r2).max())
    engine_8b.kv_reset()


def test_batched_decode_step_at_the_benchmarked_shape(engine_8b, oracle_8b):
    rng = np.random.Generator(np.random.PCG64(4242))
    prompts = [rng.integers(0, 128000, size=n) for n in (9, 5)]
    slots = [engine_8b.seq_open(p, num_predict=3, ignore_eos=True) for p in prompts]
    got = {s: [] for s in slots}
    lgs = {s: [] for s in slots}
    for _ in range(4):
        for slot, tok, lp, done in engine_8b.batch_step():
            lgs[slot].append(engine_8b.seq_logits(slot))
            got[slot].append((tok, lp))
    for s, p in zip(slots, prompts):
        ref = _oracle_run(oracle_8b, p, 3)[len(p) - 1:]                # logits the three generated tokens are drawn from
        assert len(got[s]) == 3
        for i in range(3):
            scale = float(np.abs(ref[i]).max())
            assert float(np.abs(lgs[s][i] - ref[i]).max()) <= 1e-2 * scale, (len(p), i)
            lse = float(ref[i].max() + np.log(np.exp(ref[i] - ref[i].max()).sum()))
            tok, lp = got[s][i]
            assert abs(lp - (float(ref[i][tok]) - lse)) <= 2e-2
            if tok != int(np.argmax(ref[i])):
                assert _margin(ref[i]) <= 5e-2
                break                                                   # a near-tie: the trajectories part ways here
        engine_8b.seq_close(s)
