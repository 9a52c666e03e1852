"""CPU: the context shift (gl_engine_opts context_shift; include/gridllm_native.h) -- the ABI words, the rule as the engine
compiles it (gridllm_b200/csrc/context_shift.h through tests/hostcheck/shift_shim.cpp) against its Python restatement
(tests/shift_oracle.py), the oracle's shift against a direct float64 rotation, and the service's mapping of the Ollama options."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import shift_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "gridllm_native.h")


def test_abi_layout():
    from gridllm_b200 import native as N
    assert ctypes.sizeof(N.SampleOpts) == 72
    assert N.SampleOpts.num_keep.offset == 68
    assert N.EngineOpts.GL_OPT_CONTEXT_SHIFT == 1
    assert N.EngineOpts.reserved.offset + 4 * N.EngineOpts.GL_OPT_CONTEXT_SHIFT == 40
    assert ctypes.sizeof(N.EngineOpts) == 64
    o = N.EngineOpts()
    o.context_shift = 1
    assert o.reserved[1] == 1 and o.reserved[0] == 0 and o.batch_prefix_cache == 0
    text = open(HEADER).read()
    assert re.search(r"#define GL_OPT_CONTEXT_SHIFT 1\b", text)
    assert re.search(r"int32_t\s+num_keep;\s*\}\s*gl_sample_opts;", text)
    for phrase in ("d = ceil((W - k) / 2)", "num_predict <= W", "GL_ERR_UNSUPPORTED", "record keeps positions [0, k)"):
        assert phrase in text, phrase


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """CPU build of context_shift.h through tests/hostcheck/shift_shim.cpp -- test infrastructure only"""
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    out = str(tmp_path_factory.mktemp("shift") / "libshift_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "shift_shim.cpp")])
    return ctypes.CDLL(out)


@pytest.mark.parametrize("W", [16, 17, 64, 2048, 8192])
def test_rule_matches_the_restatement(shim, W):
    for n_prompt in (1, 5, W - 1, W, W + 1, 3 * W + 7):
        for num_keep in (-1, 0, 1, 4, 15, 16, 17, W - 2, W - 1, W, W + 100):
            k = shim.cs_keep(num_keep, n_prompt, W)
            assert k == SO.keep_count(num_keep, n_prompt, W)
            assert 0 <= k <= W - 1
            d = shim.cs_discard(W, k)
            assert d == SO.discard(W, k) and d >= 1 and d == -(-(W - k) // 2)
            rows = shim.cs_rows(W, k, d)
            assert rows == W - k - d and rows >= 0
            assert d >= rows                           # the rule's discard: source and destination never overlap
            prompt = np.arange(1000, 1000 + n_prompt, dtype=np.int32)
            out = np.zeros(max(n_prompt, W), dtype=np.int32)
            m = shim.cs_cut(prompt.ctypes.data_as(ctypes.c_void_p), n_prompt, W, k, d, out.ctypes.data_as(ctypes.c_void_p))
            want = SO.cut_prompt(prompt, W, k)
            assert list(out[:m]) == want
            if n_prompt >= W:
                assert m == W - d and want[:k] == list(prompt[:k]) and (W - d - k == 0 or want[-1] == prompt[-1])


def test_num_keep_minus_one_and_clamping():
    assert SO.keep_count(-1, 10, 64) == 10
    assert SO.keep_count(-1, 100, 64) == 63 and SO.discard(64, 63) == 1
    assert SO.keep_count(100, 5, 64) == 63
    assert SO.discard(64, 4) == 30 and SO.discard(64, 0) == 32 and SO.discard(8192, 4) == 4094
    assert SO.cut_prompt(list(range(200)), 64, 63) == list(range(63))


def test_chunk_boundaries(shim):
    for W in (64, 2048):
        for pos in range(W - 40, W + 1):
            for first in (0, 1):
                for chunk, rem in ((8, 100), (32, 5), (32, 1000)):
                    n = shim.cs_chunk(chunk, rem, pos, W, first)
                    assert n == SO.chunk_steps(chunk, rem, pos, W, bool(first))
                    if pos < W or first:
                        assert n >= 1
                    assert pos + n - first <= W                # no step of the chunk writes position W


def test_oracle_shift_is_a_float64_rotation(tmp_path):
    from oracle import gguf_synth as S, llama_oracle as O
    path = str(tmp_path / "tiny.gguf")
    S.build_model(path, S.TINY, "q4_k_m", seed=3)
    m = O.load_gguf(path)
    orc = O.LlamaOracle(m, act="exact", kv_f16=True)
    rng = np.random.Generator(np.random.PCG64(5))
    for t in rng.integers(0, m.n_vocab - 3, size=40):
        orc.step(int(t))
    W, keep = 40, 4
    d = SO.discard(W, keep)
    k0 = [[np.array(r) for r in layer] for layer in orc.k]
    v0 = [[np.array(r) for r in layer] for layer in orc.v]
    SO.shift(orc, keep, d)
    assert orc.pos == W - d
    hd, kv = m.head_dim, m.n_head_kv
    for il in range(m.n_layer):
        assert len(orc.k[il]) == W - d and len(orc.v[il]) == W - d
        for j in range(keep):
            assert np.array_equal(orc.k[il][j], k0[il][j])
        for j in range(W - keep - d):
            src = k0[il][keep + d + j].reshape(kv, hd // 2, 2)
            c, s = orc.cos[d].astype(np.float64), orc.sin[d].astype(np.float64)
            ang = np.arctan2(s, c)                     # the table's own angle, rotated back in float64
            direct = np.stack([src[..., 0] * np.cos(-ang) - src[..., 1] * np.sin(-ang),
                               src[..., 0] * np.sin(-ang) + src[..., 1] * np.cos(-ang)], axis=-1).reshape(-1)
            want = direct.astype(np.float32).astype(np.float16).astype(np.float64)
            got = orc.k[il][keep + j]
            ulp = np.spacing(np.abs(want).astype(np.float16)).astype(np.float64)
            assert np.all(np.abs(got - want) <= ulp)
            assert np.array_equal(orc.v[il][keep + j], v0[il][keep + d + j])
    # the shifted cache still decodes: one more step at position W - d
    assert np.isfinite(orc.step(7)).all()


class _Info:
    def __init__(self, n_ctx):
        self.n_ctx = n_ctx
        self.has_tokenizer = 0


class _Eng:
    def __init__(self, n_ctx):
        self.info = _Info(n_ctx)


def _svc(**kw):
    from gridllm_b200.service import NativeInferenceService
    return NativeInferenceService({}, **kw)


def test_service_plan_with_the_switch_off_is_unchanged():
    svc = _svc()
    eng = _Eng(64)
    ids = np.arange(60, dtype=np.int32)
    n, _, kw, _, _ = svc._plan(eng, ids, 128, {}, None)
    assert n == 4 and "num_keep" not in kw
    n, _, kw, _, _ = svc._plan(eng, ids, -1, {"num_keep": 10}, None)
    assert n == 4 and "num_keep" not in kw
    n, _, kw, _, _ = svc._plan(eng, np.arange(10, dtype=np.int32), 20, {}, None)
    assert n == 20 and "num_keep" not in kw
    assert "context_shift" not in svc._engine_kw


def test_service_plan_with_context_shift():
    svc = _svc(context_shift=True)
    assert svc._engine_kw.get("context_shift") is True
    eng = _Eng(64)
    long_ids = np.arange(200, dtype=np.int32)                     # longer than the context: answered, not failed
    n, _, kw, _, _ = svc._plan(eng, long_ids, 30, {}, None)
    assert n == 30 and kw["num_keep"] == 4
    n, _, kw, _, _ = svc._plan(eng, long_ids, -1, {"num_keep": -1}, None)
    assert n == 64 and kw["num_keep"] == -1
    n, _, kw, _, _ = svc._plan(eng, np.arange(60, dtype=np.int32), 500, {"num_keep": 12}, None)
    assert n == 64 and kw["num_keep"] == 12                       # capped at W, not at W - len(ids)
    with pytest.raises(RuntimeError):
        svc._plan(eng, long_ids, 10, {"num_keep": -2}, None)
    batched = _svc(context_shift=True, max_batch=4)
    assert batched._engine_kw == {"context_shift": True, "max_batch": 4}
