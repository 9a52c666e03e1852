"""GPU: the streamed prompt pass (GL_PREFILL_WEIGHTS=2; gridllm_b200/csrc/prefill_weights.h) -- each layer's four 16-bit GEMM
operands dequantised into one staging buffer just before their GEMMs -- against the resident 16-bit copy (GL_PREFILL_WEIGHTS=1).

Stated properties: the 16-bit operand dequantisation equals, bit for bit, the one-element-per-thread dequantisation through
rowdot.h's accessors for every weight type and both 16-bit formats; streamed and resident give the same bits on every caller of
the prompt pass; a streamed pass launches exactly 4 kernels per layer more; and a 70B-shaped model (2 layers) streams, matches the
resident copy (512-token prompt) and the C exact oracle (64-token prompt) at the tolerances of tests/test_gpu_8b_shape.py, and serves a generateResponse."""
import asyncio
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

FIXTURES = ["tiny_gguf", "tiny128_gguf", "mid_gguf", "tiny_q8_gguf", "tiny_f16_gguf"]
F32, F16, Q8_0, Q4_K, Q6_K, BF16 = 0, 1, 8, 12, 14, 30


def _engine(path, weights, **kw):
    from gridllm_b200 import native as N
    old = os.environ.get("GL_PREFILL_WEIGHTS")
    os.environ["GL_PREFILL_WEIGHTS"] = str(weights)
    try:
        return N.Engine(path, **kw)
    finally:
        if old is None:
            del os.environ["GL_PREFILL_WEIGHTS"]
        else:
            os.environ["GL_PREFILL_WEIGHTS"] = old


def _toks(n_vocab, seed, n):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, n_vocab - 3, size=n)


# ---- the dequantisation kernel, one matrix at a time ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dq_lib():
    lib = C.CDLL(os.path.join(ROOT, "tests", "dequantcheck", "libdequantcheck.so"))
    lib.dq_check.argtypes = [C.c_int, C.c_void_p] + [C.c_int] * 7 + [C.c_void_p, C.c_void_p]
    return lib


def _gguf_rows(rng, t, rows, cols):
    from oracle import gguf_synth as S
    if t in (Q4_K, Q6_K, Q8_0):
        return np.ascontiguousarray(S.random_blocks(rng, t, rows, cols)).view(np.uint8)
    x = (rng.standard_normal((rows, cols)) * np.exp(rng.uniform(-12, 12, (rows, 1)))).astype(np.float32)
    x[0, :4] = [0.0, -0.0, 70000.0, 1e-8]                      # fp16 overflow and underflow
    if t == F32:
        return x.view(np.uint8)
    if t == F16:
        return x.astype(np.float16).view(np.uint8)
    return (x.view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)


# (type, tile sizes the engine stores it with: a plain matrix and half of a gate / up pair)
TYPES = [(Q4_K, (4, 2)), (Q6_K, (2, 1)), (Q8_0, (2, 1)), (F16, (1,)), (BF16, (1,)), (F32, (1,))]


@pytest.mark.parametrize("t,tiles", TYPES)
@pytest.mark.parametrize("cols", [256, 4096, 8192, 28672])
def test_dequant_is_bit_identical_to_the_element_accessors(dq_lib, t, tiles, cols):
    rng = np.random.Generator(np.random.PCG64(cols * 31 + t))
    for tile_rows in tiles:
        for rows, interleave in ((37, 0), (40, 1), (40, 2)):
            w = _gguf_rows(rng, t, rows, cols)
            dst_rows = 2 * rows if interleave else rows + 5
            row0 = 0 if interleave else 5
            for bf16 in (0, 1):
                new = np.zeros((dst_rows, cols), np.uint16)
                ref = np.zeros((dst_rows, cols), np.uint16)
                rc = dq_lib.dq_check(t, w.ctypes.data_as(C.c_void_p), rows, cols, tile_rows, dst_rows, row0, interleave, bf16,
                                     new.ctypes.data_as(C.c_void_p), ref.ctypes.data_as(C.c_void_p))
                assert rc == 0
                assert np.array_equal(new, ref), (t, cols, tile_rows, interleave, bf16, int((new != ref).sum()))


# ---- streamed == resident on every caller of the prompt pass ----------------------------------------------------------------
@pytest.fixture(scope="module", params=FIXTURES)
def pair(request):
    path = request.getfixturevalue(request.param)
    res = _engine(path, 1, max_ctx=8192, prefix_cache=True)
    st = _engine(path, 2, max_ctx=8192, prefix_cache=True)
    yield res, st
    res.close()
    st.close()


def test_generate_greedy_logits_and_launches(pair):
    res, st = pair
    nl = res.info.n_layer
    p = _toks(res.info.n_vocab, 1, 300)
    a = res.generate(p, num_predict=6, ignore_eos=True, want_logits=True)
    b = st.generate(p, num_predict=6, ignore_eos=True, want_logits=True)
    assert np.array_equal(a.ids, b.ids) and np.array_equal(a.logprobs, b.logprobs)
    for i in range(6):
        assert np.array_equal(res.last_logits(i), st.last_logits(i)), i
    assert b.stats.kernel_launches == a.stats.kernel_launches + 4 * nl        # one prompt pass


def test_seeded_top_k(pair):
    res, st = pair
    p = _toks(res.info.n_vocab, 2, 90)
    kw = dict(num_predict=12, ignore_eos=True, temperature=0.9, top_k=20, seed=1234)
    assert np.array_equal(res.generate(p, **kw).ids, st.generate(p, **kw).ids)


def test_prefill_longer_than_one_pass_and_in_pieces(pair):
    res, st = pair
    p = _toks(res.info.n_vocab, 3, 5000)                                         # 4096 rows, then a paged second pass
    outs = []
    for e in (res, st):
        e.kv_reset()
        lg = e.prefill(p)
        l2, _, _ = e.decode_step(int(np.argmax(lg)))
        e.kv_reset()
        lp1 = e.prefill(p[:1500])
        lp2 = e.prefill(p[1500:1700])
        l3, _, _ = e.decode_step(7)
        e.kv_reset()
        outs.append((lg, l2, lp1, lp2, l3))
    for x, y in zip(*outs):
        assert np.isfinite(x).all() and np.array_equal(x, y)


def test_packed_embed_and_a_long_sequence(pair):
    res, st = pair
    nv = res.info.n_vocab
    seqs = [_toks(nv, 10 + i, n) for i, n in enumerate((12, 200, 700, 33, 2500))]
    a, sa = res.embed(seqs)
    b, sb = st.embed(seqs)
    assert np.isfinite(a).all() and np.array_equal(a, b)
    assert sb.kernel_launches == sa.kernel_launches + 2 * 4 * res.info.n_layer     # one pack, one 2500-row pass


def test_prefix_cache_second_turn(pair):
    res, st = pair
    p1 = _toks(res.info.n_vocab, 4, 150)
    p2 = np.concatenate([p1, _toks(res.info.n_vocab, 5, 60)])
    got = []
    for e in (res, st):
        e.generate(p1, num_predict=4, ignore_eos=True)
        g = e.generate(p2, num_predict=5, ignore_eos=True, want_logits=True)
        got.append((g.ids, [e.last_logits(i) for i in range(5)], g.stats.prompt_eval_count))
    assert got[0][2] == got[1][2] < len(p2)                                      # the second turn reused the first one's pages
    assert np.array_equal(got[0][0], got[1][0])
    for x, y in zip(got[0][1], got[1][1]):
        assert np.array_equal(x, y)


# ---- a 70B-shaped model: Llama-3-70B's layer shapes, 2 layers -----------------------------------------------------------------
@pytest.fixture(scope="module")
def l70_gguf(tmp_path_factory):
    from oracle import gguf_synth as S
    shape = S.LlamaShape("llama3-70b-2layer-synth", 2, 8192, 64, 8, 28672, 128256, 500000.0, 1e-5, 8192)
    path = str(tmp_path_factory.mktemp("l70") / "l70_2layer_q4km.gguf")
    S.build_model(path, shape, "q4_k_m", seed=70, mode="random", rope_freqs=S.llama3_rope_factors(128, 500000.0))
    yield path
    os.remove(path)


def test_70b_shape_streams_like_the_resident_copy_and_the_oracle(l70_gguf):
    toks = _toks(128256, 700, 512)
    res = _engine(l70_gguf, 1, max_ctx=1024)
    st = _engine(l70_gguf, 2, max_ctx=1024)
    a = res.generate(toks, num_predict=16, ignore_eos=True, want_logits=True)
    b = st.generate(toks, num_predict=16, ignore_eos=True, want_logits=True)
    assert np.array_equal(a.ids, b.ids)
    for i in range(16):
        assert np.array_equal(res.last_logits(i), st.last_logits(i)), i
    # against exact arithmetic: the oracle steps one token at a time, so a 64-token prompt keeps it to 80 full-model steps
    toks = toks[:64]
    b = st.generate(toks, num_predict=16, ignore_eos=True, want_logits=True)
    lb = [st.last_logits(i) for i in range(16)]
    res.close()
    st.close()

    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "liboracle_cpu.so"))
    lib.oc_load.restype = C.c_void_p
    lib.oc_load.argtypes = [C.c_char_p, C.c_int]
    lib.oc_step.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.oc_free.argtypes = [C.c_void_p]
    lib.oc_set_threads.argtypes = [C.c_int]
    lib.oc_set_threads(min(32, os.cpu_count() or 8))
    h = lib.oc_load(l70_gguf.encode(), 1024)
    assert h
    try:
        ref = np.zeros(128256, np.float32)
        for t in toks:                                                          # exact mode steps one token at a time
            assert lib.oc_step(h, int(t), 0, ref.ctypes.data_as(C.c_void_p), None) == 0
        for i in range(16):
            scale = float(np.abs(ref).max())
            assert np.isfinite(lb[i]).all() and float(np.abs(lb[i] - ref).max()) <= 1e-2 * scale, i
            lse = float(ref.max() + np.log(np.exp(ref - ref.max()).sum()))
            assert abs(float(b.logprobs[i]) - (float(ref[b.ids[i]]) - lse)) <= 2e-2, i
            if int(b.ids[i]) != int(np.argmax(ref)):
                srt = np.sort(ref)
                assert float(srt[-1] - srt[-2]) <= 5e-2, i
                break                                                           # a near-tie: the trajectories part ways here
            assert lib.oc_step(h, int(b.ids[i]), 0, ref.ctypes.data_as(C.c_void_p), None) == 0
    finally:
        lib.oc_free(h)


def test_70b_shape_generate_response(l70_gguf):
    from gridllm_b200.service import NativeInferenceService
    old = os.environ.get("GL_PREFILL_WEIGHTS")
    os.environ["GL_PREFILL_WEIGHTS"] = "2"
    try:
        svc = NativeInferenceService({"l70:2layer": l70_gguf}, device=0, max_ctx=1024)
        req = {"id": "r70", "model": "l70:2layer", "prompt": "the rain in spain " * 40, "priority": "medium",
               "options": {"num_predict": 8, "temperature": 0, "ignore_eos": True}}
        r = asyncio.new_event_loop().run_until_complete(svc.generateResponse(req))
        svc.close()
    finally:
        if old is None:
            del os.environ["GL_PREFILL_WEIGHTS"]
        else:
            os.environ["GL_PREFILL_WEIGHTS"] = old
    assert r["done"] is True and r["eval_count"] == 8 and r["prompt_eval_count"] >= 40, r
