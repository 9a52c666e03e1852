"""CPU: the prefix-reuse option of gl_generate -- its place in gl_engine_opts, the reuse rule (gridllm_b200/csrc/prefix_reuse.h,
compiled for the host), and the service forwarding the option to the engine."""
import asyncio
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT


def test_engine_opts_layout_matches_the_header():
    from gridllm_b200 import native as N
    E = N.EngineOpts
    assert ctypes.sizeof(E) == 64
    old = {"max_ctx": 0, "act_bits": 4, "use_graph": 8, "use_pdl": 12, "prefill_mode": 16, "max_batch": 20, "kv_pool_tokens": 24,
           "batch_weights": 28}
    assert {k: getattr(E, k).offset for k in old} == old
    assert E.prefix_cache.offset == 32 and E.reserved.offset == 36 and E.reserved.size == 7 * 4
    assert E().prefix_cache == 0                          # a zeroed struct keeps today's behaviour: no reuse
    with open(os.path.join(ROOT, "include", "gridllm_native.h")) as f:
        hdr = f.read()
    body = re.search(r"typedef struct gl_engine_opts \{(.*?)\} gl_engine_opts;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"int32_t\s+(\w+)(\[\d+\])?;", body)
    assert [f[0] for f in fields] == [f[0] for f in E._fields_]
    assert fields[-1] == ("reserved", "[7]")
    assert re.search(r"#define GL_ABI_VERSION 2\b", hdr)


@pytest.fixture(scope="module")
def reuse_lib(tmp_path_factory):
    """CPU build of prefix_reuse.h through tests/hostcheck/prefix_shim.cpp -- test infrastructure only"""
    out = str(tmp_path_factory.mktemp("prefix") / "libprefix.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "prefix_shim.cpp")])
    lib = ctypes.CDLL(out)
    lib.pr_reuse.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return lib


def _reuse(lib, prompt, cached, min_suffix=8):
    p = np.ascontiguousarray(prompt, dtype=np.int32)
    c = np.ascontiguousarray(cached, dtype=np.int32)
    return lib.pr_reuse(p.ctypes.data if len(p) else None, len(p), c.ctypes.data if len(c) else None, len(c), min_suffix)


def _rule(prompt, cached, min_suffix=8):
    """r = max(0, min(L, n_prompt - max(min_suffix, 1))), L = longest common prefix"""
    n = min(len(prompt), len(cached))
    L = next((i for i in range(n) if prompt[i] != cached[i]), n)
    return max(0, min(L, len(prompt) - max(min_suffix, 1)))


def test_reuse_rule_cases(reuse_lib):
    rng = np.random.Generator(np.random.PCG64(5))
    base = rng.integers(0, 1000, size=300).tolist()
    # no common prefix
    assert _reuse(reuse_lib, [1] + base[1:], base) == 0
    # nothing recorded (the record was cleared)
    assert _reuse(reuse_lib, base, []) == 0
    # the same prompt again: all but the last min_suffix positions
    assert _reuse(reuse_lib, base, base) == 300 - 8
    # the previous conversation plus new tokens: the whole record
    assert _reuse(reuse_lib, base + [7] * 50, base) == 300
    # the record is longer than the prompt (the prompt is a prefix of it)
    assert _reuse(reuse_lib, base[:100], base) == 92
    # divergence at k
    for k in (1, 37, 64, 200, 292, 295, 299):
        p = list(base)
        p[k] = (p[k] + 1) % 1000
        assert _reuse(reuse_lib, p, base) == min(k, 300 - 8), k
    # a prompt shorter than min_suffix: nothing is reused
    for n in range(1, 9):
        assert _reuse(reuse_lib, base[:n], base) == 0
    # a minimum below one still evaluates the last prompt token
    assert _reuse(reuse_lib, base, base, min_suffix=0) == 299
    # random cases against the restatement
    for _ in range(200):
        n = int(rng.integers(1, 60))
        c = rng.integers(0, 3, size=int(rng.integers(0, 60))).tolist()
        p = rng.integers(0, 3, size=n).tolist()
        ms = int(rng.integers(0, 10))
        assert _reuse(reuse_lib, p, c, ms) == _rule(p, c, ms), (p, c, ms)


def test_service_forwards_prefix_cache_to_the_engine(tiny_gguf, hostcheck_lib, monkeypatch):
    import oracle_engine
    from gridllm_b200 import service as SV

    class Double(oracle_engine.OracleEngine):
        def __init__(self, gguf_path, device=0, max_ctx=0, **kw):
            super().__init__(gguf_path, device=device, max_ctx=max_ctx, **kw)
            self.kw = dict(kw)

    oracle_engine.use_hostcheck(hostcheck_lib)
    monkeypatch.setattr(SV.N, "Engine", Double)
    monkeypatch.setattr(SV.N, "device_count", lambda: 1)
    for flag in (True, None):
        svc = SV.NativeInferenceService({"tiny:latest": tiny_gguf}, device=0, **({"prefix_cache": flag} if flag else {}))
        try:
            req = {"id": "c1", "model": "tiny:latest", "prompt": "the rain in spain", "priority": "medium",
                   "options": {"num_predict": 4, "temperature": 0, "ignore_eos": True}}
            res = asyncio.new_event_loop().run_until_complete(svc.generateResponse(req))
            eng = svc._engine("tiny:latest")
            assert eng.kw.get("prefix_cache", False) is (flag is True)
            # a second turn that sends the context back still goes to the same engine, whole prompt in hand
            ctx = res["metadata"]["context"] if "metadata" in res and "context" in res["metadata"] else res.get("context")
            assert ctx and ctx[: len(eng.tokenize(req["prompt"]))] == [int(t) for t in eng.tokenize(req["prompt"])]
            req2 = dict(req, id="c2", prompt=" falls mainly", metadata={"context": ctx})
            asyncio.new_event_loop().run_until_complete(svc.generateResponse(req2))
            assert svc._engine("tiny:latest") is eng
        finally:
            svc.close()


def test_napi_shim_reads_the_option():
    with open(os.path.join(ROOT, "host", "napi", "addon.cc")) as f:
        src = f.read()
    assert '"prefixCache"' in src and "o.prefix_cache" in src
    with open(os.path.join(ROOT, "host", "src", "NativeInferenceService.ts")) as f:
        ts = f.read()
    assert "prefixCache" in ts
