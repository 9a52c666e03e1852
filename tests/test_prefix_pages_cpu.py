"""CPU: prompt-prefix page sharing between batch slots (gl_engine_opts batch_prefix_cache) -- the page pool and prefix index of
gridllm_b200/csrc/prefix_pages.h compiled for the host and checked against a Python restatement, the option's place in
gl_engine_opts, and its forwarding by the service and the N-API shim."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

PAGE = 16


@pytest.fixture(scope="module")
def pages_lib(tmp_path_factory):
    """CPU build of prefix_pages.h through tests/hostcheck/pages_shim.cpp -- test infrastructure only"""
    out = str(tmp_path_factory.mktemp("pages") / "libpages.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "pages_shim.cpp")])
    lib = ctypes.CDLL(out)
    vp, i32, p32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p
    lib.pp_new.restype = vp
    lib.pp_new.argtypes = [i32]
    lib.pp_delete.argtypes = [vp]
    lib.pp_alloc.argtypes = [vp, i32, p32]
    lib.pp_ref.argtypes = [vp, i32]
    lib.pp_release.argtypes = [vp, i32]
    lib.pp_match.argtypes = [vp, p32, i32, p32]
    lib.pp_insert.argtypes = [vp, i32, p32, i32]
    lib.pp_forget.argtypes = [vp, i32]
    lib.pp_state.argtypes = [vp, p32, p32, p32]
    lib.pp_reuse.argtypes = [i32, i32, i32]
    return lib


class Pool:
    """the shim's PagePool"""

    def __init__(self, lib, n):
        self.lib, self.n, self.h = lib, n, lib.pp_new(n)

    def close(self):
        self.lib.pp_delete(self.h)

    def alloc(self, k):
        out = np.zeros(max(k, 1), np.int32)
        r = self.lib.pp_alloc(self.h, k, out.ctypes.data)
        return None if r < 0 else out[:k].tolist()

    def ref(self, p):
        self.lib.pp_ref(self.h, p)

    def release(self, p):
        self.lib.pp_release(self.h, p)

    def match(self, ids):
        a = np.ascontiguousarray(ids, np.int32)
        out = np.zeros(len(a) // PAGE + 1, np.int32)
        l = self.lib.pp_match(self.h, a.ctypes.data if len(a) else None, len(a), out.ctypes.data)
        return out[:l].tolist()

    def insert(self, parent, ids16, page):
        a = np.ascontiguousarray(ids16, np.int32)
        return bool(self.lib.pp_insert(self.h, parent, a.ctypes.data, page))

    def forget(self, p):
        self.lib.pp_forget(self.h, p)

    def state(self):
        c, refs, idx = np.zeros(2, np.int32), np.zeros(self.n, np.int32), np.zeros(self.n, np.int32)
        self.lib.pp_state(self.h, c.ctypes.data, refs.ctypes.data, idx.ctypes.data)
        return int(c[0]), int(c[1]), refs.tolist(), idx.tolist()


class Model:
    """Restatement: free list handed out from its back; retained = indexed with no reference; eviction takes the retained page
    with no indexed child released longest ago; the index maps (parent page, 16 ids) to a page."""

    def __init__(self, n):
        self.n = n
        self.free = list(range(n))
        self.refs = [0] * n
        self.node = {}                     # page -> (parent, ids)
        self.key = {}                      # (parent, ids) -> page
        self.stamp = [0] * n
        self.clock = 0
        self.evicted = []

    def children(self, p):
        return sum(1 for q, (par, _) in self.node.items() if par == p)

    def retained(self):
        return [p for p in self.node if self.refs[p] == 0]

    def alloc(self, k):
        if k > len(self.free) + len(self.retained()):
            return None
        out = []
        for _ in range(k):
            if self.free:
                p = self.free.pop()
            else:
                p = min((self.stamp[q], q) for q in self.retained() if self.children(q) == 0)[1]
                self.evicted.append(p)
                self.unindex(p)
            self.refs[p] = 1
            out.append(p)
        return out

    def unindex(self, p):
        par, ids = self.node.pop(p)
        del self.key[(par, ids)]

    def ref(self, p):
        self.refs[p] += 1

    def release(self, p):
        self.refs[p] -= 1
        if self.refs[p] == 0:
            if p in self.node:
                self.clock += 1
                self.stamp[p] = self.clock
            else:
                self.free.append(p)

    def match(self, ids):
        out, parent = [], -1
        for j in range(len(ids) // PAGE):
            p = self.key.get((parent, tuple(ids[j * PAGE:(j + 1) * PAGE])))
            if p is None:
                break
            out.append(p)
            parent = p
        return out

    def insert(self, parent, ids16, page):
        k = (parent, tuple(ids16))
        if k in self.key:
            return False
        self.key[k] = page
        self.node[page] = k
        return True

    def forget(self, p):
        if p in self.node and self.children(p) == 0:
            self.unindex(p)


def _rule(L, n, prefill_min=8):
    """r = 16 floor(min(16 L, n - max(prefill_min, 1)) / 16), at least 0"""
    return max(0, min(PAGE * L, n - max(prefill_min, 1))) // PAGE * PAGE


def test_reuse_rule_cases(pages_lib):
    r = pages_lib.pp_reuse
    assert r(0, 100, 8) == 0                              # nothing indexed
    assert r(4, 100, 8) == 64                             # the whole chain: 92 positions would be allowed
    assert r(6, 100, 8) == 80                             # capped at n - 8 = 92, cut down to a page boundary
    assert r(6, 96, 8) == 80                              # a prompt equal to a cached one of 6 full pages: 88 -> 80
    assert r(2, 40, 8) == 32 and r(2, 39, 8) == 16        # the prefill_min floor moves the cut across a page boundary
    assert r(1, 23, 8) == 0 and r(1, 24, 8) == 16
    assert r(3, 64, 0) == 48 and r(4, 64, 0) == 48        # a minimum below one still evaluates the last prompt token
    assert r(5, 8, 8) == 0 and r(5, 1, 8) == 0            # prompts not longer than the minimum share nothing
    for L in range(0, 12):
        for n in range(1, 200, 7):
            for pm in (0, 1, 8, 20):
                got = r(L, n, pm)
                assert got == _rule(L, n, pm) and got % PAGE == 0 and got <= PAGE * L, (L, n, pm)
                assert got == 0 or n - got >= max(pm, 1), (L, n, pm)


def test_match_is_exact_and_page_aligned(pages_lib):
    pool = Pool(pages_lib, 32)
    try:
        ids = list(range(100, 150))                       # 3 full pages + 2 ids
        pages = pool.alloc(4)
        parent = -1
        for j in range(3):
            assert pool.insert(parent, ids[16 * j:16 * j + 16], pages[j])
            parent = pages[j]
        assert pool.match(ids) == pages[:3]
        assert pool.match(ids[:47]) == pages[:2]          # only full pages of the query count
        for k in (0, 15, 16, 31, 40):                     # an id mismatch inside a page ends the chain before that page
            q = list(ids)
            q[k] += 1
            assert pool.match(q) == pages[:k // 16]
        # the same 16 ids under another parent are another node
        assert pool.match(ids[16:32] + ids[16:32]) == []
        assert not pool.insert(-1, ids[:16], pages[3])    # a key is indexed once
    finally:
        pool.close()


def _check(pool, model, live):
    """shim == restatement, and the invariants stated in prefix_pages.h"""
    n_free, n_ret, refs, idx = pool.state()
    assert refs == model.refs
    assert [p for p in range(pool.n) if idx[p]] == sorted(model.node)
    assert n_free == len(model.free) and n_ret == len(model.retained())
    held = [p for t in live.values() for p in t]
    counts = np.bincount(np.asarray(held, np.int64), minlength=pool.n) if held else np.zeros(pool.n, np.int64)
    assert counts.tolist() == refs                        # every reference is one table entry of a live holder
    referenced = sum(1 for c in refs if c > 0)
    assert n_free + n_ret + referenced == pool.n          # pages are conserved
    for p in model.node:                                  # a referenced indexed page's parent is referenced too
        par = model.node[p][0]
        if refs[p] > 0 and par >= 0:
            assert refs[par] > 0


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_operations_against_the_restatement(pages_lib, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    N = 96
    pool, model = Pool(pages_lib, N), Model(N)
    bases = [rng.integers(0, 4, size=160).tolist() for _ in range(3)]
    live = {}                                             # holder -> its table (shared pages first)
    nxt = 0
    try:
        for step in range(1500):
            op = rng.random()
            if op < 0.45:                                 # open a sequence: share, allocate its own pages, index its prompt
                b = bases[int(rng.integers(0, 3))]
                n = int(rng.integers(1, 150))
                pre = int(rng.integers(0, n + 1))
                prompt = b[:pre] + rng.integers(0, 4, size=n - pre).tolist()
                n_pred = int(rng.integers(1, 40))
                m = pool.match(prompt)
                assert m == model.match(prompt)
                r = _rule(len(m), n)
                shared = m[:r // PAGE]
                for p in shared:
                    pool.ref(p)
                    model.ref(p)
                own_n = (n + n_pred + PAGE - 1) // PAGE - r // PAGE
                before = {p for t in live.values() for p in t}
                ev0 = len(model.evicted)
                own = pool.alloc(own_n)
                assert own == model.alloc(own_n)
                if own is None:
                    for p in shared:
                        pool.release(p)
                        model.release(p)
                    _check(pool, model, live)
                    continue
                assert not (set(own) & before) and not (set(own) & set(shared))   # never a referenced page
                assert len(set(own)) == len(own)
                for p in model.evicted[ev0:]:
                    assert p in own
                table = shared + own
                for j in range(r // PAGE, n // PAGE):
                    par = table[j - 1] if j else -1
                    ok = pool.insert(par, prompt[PAGE * j:PAGE * (j + 1)], table[j])
                    assert ok == model.insert(par, tuple(prompt[PAGE * j:PAGE * (j + 1)]), table[j])
                    if not ok:
                        break
                live[nxt] = table
                nxt += 1
            elif op < 0.85 and live:                      # close one
                k = list(live)[int(rng.integers(0, len(live)))]
                for p in live.pop(k):
                    pool.release(p)
                    model.release(p)
            elif op < 0.95:                               # a private allocation under pressure (gl_generate's pages)
                k = int(rng.integers(1, 30))
                got = pool.alloc(k)
                assert got == model.alloc(k)
                if got is not None:
                    live[nxt] = got
                    nxt += 1
            elif live:                                    # a pass that failed: its newest leaf leaves the index again
                k = list(live)[-1]
                p = live[k][-1]
                pool.forget(p)
                model.forget(p)
            _check(pool, model, live)
        assert model.evicted, "the sequence never put the pool under pressure"
        for t in live.values():
            for p in t:
                pool.release(p)
                model.release(p)
        live.clear()
        _check(pool, model, live)
        assert pool.alloc(N) is not None                  # with nothing open, every retained page can be evicted
    finally:
        pool.close()


def test_eviction_takes_least_recently_released_leaves_first(pages_lib):
    pool = Pool(pages_lib, 8)
    try:
        a, b = pool.alloc(3), pool.alloc(3)               # two chains of three indexed pages
        for t, base in ((a, 0), (b, 100)):
            par = -1
            for j, p in enumerate(t):
                assert pool.insert(par, list(range(base + 16 * j, base + 16 * j + 16)), p)
                par = p
        for p in a:                                       # a closes first: a[0] is the oldest page, but not a leaf
            pool.release(p)
        for p in b:
            pool.release(p)
        n_free, n_ret, _, _ = pool.state()
        assert (n_free, n_ret) == (2, 6)
        assert pool.alloc(2) is not None                  # the free pages go first
        assert pool.alloc(1) == [a[2]]                    # then a's leaf, then its parent (now a leaf), ...
        assert pool.alloc(2) == [a[1], a[0]]
        assert pool.alloc(1) == [b[2]]
        assert pool.alloc(3) is None                      # live references hold the rest: nothing is taken
        assert pool.state()[:2] == (0, 2)
    finally:
        pool.close()


def test_engine_opts_keep_their_layout_with_the_option():
    from gridllm_b200 import native as N
    E = N.EngineOpts
    assert ctypes.sizeof(E) == 64 and E.prefix_cache.offset == 32 and E.reserved.offset == 36
    o = E()
    assert o.batch_prefix_cache == 0                      # a zeroed struct: off
    o.batch_prefix_cache = 1
    assert list(o.reserved) == [1, 0, 0, 0, 0, 0, 0] and o.prefix_cache == 0
    with open(os.path.join(ROOT, "include", "gridllm_native.h")) as f:
        hdr = f.read()
    assert re.search(r"#define GL_OPT_BATCH_PREFIX_CACHE\s+0\b", hdr) and E.GL_OPT_BATCH_PREFIX_CACHE == 0
    with open(os.path.join(ROOT, "gridllm_b200", "csrc", "c_api.cpp")) as f:
        assert "GL_OPT_BATCH_PREFIX_CACHE" in f.read()


def test_service_forwards_batch_prefix_cache(tiny_gguf, monkeypatch):
    from gridllm_b200 import service as SV

    class Double:
        def __init__(self, gguf_path, device=0, max_ctx=0, **kw):
            self.kw = dict(kw)

        def close(self):
            pass

    monkeypatch.setattr(SV.N, "Engine", Double)
    monkeypatch.setattr(SV.N, "device_count", lambda: 1)
    for flag in (True, None):
        svc = SV.NativeInferenceService({"tiny:latest": tiny_gguf}, device=0, max_batch=8,
                                        **({"batch_prefix_cache": flag} if flag else {}))
        eng = svc._engine("tiny:latest")
        assert eng.kw.get("batch_prefix_cache", False) is (flag is True) and eng.kw["max_batch"] == 8


def test_napi_shim_and_ts_pass_the_option():
    with open(os.path.join(ROOT, "host", "napi", "addon.cc")) as f:
        src = f.read()
    assert '"batchPrefixCache"' in src and "GL_OPT_BATCH_PREFIX_CACHE" in src
    with open(os.path.join(ROOT, "host", "src", "NativeInferenceService.ts")) as f:
        assert "batchPrefixCache" in f.read()
