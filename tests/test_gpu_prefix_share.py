"""GPU: prompt-prefix KV pages shared between batch slots (gl_engine_opts batch_prefix_cache).

Every case runs the same opens, steps and closes, in the same order and batch composition, on an engine with the option off
and on one with it on, and requires the same bits: first-token logits (gl_seq_logits right after the open), every id and
logprob, and the logits of every step.  On the engine with the option, prompt_eval_count and gl_batch_counters out[7] show how
much of each prompt came from shared pages."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIXTURES = ["tiny_gguf", "tiny128_gguf"]          # head dim 64 (GQA 2:1) and 128 (GQA 4:1)
SCHEMA = {"type": "object", "properties": {"a": {"type": "integer"}, "b": {"type": "string"}}, "required": ["a"]}


def _engine(path, on, **kw):
    from gridllm_b200 import native as N
    kw.setdefault("max_batch", 32)
    kw.setdefault("max_ctx", 4096)
    return N.Engine(path, batch_prefix_cache=on, **kw)


def _toks(e, seed, n):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, e.info.n_vocab - 3, size=n).astype(np.int32)


class Run:
    """one engine and what it produced, in order"""

    def __init__(self, e):
        self.e, self.bits, self.evals = e, [], []

    def open(self, prompts, opts=None):
        opts = opts or [{}] * len(prompts)
        full = [dict({"num_predict": 64, "ignore_eos": True}, **o) for o in opts]
        slots = self.e.seq_open_many(prompts, full) if len(prompts) > 1 else [self.e.seq_open(prompts[0], **full[0])]
        assert all(s >= 0 for s in slots), slots
        for s in slots:
            self.bits.append(("first", self.e.seq_logits(s)))
            self.evals.append(self.e.seq_stats(s).prompt_eval_count)
        return slots

    def step(self, k):
        for _ in range(k):
            for slot, tok, lp, done in self.e.batch_step():
                self.bits.append(("step", np.array([slot, tok], np.int64), np.float32(lp), self.e.seq_logits(slot)))

    def close(self, slots):
        for s in slots:
            self.e.seq_close(s)

    def generate(self, prompt, n):
        g = self.e.generate(prompt, num_predict=n, ignore_eos=True, want_logits=True)
        self.bits.append(("gen", g.ids, g.logprobs, np.stack([self.e.last_logits(i) for i in range(n)])))
        return g


def _same(off, on):
    assert len(off.bits) == len(on.bits)
    for i, (a, b) in enumerate(zip(off.bits, on.bits)):
        assert a[0] == b[0], i
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(np.asarray(x), np.asarray(y)), (i, a[0])


def _both(path, scenario, **kw):
    runs = []
    for on in (False, True):
        e = _engine(path, on, **kw)
        r = Run(e)
        scenario(r)
        runs.append(r)
        r.counters = e.batch_counters()
        e.close()
    _same(*runs)
    return runs


@pytest.mark.parametrize("fixture", FIXTURES)
def test_retained_pages_and_a_sharer_that_decodes(fixture, request):
    path = request.getfixturevalue(fixture)
    e0 = _engine(path, False)
    pre, a_suf, b_suf = _toks(e0, 1, 100), _toks(e0, 2, 20), _toks(e0, 3, 37)
    e0.close()
    A, B = np.concatenate([pre, a_suf]), np.concatenate([pre, b_suf])

    def scenario(r):
        [a] = r.open([A])
        r.step(5)
        r.close([a])                                   # A's six full prompt pages stay retained
        [b] = r.open([B])                              # 1: shares 96 positions of A's closed pages
        r.step(64)                                     # 2: a sharer decodes 64 tokens ...
        r.close([b])
        [a2] = r.open([A])                             # ... and the shared pages still hold A's prompt, bit for bit
        r.step(3)
        r.close([a2])

    off, on = _both(path, scenario)
    assert off.evals == [120, 137, 120]
    assert on.evals == [120, 137 - 96, 120 - 112]      # A again: all seven full pages, down to the 8-token minimum
    assert off.counters["shared_tokens"] == 0 and on.counters["shared_tokens"] == 96 + 112
    assert on.counters["prefill_tokens"] == 120 + 41 + 8


@pytest.mark.parametrize("fixture", FIXTURES)
@pytest.mark.parametrize("n_seq", [8, 24])
def test_one_call_with_a_common_prefix(fixture, n_seq, request):
    path = request.getfixturevalue(fixture)
    e0 = _engine(path, False)
    pre = _toks(e0, 10, 200)
    prompts = [np.concatenate([pre, _toks(e0, 100 + i, 30 + i)]) for i in range(n_seq)]
    e0.close()

    def scenario(r):
        slots = r.open(prompts)                        # the first owns the prefix, the others share it in the same pack(s)
        r.step(4)
        r.close(slots)

    off, on = _both(path, scenario)
    assert off.evals == [len(p) for p in prompts]
    assert on.evals == [len(prompts[0])] + [len(p) - 192 for p in prompts[1:]]
    assert on.counters["shared_tokens"] == 192 * (n_seq - 1)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_prompt_longer_than_a_pack(fixture, request):
    path = request.getfixturevalue(fixture)
    e0 = _engine(path, False)
    A = _toks(e0, 20, 2200)
    B = np.concatenate([A[:2100], _toks(e0, 21, 150)])
    e0.close()

    def scenario(r):
        [a] = r.open([A], [{"num_predict": 8}])
        r.step(2)
        r.close([a])
        [b] = r.open([B], [{"num_predict": 8}])        # a single-sequence prompt pass from position 2096
        r.step(8)
        r.close([b])

    off, on = _both(path, scenario)
    assert on.evals == [2200, 2250 - 2096]


def test_penalties_json_and_schema_rows_among_sharers(tiny_gguf):
    e0 = _engine(tiny_gguf, False)
    pre = _toks(e0, 30, 70)
    prompts = [np.concatenate([pre, _toks(e0, 300 + i, 12 + 3 * i)]) for i in range(5)]
    e0.close()
    opts = [{}, {"repeat_penalty": 1.3, "presence_penalty": 0.5, "repeat_last_n": -1},
            {"format": "json", "num_predict": 24, "ignore_eos": False}, {"format": SCHEMA, "num_predict": 24, "ignore_eos": False},
            {"temperature": 0.8, "top_k": 20, "seed": 7, "frequency_penalty": 0.4}]

    def scenario(r):
        slots = r.open(prompts, opts)
        r.step(24)
        r.close(slots)

    off, on = _both(tiny_gguf, scenario)
    assert on.evals == [len(prompts[0])] + [len(p) - 64 for p in prompts[1:]]


def test_only_prompt_pass_pages_are_shared(tiny_gguf):
    e0 = _engine(tiny_gguf, False)
    A = _toks(e0, 40, 40)                              # two full prompt pages, then a partial one
    e0.close()
    gen = []

    def scenario(r):
        [a] = r.open([A], [{"num_predict": 30}])
        before = len(r.bits)
        r.step(30)
        ids = [int(b[1][1]) for b in r.bits[before:]]
        gen.append(ids)
        r.close([a])
        B = np.concatenate([A, np.asarray(ids, np.int32), _toks(r.e, 41, 10)])   # the closed prompt, its reply, a new turn
        [b] = r.open([B])
        r.step(4)
        r.close([b])

    off, on = _both(tiny_gguf, scenario)
    assert gen[0] == gen[1]
    assert on.evals == [40, 40 + 30 + 10 - 32]          # pages of decode-step rows are never indexed


@pytest.mark.parametrize("fixture", FIXTURES)
def test_small_pool_evicts_retained_pages(fixture, request):
    from gridllm_b200 import native as N
    path = request.getfixturevalue(fixture)
    kw = dict(max_batch=4, max_ctx=512, kv_pool_tokens=512)           # 32 pages
    e0 = _engine(path, False, **kw)
    pre = _toks(e0, 50, 64)
    ps = [np.concatenate([pre, _toks(e0, 500 + i, 40)]) for i in range(3)] + [_toks(e0, 600 + i, 100) for i in range(3)]
    big = _toks(e0, 700, 300)
    e0.close()
    nomem = []

    def scenario(r):
        for p in ps:                                   # each leaves up to six indexed pages retained
            [s] = r.open([p], [{"num_predict": 16}])
            r.step(2)
            r.close([s])
        [s] = r.open([big], [{"num_predict": 180}])    # 30 of the 32 pages: taken by eviction on the engine with the option
        try:
            r.e.seq_open(_toks(r.e, 701, 40), num_predict=16, ignore_eos=True)
            nomem.append(False)
        except N.NativeError as err:
            nomem.append(N.STATUS_NAMES.get(err.code) == "GL_ERR_NOMEM")
        r.step(3)
        r.close([s])
        r.generate(ps[0], 8)                           # gl_generate's pages come out of the same pool
        [t] = r.open([ps[1]], [{"num_predict": 16}])
        r.step(2)
        r.close([t])

    off, on = _both(path, scenario, **kw)
    assert nomem == [True, True]                       # live sequences hold the pool: NOMEM with and without the option
    assert on.evals[1] == 104 - 64 and on.evals[2] == 104 - 64


@pytest.mark.parametrize("fixture", FIXTURES)
def test_no_match_gives_the_launches_of_the_option_off(fixture, request):
    path = request.getfixturevalue(fixture)
    e0 = _engine(path, False)
    prompts = [_toks(e0, 800 + i, 20 + 17 * i) for i in range(6)]
    e0.close()
    launches = []

    def scenario(r):
        slots = r.open(prompts)
        launches.append([r.e.seq_stats(s).kernel_launches for s in slots])
        r.step(6)
        r.close(slots)

    off, on = _both(path, scenario)
    assert launches[0] == launches[1]
    assert off.counters["launches"] == on.counters["launches"] and on.counters["shared_tokens"] == 0
    assert on.evals == off.evals == [len(p) for p in prompts]
