"""GPU parity of continuous batching inside one engine (SURVEY.md section 8f.1; gl_seq_open / gl_batch_step / gl_seq_close).

Reference side: the worker drops a second assignment while busy (client/src/services/WorkerClientService.ts:500-505) and the
server hands out MAX_CONCURRENT_JOBS_PER_WORKER = 1 job per worker (server/src/config/index.ts:31); with the limit raised the
native worker steps all the jobs it holds together.  The contract checked here:
  * every sequence of a batch matches the ORACLE run on that sequence alone (logits within the batched-GEMM tolerance of
    tests/test_gpu_decode.py -- 1e-2 * max|logit| vs exact activations, fp16 tensor-core arithmetic -- logprob within 2e-2,
    token ids equal wherever the oracle's top-1/top-2 margin exceeds 5e-2);
  * a sequence's tokens do not depend on who shares its batch: alone or among others, same ids and (same bucket) same bits;
  * sequences join and leave between steps; closing returns pages; running out of slots / pages is an error, not a crash;
  * per-sequence sampling options (greedy and the seeded top-k / top-p draw) are honoured inside one batch;
  * stop tokens end one sequence without disturbing the others."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODES = [1, 2]          # gl_engine_opts.batch_weights: 1 = resident 16-bit copy, 2 = quantised weights dequantised inside the GEMM


def _engine(path, **kw):
    from gridllm_b200 import native as N
    kw.setdefault("max_batch", 16)
    return N.Engine(path, **kw)


def _drain(e, want, logits=None):
    """step until every slot in `want` (slot -> number of tokens) has produced its tokens; returns slot -> (ids, logprobs)"""
    out = {s: ([], []) for s in want}
    guard = 0
    while any(len(out[s][0]) < want[s] for s in want):
        guard += 1
        assert guard < 10000
        for slot, tok, lp, done in e.batch_step():
            if slot in out and len(out[slot][0]) < want[slot]:
                if logits is not None:
                    logits.setdefault(slot, []).append(e.seq_logits(slot))
                out[slot][0].append(int(tok))
                out[slot][1].append(float(lp))
    return out


def _check_against_oracle(ref, ids, lps, logits, tag):
    for i in range(len(ids)):
        scale = float(np.abs(ref["logits"][i]).max())
        err = float(np.abs(logits[i] - ref["logits"][i]).max())
        assert err <= 1e-2 * scale, (tag, "logits", i, err, scale)
        assert abs(lps[i] - float(ref["logprobs"][i])) <= 2e-2, (tag, "logprob", i)
        if ids[i] != int(ref["ids"][i]):
            assert ref["margins"][i] <= 5e-2, (tag, "token id", i, ref["margins"][i])
            return i                                   # trajectories part ways on a near-tie: nothing further to compare
    return len(ids)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("fixture", ["tiny_gguf", "tiny128_gguf", "mid_gguf"])
def test_every_sequence_of_a_batch_matches_the_oracle(fixture, mode, request):
    from oracle import llama_oracle as O
    path = request.getfixturevalue(fixture)
    m = O.load_gguf(path)
    e = _engine(path, batch_weights=mode)
    lens = (5, 40, 17, 130, 9, 64)                     # below and above the batched-prefill threshold, across page boundaries
    prompts = [np.random.Generator(np.random.PCG64(100 + i)).integers(0, m.n_vocab - 3, size=n) for i, n in enumerate(lens)]
    slots = [e.seq_open(p, num_predict=10, ignore_eos=True) for p in prompts]
    lg = {}
    got = _drain(e, {s: 10 for s in slots}, lg)
    for s, p in zip(slots, prompts):
        ref = O.LlamaOracle(m, act="exact", kv_f16=True).generate(p, 10)
        n_ok = _check_against_oracle(ref, got[s][0], got[s][1], lg[s], (fixture, mode, len(p)))
        assert n_ok >= 1
        e.seq_close(s)
    e.close()


@pytest.mark.parametrize("mode", MODES)
def test_tokens_do_not_depend_on_who_shares_the_batch(tiny128_gguf, mode):
    e = _engine(tiny128_gguf, batch_weights=mode)
    rng = np.random.Generator(np.random.PCG64(7))
    prompts = [rng.integers(0, e.info.n_vocab - 3, size=n) for n in (33, 12, 70, 20)]
    alone = []
    for p in prompts:                                   # each sequence on its own (batch of one)
        s = e.seq_open(p, num_predict=12, ignore_eos=True)
        lg = {}
        ids, lps = _drain(e, {s: 12}, lg)[s]
        alone.append((ids, lps, lg[s]))
        e.seq_close(s)
    slots = [e.seq_open(p, num_predict=12, ignore_eos=True) for p in prompts]      # ... and all together
    lg = {}
    got = _drain(e, {s: 12 for s in slots}, lg)
    for s, (ids, lps, lgs) in zip(slots, alone):
        assert got[s][0] == ids                        # who shares the batch does not change a sequence
        # same bucket (<= 8 rows): the same kernels, grids and summation orders ran -- bit-identical logits
        assert all(np.array_equal(a, b) for a, b in zip(lg[s], lgs))
        e.seq_close(s)
    # against the single-sequence path (a different GEMV arithmetic: int dot products vs fp16 tensor cores): ids agree
    # wherever that path's own top-1/top-2 margin is clear of the two paths' tolerance
    for p, (ids, _lps, _lg) in zip(prompts, alone):
        g = e.generate(p, num_predict=12, ignore_eos=True, want_logits=True)
        for i in range(12):
            if int(g.ids[i]) != ids[i]:
                lgi = e.last_logits(i)
                srt = np.sort(lgi)
                assert srt[-1] - srt[-2] <= 2e-2 * float(np.abs(lgi).max()), (i, srt[-1] - srt[-2])
                break
    e.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode,n_seq,max_batch", [pytest.param(m_, 28, 32, id=str(m_)) for m_ in MODES] +
                         [pytest.param(m_, n_, b_, id=f"{m_}-{n_}seq") for n_, b_ in ((40, 64), (100, 128)) for m_ in MODES])
def test_large_batch_long_contexts(tiny128_gguf, mode, n_seq, max_batch):
    """28 sequences (the 32-row bucket: two attention splits per KV head) with 300..700-token contexts (20+ KV pages per split:
    several TMA tiles per CTA, partial merge) -- the shape of BASELINE config 3 at test size.  40 sequences run bucket 64
    (qgemm with NB = 64 under batch_weights 2) and 100 sequences bucket 128 (gemm_tc5 at m = 128 on the resident 16-bit
    weights).  Spot-checked against the oracle on four of them; all of them must finish, with finite logprobs."""
    from oracle import llama_oracle as O
    m = O.load_gguf(tiny128_gguf)
    e = _engine(tiny128_gguf, max_batch=max_batch, max_ctx=1024, batch_weights=mode)
    rng = np.random.Generator(np.random.PCG64(2024))
    lens = [int(x) for x in rng.integers(300, 700, size=n_seq)]
    prompts = [rng.integers(0, m.n_vocab - 3, size=n) for n in lens]
    slots = [e.seq_open(p, num_predict=6, ignore_eos=True) for p in prompts]
    lg = {}
    got = _drain(e, {s: 6 for s in slots}, lg)
    assert all(len(got[s][0]) == 6 and np.isfinite(got[s][1]).all() for s in slots)
    for k in (0, 9, 17, n_seq - 1):
        ref = O.LlamaOracle(m, act="exact", kv_f16=True).generate(prompts[k], 6)
        assert _check_against_oracle(ref, got[slots[k]][0], got[slots[k]][1], lg[slots[k]], ("large", mode, lens[k])) >= 1
    for s in slots:
        e.seq_close(s)
    ms, launches, wbytes = e.time_batch_step(min(max_batch, 32), 500, iters=4)
    assert ms > 0 and launches > 0
    e.close()


@pytest.mark.parametrize("mode", MODES)
def test_open_many_equals_open_one_by_one(tiny128_gguf, mode):
    """gl_seq_open_many: the prompts share packed prompt passes (each attends only to itself, caches K / V through its own page
    table) and one lm_head pass.  Every sequence must continue exactly as if it had been opened alone: same first token and
    logits bits (its rows never see a neighbour), same later tokens; prompts that do not fit come back as -1 and can be retried."""
    e = _engine(tiny128_gguf, max_batch=8, max_ctx=1024, batch_weights=mode)
    rng = np.random.Generator(np.random.PCG64(99))
    lens = (300, 9, 512, 130, 4, 77, 256, 600, 33, 20)              # one shorter than the packed pass takes, several packs, 10 > 8 slots
    prompts = [rng.integers(0, e.info.n_vocab - 3, size=n) for n in lens]
    opts = [dict(num_predict=6, ignore_eos=True) for _ in lens]
    opts[3] = dict(num_predict=6, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.9, seed=11)       # a sampled one among them
    alone = []
    for p, o in zip(prompts, opts):
        s = e.seq_open(p, **o)
        lg = {}
        ids, lps = _drain(e, {s: 6}, lg)[s]
        alone.append((ids, lps, lg[s]))
        e.seq_close(s)
    slots = e.seq_open_many(prompts, opts)
    assert len(slots) == 10 and sum(1 for s in slots if s >= 0) == 8 and slots[8] == -1 and slots[9] == -1     # in order, until the slots run out
    live = [s for s in slots if s >= 0]
    assert len(set(live)) == 8
    lg = {}
    got = _drain(e, {s: 6 for s in live}, lg)
    for i, s in enumerate(slots[:8]):
        assert got[s][0] == alone[i][0], (i, lens[i])
        assert np.array_equal(lg[s][0], alone[i][2][0]), (i, "first-token logits")
        e.seq_close(s)
    rest = e.seq_open_many(prompts[8:], opts[8:])                    # the two that did not fit
    assert all(s >= 0 for s in rest)
    got = _drain(e, {s: 6 for s in rest})
    assert [got[s][0] for s in rest] == [alone[8][0], alone[9][0]]
    e.close()


def test_sequences_join_and_leave_between_steps(tiny128_gguf):
    e = _engine(tiny128_gguf)
    rng = np.random.Generator(np.random.PCG64(17))
    p = [rng.integers(0, e.info.n_vocab - 3, size=20) for _ in range(3)]
    ref = []
    for x in p:
        s = e.seq_open(x, num_predict=10, ignore_eos=True)
        ref.append(_drain(e, {s: 10})[s][0])
        e.seq_close(s)
    a = e.seq_open(p[0], num_predict=10, ignore_eos=True)
    out = {a: []}
    for _ in range(4):
        for slot, tok, _lp, _d in e.batch_step():
            out[slot].append(int(tok))
    b = e.seq_open(p[1], num_predict=10, ignore_eos=True)          # joins while a is mid-way
    out[b] = []
    for _ in range(3):
        for slot, tok, _lp, _d in e.batch_step():
            out[slot].append(int(tok))
    a_tokens = list(out[a])
    e.seq_close(a)                                                  # leaves early
    c = e.seq_open(p[2], num_predict=10, ignore_eos=True)          # reuses a's slot and pages
    out[c] = []
    dones = {}
    for _ in range(40):
        res = e.batch_step()
        if not res:
            break
        for slot, tok, _lp, d in res:
            out[slot].append(int(tok))
            dones[slot] = d
    assert a_tokens == ref[0][:7] and out[b] == ref[1] and out[c] == ref[2]
    assert dones[b] and dones[c]                                   # the 10th token carries done = 1; afterwards the step is empty
    assert e.batch_step() == []
    e.close()


def test_per_sequence_sampling_stop_tokens_and_capacity(tiny_gguf):
    from gridllm_b200 import native as N
    e = _engine(tiny_gguf, max_batch=6, max_ctx=256, kv_pool_tokens=6 * 64)
    p = np.random.Generator(np.random.PCG64(9)).integers(0, e.info.n_vocab - 3, size=16)
    ref_greedy = [int(t) for t in e.generate(p, num_predict=8, ignore_eos=True).ids]
    ref_sampled = [int(t) for t in e.generate(p, num_predict=8, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.9, seed=5).ids]
    g = e.seq_open(p, num_predict=8, ignore_eos=True)
    s = e.seq_open(p, num_predict=8, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.9, seed=5)
    s2 = e.seq_open(p, num_predict=8, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.9, seed=6)
    got = _drain(e, {g: 8, s: 8, s2: 8})
    # the greedy and the sampled sequences share every step; each follows its own options.  (The batched step computes the
    # logits with fp16 tensor-core GEMMs, gl_generate with integer dot products, so whole trajectories are compared against the
    # oracle elsewhere; here: the FIRST token -- drawn from the same prefill in both paths -- equals gl_generate's, draws are
    # reproducible, and seeds matter.)
    assert got[g][0][0] == ref_greedy[0] and got[s][0][0] == ref_sampled[0]
    assert got[s][0] != got[s2][0] or got[s][0] != got[g][0]
    for x in (g, s, s2):
        e.seq_close(x)
    s3 = e.seq_open(p, num_predict=8, ignore_eos=True, temperature=0.8, top_k=40, top_p=0.9, seed=5)
    assert _drain(e, {s3: 8})[s3][0] == got[s][0]                   # same seed, same sequence: same draw
    e.seq_close(s3)
    # a stop token ends ONE sequence (id -1, done) and leaves the other running
    stop = got[g][0][3]
    stops = {stop, int(e.info.eos_id), int(e.info.eot_id)}          # ignore_eos = False also stops at the model's own end tokens
    first = min(i for i, t in enumerate(got[g][0]) if t in stops)
    a = e.seq_open(p, num_predict=8, ignore_eos=True)
    b = e.seq_open(p, num_predict=8, ignore_eos=False, stop_ids=[stop])
    seen = {a: [], b: []}
    ended = {}
    for _ in range(12):
        for slot, tok, _lp, d in e.batch_step():
            seen[slot].append(tok)
            if d:
                ended[slot] = tok
    assert seen[a] == got[g][0] and ended[a] == got[g][0][-1]
    assert ended[b] == -1 and seen[b] == got[g][0][:first] + [-1]
    e.seq_close(a)
    e.seq_close(b)
    # the slot table / page pool is finite: running out is an error the caller can handle, and everything comes back on close
    opened = []
    with pytest.raises(N.NativeError) as ei:
        for _ in range(64):
            opened.append(e.seq_open(p, num_predict=8, ignore_eos=True))
    assert ei.value.code == -6 and 1 <= len(opened) <= 6           # GL_ERR_NOMEM
    for slot in opened:
        e.seq_close(slot)
    again = e.seq_open(p, num_predict=8, ignore_eos=True)
    assert _drain(e, {again: 8})[again][0] == got[g][0]
    with pytest.raises(N.NativeError):
        e.seq_close(5 if again != 5 else 4)                          # not open
    e.close()


def test_batching_is_off_unless_asked_for(tiny_gguf):
    from gridllm_b200 import native as N
    e = N.Engine(tiny_gguf)
    with pytest.raises(N.NativeError) as ei:
        e.seq_open([1, 2, 3], num_predict=4)
    assert ei.value.code == -4                                       # GL_ERR_UNSUPPORTED, with a message saying how to turn it on
    e.close()


def test_time_batch_step_reports_a_step(tiny128_gguf):
    e = _engine(tiny128_gguf, max_batch=32)
    ms, launches, wbytes = e.time_batch_step(24, 100, iters=4)
    assert ms > 0 and launches > 0 and wbytes > 0
    s = e.seq_open([1, 2, 3, 4, 5, 6, 7, 8, 9], num_predict=3, ignore_eos=True)    # the engine is usable afterwards
    assert len(_drain(e, {s: 3})[s][0]) == 3
    e.close()
