"""CPU: repetition / presence / frequency penalties and min_p -- the CPU restatement (tests/penalty_oracle.py) against independent
implementations (Hugging Face transformers' logits processors, the OpenAI formula, hand-computed answers), the C ABI layout of
the new gl_sample_opts fields, and the service's option mapping end to end over the oracle-backed engine double."""
import asyncio
import ctypes

import numpy as np
import pytest

import penalty_oracle as PO
from oracle import sampler as SM


def _hf_repetition(logits, window_ids, penalty):
    import torch
    from transformers import RepetitionPenaltyLogitsProcessor
    proc = RepetitionPenaltyLogitsProcessor(penalty=float(penalty))
    ids = torch.tensor(np.asarray(window_ids, dtype=np.int64)[None, :])
    return proc(ids, torch.tensor(np.asarray(logits, dtype=np.float32)[None, :]).clone())[0].numpy()


@pytest.mark.parametrize("penalty", [1.3, 0.7, 2.0])
def test_repeat_penalty_equals_transformers(penalty):
    rng = np.random.Generator(np.random.PCG64(5))
    n = 1000
    logits = (rng.standard_normal(n) * 3).astype(np.float32)
    logits[rng.integers(0, n, 20)] = 0.0                        # a <= 0 multiplies: zero stays zero either way
    hist = np.concatenate([[0, n - 1, 0, n - 1], rng.integers(0, 40, 60), [n - 1]])     # repeated ids, both ends of the vocabulary
    for last_n in (1, 8, 64, len(hist), len(hist) + 50, -1):
        got = PO.penalize(logits, hist, repeat_penalty=penalty, repeat_last_n=last_n)
        win = hist if last_n < 0 else hist[-last_n:]           # a window longer than the history is the whole history
        ref = _hf_repetition(logits, win, penalty)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), last_n
    # repeat_last_n 0: no penalty of any kind; penalty 1 or 0: off
    assert np.array_equal(PO.penalize(logits, hist, penalty, 0, 0.5, 0.5), logits)
    assert np.array_equal(PO.penalize(logits, hist, 1.0, 64), logits)
    assert np.array_equal(PO.penalize(logits, hist, 0.0, 64), logits)
    assert np.array_equal(PO.penalize(logits, [], penalty, -1), logits)


def test_presence_and_frequency_known_answers():
    logits = np.array([1.0, -2.0, 0.5, 3.0], dtype=np.float32)
    hist = [0, 0, 3, 1, 0]
    got = PO.penalize(logits, hist, repeat_penalty=1.0, repeat_last_n=-1, presence_penalty=0.25, frequency_penalty=0.5)
    # id 0: 3 times, id 1 and 3: once, id 2: never
    assert got.tolist() == [1.0 - 1.75, -2.0 - 0.75, 0.5, 3.0 - 0.75]
    # with repeat_penalty 2: divide the positive, multiply the negative, then subtract
    got = PO.penalize(logits, hist, repeat_penalty=2.0, repeat_last_n=-1, presence_penalty=0.25, frequency_penalty=0.5)
    assert got.tolist() == [0.5 - 1.75, -4.0 - 0.75, 0.5, 1.5 - 0.75]
    # window of 3: [3, 1, 0], each once
    got = PO.penalize(logits, hist, repeat_penalty=1.0, repeat_last_n=3, presence_penalty=0.0, frequency_penalty=1.0)
    assert got.tolist() == [0.0, -3.0, 0.5, 2.0]


def test_presence_and_frequency_follow_the_openai_formula():
    """OpenAI's documented form: mu[j] - c[j] * alpha_frequency - float(c[j] > 0) * alpha_presence, over the window counts."""
    rng = np.random.Generator(np.random.PCG64(11))
    n = 300
    logits = (rng.standard_normal(n) * 4).astype(np.float32)
    hist = rng.integers(0, 50, 400)
    for a_f, a_p, last_n in ((0.3, 0.0, 64), (0.0, 0.6, 100), (1.2, -0.4, -1), (-0.5, 0.7, 17)):
        got = PO.penalize(logits, hist, 1.0, last_n, a_p, a_f)
        win = hist if last_n < 0 else hist[-last_n:]
        c = np.bincount(win, minlength=n).astype(np.float64)
        ref = logits.astype(np.float64) - c * a_f - (c > 0) * a_p
        assert np.abs(got - ref).max() <= 1e-5 * max(1.0, float(np.abs(ref).max())), (a_f, a_p, last_n)


@pytest.mark.parametrize("min_p", [0.02, 0.1, 0.5])
@pytest.mark.parametrize("temperature", [0.5, 1.0, 1.7])
def test_min_p_equals_transformers_after_temperature(min_p, temperature):
    import torch
    from transformers import MinPLogitsWarper, TemperatureLogitsWarper
    rng = np.random.Generator(np.random.PCG64(3))
    logits = (rng.standard_normal(700) * 2.5).astype(np.float32)     # fewer than the 1024 candidates: min-p alone decides
    ids, _ = PO.distribution(logits, temperature, 0, 1.0, min_p)
    t = torch.tensor(logits[None, :])
    t = TemperatureLogitsWarper(temperature)(None, t)
    t = MinPLogitsWarper(min_p)(None, t)
    kept = set(np.nonzero(np.isfinite(t[0].numpy()))[0].tolist())
    assert set(ids.tolist()) == kept
    # the cut is a prefix of the candidate order, after top-p: n_keep = min(top-p keep, min-p keep)
    ids_p, _ = PO.distribution(logits, temperature, 0, 0.9, 0.0)
    ids_both, _ = PO.distribution(logits, temperature, 0, 0.9, min_p)
    assert len(ids_both) == min(len(ids_p), len(ids)) and list(ids_both) == list(ids[: len(ids_both)])
    # the draw comes from the kept prefix, inside its own interval
    for seed in range(16):
        tok, _, _ = PO.sample(logits, temperature, 0, 0.9, seed, seed, min_p=min_p)
        assert tok in set(ids_both.tolist()) and PO.interval_error(logits, tok, temperature, 0, 0.9, seed, seed, min_p=min_p) == 0.0


def test_min_p_off_changes_nothing():
    rng = np.random.Generator(np.random.PCG64(8))
    logits = (rng.standard_normal(3000) * 2).astype(np.float32)
    for k, p in ((0, 1.0), (40, 0.9), (1000, 0.5)):
        a = SM.distribution(logits, 0.8, k, p)
        b = PO.distribution(logits, 0.8, k, p, 0.0)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert SM.sample(logits, 0.8, k, p, 9, 3) == PO.sample(logits, 0.8, k, p, 9, 3, min_p=0.0)


def test_sample_opts_layout_is_unchanged():
    from gridllm_b200 import native as N
    S = N.SampleOpts
    assert ctypes.sizeof(S) == 72
    old = {"num_predict": 0, "temperature": 4, "top_k": 8, "top_p": 12, "seed": 16, "ignore_eos": 24, "n_stop_ids": 28, "stop_ids": 32,
           "want_logits": 40}
    assert {k: getattr(S, k).offset for k in old} == old
    new = {"repeat_penalty": 44, "repeat_last_n": 48, "presence_penalty": 52, "frequency_penalty": 56, "min_p": 60, "reserved": 64}
    assert {k: getattr(S, k).offset for k in new} == new
    assert "gl_penalize_logits" in N.ABI_SYMBOLS
    # a zeroed struct (what every caller that does not know the fields sends) means: no penalty, no min-p
    z = S()
    assert (z.repeat_penalty, z.repeat_last_n, z.presence_penalty, z.frequency_penalty, z.min_p) == (0.0, 0, 0.0, 0.0, 0.0)


def _service(**kw):
    from gridllm_b200 import service as SV
    return SV.NativeInferenceService({}, **kw)


def test_service_penalty_mapping():
    from gridllm_b200 import service as SV
    s = _service()
    assert s._penalties({}) == {}
    assert s._penalties({"temperature": 0.5, "top_k": 10}) == {}
    assert s._sampling({}) == {}                                                    # the sampling map is untouched
    assert s._penalties({"repeat_penalty": 1.3}) == {"repeat_penalty": 1.3, "repeat_last_n": 64}           # Ollama's window
    assert s._penalties({"repeat_penalty": 1.3, "repeat_last_n": -1}) == {"repeat_penalty": 1.3, "repeat_last_n": -1}
    assert s._penalties({"repeat_last_n": 0, "repeat_penalty": 1.2}) == {"repeat_penalty": 1.2, "repeat_last_n": 0}
    assert s._penalties({"min_p": 0.05}) == {"min_p": 0.05}
    # the OpenAI routes' names are the same keys
    assert s._penalties({"frequency_penalty": 0.5, "presence_penalty": -0.25}) == {"frequency_penalty": 0.5, "presence_penalty": -0.25,
                                                                                   "repeat_last_n": 64}
    for bad in ({"repeat_penalty": -0.1}, {"repeat_last_n": -2}, {"repeat_last_n": 3.5}, {"min_p": 1.5}, {"min_p": -0.1},
                {"presence_penalty": float("nan")}, {"frequency_penalty": float("inf")}, {"repeat_penalty": "x"}, {"min_p": True}):
        with pytest.raises(RuntimeError):
            s._penalties(bad)
    # Ollama's penalty defaults are opt-in, in their own dict
    assert SV.NativeInferenceService.OLLAMA_PENALTY_DEFAULTS == {"repeat_penalty": 1.1, "repeat_last_n": 64}
    assert "repeat_penalty" not in SV.NativeInferenceService.OLLAMA_SAMPLING_DEFAULTS
    d = _service(penalty_defaults=SV.NativeInferenceService.OLLAMA_PENALTY_DEFAULTS)
    assert d._penalties({}) == {"repeat_penalty": 1.1, "repeat_last_n": 64}
    assert d._penalties({"repeat_penalty": 1.0}) == {"repeat_penalty": 1.0, "repeat_last_n": 64}


def _penalised_greedy(m, prompt, n, **pen):
    """the oracle's own penalised greedy loop: penalise the step's logits with the history so far, take the argmax"""
    from oracle import llama_oracle as O
    orc = O.LlamaOracle(m, act="i16", kv_f16=True)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    hist, ids = [int(t) for t in prompt], []
    for _ in range(n):
        pl = PO.penalize(logits, hist, **pen)
        tok = int(np.argmax(pl))
        ids.append(tok)
        hist.append(tok)
        logits = orc.step(tok)
    return ids


def test_penalised_greedy_request_end_to_end(tiny_gguf, hostcheck_lib, monkeypatch):
    import oracle_engine
    from gridllm_b200 import service as SV

    class PenaltyDouble(oracle_engine.OracleEngine):
        """the engine double, with the penalty keywords of native.Engine.generate (greedy: the oracle's penalised argmax)"""
        def generate(self, prompt, num_predict=128, ignore_eos=False, on_token=None, want_logits=False, stop_ids=(), temperature=0.0,
                     top_k=0, top_p=1.0, seed=0, repeat_penalty=1.0, repeat_last_n=64, presence_penalty=0.0, frequency_penalty=0.0,
                     min_p=0.0):
            pen = dict(repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n, presence_penalty=presence_penalty,
                       frequency_penalty=frequency_penalty)
            self.pen_calls = getattr(self, "pen_calls", []) + [dict(pen, min_p=min_p)]
            assert temperature == 0.0 and ignore_eos
            ids = _penalised_greedy(self.m, prompt, num_predict, **pen)
            from types import SimpleNamespace
            st = SimpleNamespace(prompt_eval_count=len(prompt), eval_count=len(ids), prompt_eval_duration_ns=1, eval_duration_ns=1,
                                 total_duration_ns=2, load_duration_ns=1, done_reason=1, kernel_launches=0)
            return SimpleNamespace(ids=np.array(ids, dtype=np.int32), logprobs=np.zeros(len(ids), np.float32), stats=st)

    oracle_engine.use_hostcheck(hostcheck_lib)
    monkeypatch.setattr(SV.N, "Engine", PenaltyDouble)
    monkeypatch.setattr(SV.N, "device_count", lambda: 1)
    svc = SV.NativeInferenceService({"tiny:latest": tiny_gguf}, device=0)
    try:
        req = {"id": "p1", "model": "tiny:latest", "prompt": "the rain in spain falls mainly", "priority": "medium",
               "options": {"num_predict": 10, "temperature": 0, "ignore_eos": True, "repeat_penalty": 1.3}}
        res = asyncio.new_event_loop().run_until_complete(svc.generateResponse(req))
        eng = svc._engine("tiny:latest")
        assert eng.pen_calls[-1] == {"repeat_penalty": 1.3, "repeat_last_n": 64, "presence_penalty": 0.0, "frequency_penalty": 0.0,
                                     "min_p": 0.0}
        prompt = eng.tokenize(req["prompt"])
        assert res["token_ids"] == _penalised_greedy(eng.m, prompt, 10, repeat_penalty=1.3, repeat_last_n=64)
        # a presence penalty far larger than the logits' spread over the whole history: no id of the history comes back
        req2 = dict(req, id="p2", options={"num_predict": 10, "temperature": 0, "ignore_eos": True, "presence_penalty": 1e4,
                                           "repeat_last_n": -1})
        res2 = asyncio.new_event_loop().run_until_complete(svc.generateResponse(req2))
        ids = res2["token_ids"]
        assert len(set(ids)) == len(ids) and not set(ids) & set(int(t) for t in prompt)
        # a bad value fails the request, as a bad temperature does
        with pytest.raises(RuntimeError):
            asyncio.new_event_loop().run_until_complete(svc.generateResponse(dict(req, id="p3", options={"repeat_penalty": -1})))
    finally:
        svc.close()
