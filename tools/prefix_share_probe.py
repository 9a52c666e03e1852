"""Measurement driver: prompt-prefix page sharing between batch slots (gl_engine_opts batch_prefix_cache) on the bench model,
with the option off and on in interleaved rounds (a fresh engine per case and round).
  * 32 chat requests with one shared 1 024-token preamble and distinct 64-token suffixes, opened in ONE gl_seq_open_many:
    prompt-pass device time, prompt tokens evaluated / taken from shared pages, and the KV pages the 32 slots hold after the
    open (from the reservation rule of include/gridllm_native.h: shared pages once, then each slot's own);
  * the batched step at B = 32 over those rows (device time per step, 32 steps);
  * a three-turn conversation (turn t's prompt = turn t-1's prompt + its 48-token reply + 64 new tokens) through gl_seq_open:
    host wall time of each open, which ends with the first token drawn (time to first token), and the tokens it evaluated.
The bench model carries no vocabulary, so the conversation is token ids, not the chat endpoints.
usage: prefix_share_probe.py [rounds]   -- one JSON line per case and round."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_SEQ, PRE, SUF, N_PRED, PAGE = 32, 1024, 64, 64, 16


def pages_held(prompts, shared_pos):
    """pages the slots hold: each slot's own pages, plus every shared page once (the first slot owns the preamble's)"""
    return sum((len(p) + N_PRED + PAGE - 1) // PAGE - r // PAGE for p, r in zip(prompts, shared_pos))


def one_round(path, on, rnd):
    from gridllm_b200 import native as N
    e = N.Engine(path, max_ctx=2048, max_batch=N_SEQ, batch_weights=2, batch_prefix_cache=on)
    rng = np.random.Generator(np.random.PCG64(11))
    pre = rng.integers(0, e.info.n_vocab - 3, size=PRE)
    prompts = [np.concatenate([pre, rng.integers(0, e.info.n_vocab - 3, size=SUF)]) for _ in range(N_SEQ)]
    opts = [dict(num_predict=N_PRED, ignore_eos=True)] * N_SEQ
    # warm-up: a burst of unrelated prompts (captures the packed-pass and step variants); closed before the measured open
    warm = e.seq_open_many([rng.integers(0, e.info.n_vocab - 3, size=PRE + SUF) for _ in range(4)], opts[:4])
    for _ in range(3):
        e.batch_step()
    for s in warm:
        e.seq_close(s)
    e.batch_counters(reset=True)
    slots = e.seq_open_many(prompts, opts)
    assert all(s >= 0 for s in slots)
    c = e.batch_counters(reset=True)
    evals = [e.seq_stats(s).prompt_eval_count for s in slots]
    e.batch_step()                                   # the first tokens, drawn at the open
    for _ in range(4):
        e.batch_step()
    e.batch_counters(reset=True)
    for _ in range(32):
        e.batch_step()
    cs = e.batch_counters(reset=True)
    for s in slots:
        e.seq_close(s)
    print(json.dumps({"round": rnd, "batch_prefix_cache": on, "case": "open32", "prefill_ms": c["prefill_ns"] / 1e6,
                      "prompt_tokens_evaluated": c["prefill_tokens"], "prompt_tokens_shared": c["shared_tokens"],
                      "pages_held": pages_held(prompts, [len(p) - n for p, n in zip(prompts, evals)]),
                      "step_ms_b32": cs["step_ns"] / 1e6 / max(1, cs["steps"])}), flush=True)
    # three turns of one conversation
    conv = rng.integers(0, e.info.n_vocab - 3, size=PRE + SUF)
    for turn in range(3):
        t0 = time.perf_counter()
        s = e.seq_open(conv, num_predict=48, ignore_eos=True)
        ttft = time.perf_counter() - t0
        ev = e.seq_stats(s).prompt_eval_count
        reply = []
        while len(reply) < 48:
            reply += [t for sl, t, _, _ in e.batch_step() if sl == s]
        e.seq_close(s)
        print(json.dumps({"round": rnd, "batch_prefix_cache": on, "case": "chat", "turn": turn + 1, "prompt_tokens": len(conv),
                          "evaluated": ev, "ttft_ms": ttft * 1e3}), flush=True)
        conv = np.concatenate([conv, np.asarray(reply[:48]), rng.integers(0, e.info.n_vocab - 3, size=64)])
    e.close()


def main():
    import bench
    path = bench.build_model_once("llama3_8b_q4km", 0, lambda: None)
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    for rnd in range(rounds):
        for on in (False, True):
            one_round(path, on, rnd)


if __name__ == "__main__":
    main()
