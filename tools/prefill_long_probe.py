"""Prompt passes longer than one 4 096-row pass, and prefix reuse, on the Llama-3-8B-shaped synthetic q4_K_M model (random
weights, synthetic vocabulary), one engine at a time:
  - prompt-pass device time (prompt_eval_duration) of gl_generate for 4 096, 8 192 and 16 384 prompt tokens, best of three;
  - 8 192 tokens once on a prefill_mode=1 engine (every prompt token a decode step: what such a prompt cost before it could
    take the tensor-core pass), and the worst |delta first-token logit| / max|logit| between the two paths;
  - a two-turn conversation: a 4 096-token first turn with 128 tokens out, then its context plus 256 new tokens; the second
    turn's prompt-pass time without reuse (record cleared) and with prefix_cache, interleaved, best of three;
  - the device time per launch of the PAGED prompt attention (the second 4 096-row pass of the 8 192-token prompt) beside the
    first pass's attention, from a torch.profiler (CUPTI) trace of a separate run.
The engine context is 16 384 + 128 tokens (a 16 384-token prompt plus its first output).  The first line names the card, its
power limit and its maximum SM clock."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAX_CTX = 16384 + 128


def _prompt(n, seed):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, 128000, size=n)


def _pass_times(e):
    for n in (4096, 8192, 16384):
        p = _prompt(n, n)
        ms = []
        for _ in range(3):
            e.kv_reset()                                      # a cold pass each time (the engine has prefix_cache on)
            g = e.generate(p, num_predict=1, ignore_eos=True)
            assert g.stats.prompt_eval_count == n
            ms.append(g.stats.prompt_eval_duration_ns / 1e6)
        print(json.dumps({"prompt_tokens": n, "prompt_pass_ms_best_of_3": round(min(ms), 2), "all_ms": [round(x, 2) for x in ms]}), flush=True)


def _two_turns(e):
    p1 = _prompt(4096, 77)
    new = [int(t) for t in _prompt(256, 78)]
    best = {}
    for rnd in range(3):
        for case in ("off", "on"):
            e.kv_reset()
            g1 = e.generate(p1, num_predict=128, ignore_eos=True)
            p2 = [int(t) for t in p1] + [int(t) for t in g1.ids] + new
            if case == "off":
                e.kv_reset()                                  # no record: the whole conversation again, as without prefix_cache
            g2 = e.generate(p2, num_predict=1, ignore_eos=True)
            ms = g2.stats.prompt_eval_duration_ns / 1e6
            best[case] = min(best.get(case, ms), ms)
            print(json.dumps({"round": rnd, "prefix_cache": case, "turn2_prompt_tokens": len(p2),
                              "turn2_prompt_eval_count": int(g2.stats.prompt_eval_count), "turn2_prompt_pass_ms": round(ms, 2)}), flush=True)
    print(json.dumps({"turn2_prompt_pass_ms_best_of_3": {k: round(v, 2) for k, v in best.items()}}), flush=True)


def _attention_kernel_times(e):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    p = _prompt(8192, 8192)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.generate(p, num_predict=1, ignore_eos=True)
    durs = {}
    for ev in prof.events():
        if "flash_prefill_kernel" in ev.name:
            key = "paged" if ("true>" in ev.name or "Lb1E" in ev.name) else "scratch"      # demangled or mangled <HD, PAGED>

            durs.setdefault(key, []).append(getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0))
    for k, d in durs.items():
        print(json.dumps({"prompt_attention": k, "launches": len(d), "mean_us": round(float(np.mean(d)), 1),
                          "p50_us": round(float(np.median(d)), 1)}), flush=True)


def main():
    from gridllm_b200 import native as N
    path = os.environ.get("GL_PROBE_MODEL", "/dev/shm/prefill_llama3_8b.gguf")
    if not os.path.exists(path):
        from oracle import gguf_synth as S
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=True)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:
        card = f"nvidia-smi unavailable ({ex})"
    print(json.dumps({"card": card}), flush=True)

    e = N.Engine(path, max_ctx=MAX_CTX, prefix_cache=True)
    _pass_times(e)
    p8 = _prompt(8192, 8192)
    e.kv_reset()
    g = e.generate(p8, num_predict=1, ignore_eos=True, want_logits=True)
    l_tc = e.last_logits(0)
    t_tc = g.stats.prompt_eval_duration_ns / 1e6
    _two_turns(e)
    e.close()

    es = N.Engine(path, max_ctx=MAX_CTX, prefill_mode=1)
    g = es.generate(p8, num_predict=1, ignore_eos=True, want_logits=True)
    l_seq = es.last_logits(0)
    es.close()
    print(json.dumps({"prompt_tokens": 8192, "sequential_prompt_ms": round(g.stats.prompt_eval_duration_ns / 1e6, 1),
                      "tensor_core_prompt_ms": round(t_tc, 2),
                      "first_token_max_abs_dlogit_over_max_logit": float(np.abs(l_tc - l_seq).max() / np.abs(l_seq).max())}), flush=True)

    e = N.Engine(path, max_ctx=MAX_CTX)
    try:
        _attention_kernel_times(e)
    except Exception as ex:                                   # the numbers above stand without it
        print(json.dumps({"attention_kernel_time": f"unavailable ({ex})"}), flush=True)
    e.close()


if __name__ == "__main__":
    main()
