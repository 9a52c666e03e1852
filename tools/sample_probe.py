"""Cost of the seeded top-k / top-p sampler and of the repetition penalty inside a request: 512-in / 128-out on the
Llama-3-8B-shaped synthetic model, greedy against temperature 0.8 / top_k 40 / top_p 0.9 (and top_k off = 1024 candidates),
and greedy against greedy with repeat_penalty 1.1 over the last 64 ids / the whole history.  Device time of the decode part;
the cases are interleaved round by round and the best of the rounds is reported.  The first line names the card."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from gridllm_b200 import native as N
    path = os.environ.get("GL_PROBE_MODEL", "/dev/shm/prof_llama3_8b.gguf")      # e.g. the synthetic model bench.py built
    if not os.path.exists(path):
        from oracle import gguf_synth as S
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=False)
    pdl = os.environ.get("GL_PDL", "1")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                              # the numbers below still stand; the card is then named by the runtime only
        card = f"nvidia-smi unavailable ({ex})"
    e = N.Engine(path, max_ctx=2048)
    print(json.dumps({"card": card, "device": e.info.device}), flush=True)
    prompt = np.random.Generator(np.random.PCG64(1000)).integers(0, 128000, size=512)
    cases = (("greedy", {}), ("t0.8_k40_p0.9", dict(temperature=0.8, top_k=40, top_p=0.9, seed=1)),
             ("t0.8_k1024", dict(temperature=0.8, top_k=0, top_p=1.0, seed=1)),
             ("greedy_rp1.1_last64", dict(repeat_penalty=1.1, repeat_last_n=64)),
             ("greedy_rp1.1_all", dict(repeat_penalty=1.1, repeat_last_n=-1)))
    best, last = {}, {}
    for _ in range(int(os.environ.get("GL_PROBE_ROUNDS", "5"))):
        for name, kw in cases:
            g = e.generate(prompt, num_predict=128, ignore_eos=True, **kw)
            ms = g.stats.eval_duration_ns / 1e6 / g.stats.eval_count
            best[name] = min(best.get(name, ms), ms)
            last[name] = g
    for name, _ in cases:
        g = last[name]
        print(json.dumps({"pdl": pdl, "sampler": name, "decode_ms_per_token": round(best[name], 4),
                          "over_greedy": round(best[name] / best["greedy"] - 1.0, 4), "kernel_launches": int(g.stats.kernel_launches),
                          "distinct_tokens": int(len(set(g.ids.tolist())))}), flush=True)
    e.close()


if __name__ == "__main__":
    main()
