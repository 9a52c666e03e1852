"""Cost of the JSON grammar mask (format: "json", schema_mask.cu over the built-in any-object schema) on the Llama-3-8B-shaped synthetic model with its synthetic
vocabulary (256 byte tokens, a few dozen merges, <filler_N> pieces -- not Llama-3's, so the bytes per token differ from a real
model's):
  - decode device time per token, 512 in / 128 out, greedy vs greedy + JSON and top_k 40 vs top_k 40 + JSON, the cases
    interleaved round by round, best of the rounds (a JSON request may end early on its stop token: eval_count is printed);
  - one batched step at B = 32 (top_k 40 rows), every row JSON vs none (steps in which all 32 rows are still running);
  - the mask kernel's own device time per launch, from a torch.profiler (CUPTI) trace of JSON requests (beside the top-k
    sampler's and the mean weight GEMV's, for scale).
JSON requests are timed on prompts / seeds for which the document stays open for all 128 tokens (found by trying them).
The first line names the card and its power limit."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _open_requests(e, kw, want, tries=64):
    """(prompt, seed) pairs of 512-token prompts for which the JSON request runs all 128 tokens: the random-weight model often
    closes the document at once, and a request that stops early still runs the rest of its 32-step decode chunk"""
    found = []
    for k in range(tries):
        prompt = np.random.Generator(np.random.PCG64(1000 + k)).integers(0, 128000, size=512)
        g = e.generate(prompt, num_predict=128, format="json", **dict(kw, **({"seed": k} if kw else {})))
        if g.stats.eval_count == 128:
            found.append((prompt, k))
            if len(found) == want:
                break
    return found


SAMP = dict(temperature=0.8, top_k=40, top_p=0.9)


def _decode(e, rounds):
    cases = []
    for label, kw in (("greedy", {}), ("t0.8_k40_p0.9", SAMP)):
        got = _open_requests(e, kw, 1)
        if not got:
            print(json.dumps({"case": label + "_json", "decode_ms_per_token": None,
                              "note": "every JSON request closed its document within a few tokens on this model: not measured"}), flush=True)
            continue
        prompt, k = got[0]
        kk = dict(kw, seed=k) if kw else {}
        print(json.dumps({"case": label, "prompt_seed": 1000 + k, "sampling_seed": k if kw else None}), flush=True)
        cases += [(label, label, prompt, dict(kk, ignore_eos=True)), (label + "_json", label, prompt, dict(kk, format="json"))]
    best, last = {}, {}
    for _ in range(rounds):
        for name, _, prompt, kw in cases:
            g = e.generate(prompt, num_predict=128, **kw)
            ms = g.stats.eval_duration_ns / 1e6 / max(1, g.stats.eval_count)
            best[name] = min(best.get(name, ms), ms)
            last[name] = g
    for name, base, _, kw in cases:
        g = last[name]
        print(json.dumps({"case": name, "decode_ms_per_token": round(best[name], 4), "over_plain": round(best[name] / best[base] - 1.0, 4),
                          "eval_count": int(g.stats.eval_count), "kernel_launches": int(g.stats.kernel_launches),
                          "done_reason": int(g.stats.done_reason)}), flush=True)
    return cases[-1][2], cases[-1][3].get("seed", 0)


def _mask_kernel_time(e, prompt, seed):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            e.generate(prompt, num_predict=64, format="json", seed=seed, **SAMP)
    durs = {}
    for ev in prof.events():
        name = ev.name
        for k in ("schema_mask_kernel", "sample_topk_fast_kernel", "gemv_kernel"):
            if k in name:
                durs.setdefault(k, []).append(getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0))
    for name, d in durs.items():
        print(json.dumps({"kernel": name, "launches": len(d), "mean_us": round(float(np.mean(d)), 2), "p50_us": round(float(np.median(d)), 2)}),
              flush=True)


def _batched(path, steps):
    """B = 32 sampled rows (top_k 40), every row JSON vs none: 8 (prompt, seed) pairs that keep the document open, 4 rows each"""
    from gridllm_b200 import native as N
    e = N.Engine(path, max_ctx=1024, max_batch=32)
    pairs = _open_requests(e, SAMP, 8)
    if len(pairs) < 8:
        print(json.dumps({"batched_step_B32": None, "note": "too few open JSON requests on this model: not measured"}), flush=True)
        e.close()
        return
    prompts = [p for p, _ in pairs] * 4
    out = {}
    for rnd in range(2):
        for name, extra in (("none", dict(ignore_eos=True)), ("json", dict(format="json"))):
            opts = [dict(SAMP, seed=k, num_predict=steps + 8, **extra) for _, k in pairs] * 4
            slots = e.seq_open_many(prompts, opts)
            e.batch_step()                                   # the first tokens (drawn at open)
            ms = []
            for _ in range(steps):
                c0 = e.batch_counters()
                e.batch_step()
                c1 = e.batch_counters()
                if c1["rows"] - c0["rows"] == 32:
                    ms.append((c1["step_ns"] - c0["step_ns"]) / 1e6)
            for s_ in slots:
                e.seq_close(s_)
            if ms:
                out[name] = min(out.get(name, 1e9), float(np.median(ms)))
            print(json.dumps({"round": rnd, "rows": name, "steps_with_32_rows": len(ms)}), flush=True)
    for name in ("none", "json"):
        if name in out and "none" in out:
            print(json.dumps({"batched_step_B32_top_k40": name, "ms_per_step": round(out[name], 4),
                              "over_none": round(out[name] / out["none"] - 1.0, 4)}), flush=True)
    e.close()


def main():
    from gridllm_b200 import native as N
    path = os.environ.get("GL_PROBE_MODEL", "/dev/shm/json_llama3_8b.gguf")
    if not os.path.exists(path):
        from oracle import gguf_synth as S
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=True)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:
        card = f"nvidia-smi unavailable ({ex})"
    e = N.Engine(path, max_ctx=2048)
    print(json.dumps({"card": card, "device": e.info.device, "n_vocab": e.info.n_vocab}), flush=True)
    prompt, seed = _decode(e, int(os.environ.get("GL_PROBE_ROUNDS", "4")))
    try:
        _mask_kernel_time(e, prompt, seed)
    except Exception as ex:                              # the decode numbers above stand without it
        print(json.dumps({"mask_kernel_time": f"unavailable ({ex})"}), flush=True)
    e.close()
    _batched(path, int(os.environ.get("GL_PROBE_STEPS", "24")))


if __name__ == "__main__":
    main()
