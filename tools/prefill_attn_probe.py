"""Prompt-pass probe on the GPU box: the Llama-3-8B-shaped model's batched prefill under a list of switch settings
(PROBE_VARIANTS="GL_PREFILL_FLASH=1;GL_PREFILL_FLASH=0" by default: the fused attention kernel of prefill_attn.cu against the
three-launch path), at the prompt lengths given on the
command line: device time of the prompt pass and agreement of the first generated token's logits with the first variant's."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gguf_synth as S  # noqa: E402


def main():
    from gridllm_b200 import native as N
    path = "/dev/shm/prof_llama3_8b.gguf"
    if not os.path.exists(path):
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=False)
    lens = [int(a) for a in sys.argv[1:]] or [512, 2048]
    for T in lens:
        prompt = np.random.Generator(np.random.PCG64(1000 + T)).integers(0, 128000, size=T)
        ref = None
        for var in os.environ.get("PROBE_VARIANTS", "GL_PREFILL_FLASH=1;GL_PREFILL_FLASH=0").split(";"):
            for kv in var.split(","):
                k, v = kv.split("=")
                os.environ[k] = v
            e = N.Engine(path, max_ctx=T + 16)
            best = 1e9
            for _ in range(3):
                g = e.generate(prompt, num_predict=2, ignore_eos=True, want_logits=True)
                best = min(best, g.stats.prompt_eval_duration_ns / 1e6)
            lg = e.last_logits(0).copy()
            out = {"tokens": T, "variant": var, "prefill_ms": round(best, 3), "launches": int(g.stats.kernel_launches), "ids": g.ids[:2].tolist(),
                   "finite": bool(np.isfinite(lg).all())}
            if ref is None:
                ref = lg
            else:
                out["max_abs_diff_vs_first"] = float(np.abs(lg - ref).max())
                out["max_abs_logit"] = float(np.abs(ref).max())
            print(json.dumps(out), flush=True)
            e.close()


if __name__ == "__main__":
    main()
