"""Prefill probe on the GPU box: 512-token prompt of the Llama-3-8B-shaped model through the batched prefill with the
wgmma GEMM and with the mma.sync GEMM; time and agreement of the first generated token's logits."""
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
    prompt = np.random.Generator(np.random.PCG64(1000)).integers(0, 128000, size=512)
    ref = None
    for tc5 in ("1", "0"):
        os.environ["GL_PREFILL_TC5"] = tc5
        e = N.Engine(path, max_ctx=1024)
        best = 1e9
        for _ in range(3):
            g = e.generate(prompt, num_predict=2, ignore_eos=True, want_logits=True)
            best = min(best, g.stats.prompt_eval_duration_ns / 1e6)
        lg = e.last_logits(0).copy()
        out = {"tc5": tc5, "prefill_ms": round(best, 3), "ids": g.ids[:2].tolist(), "finite": bool(np.isfinite(lg).all())}
        if ref is None:
            ref = lg
        else:
            out["max_abs_diff_vs_tc5"] = float(np.abs(lg - ref).max())
            out["max_abs_logit"] = float(np.abs(ref).max())
        print(json.dumps(out), flush=True)
        e.close()


if __name__ == "__main__":
    main()
