"""Batch-1 decode A/B on the GPU box: ms per token of the Llama-3-8B-shaped q4_K_M model at ctx 1 / 576 / 2000 under a list of
switch settings (DECODE_VARIANTS="GL_NONE=1;GL_ATTN_CLUSTER=1,GL_ATTN_SPLITS=8;..."), CUDA events around graph replays
(gl_time_decode).  The roofline fraction is algorithmic weight bytes / time / the measured HBM peak."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gguf_synth as S  # noqa: E402


def main():
    from gridllm_b200 import native as N
    path = "/dev/shm/prof_llama3_8b.gguf"
    if not os.path.exists(path):
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=False)
    peak = 3350.0                    # H100 SXM data sheet (HBM3); MEASURED_PEAKS.json replaces it
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    touched = set()
    for var in os.environ.get("DECODE_VARIANTS", "GL_NONE=1").split(";"):
        for k in touched:
            os.environ.pop(k, None)
        for kv in var.split(","):
            k, v = kv.split("=")
            os.environ[k] = v
            touched.add(k)
        os.environ["GL_PREFILL"] = "1"          # no 16-bit copy: the probe only times decode steps
        e = N.Engine(path, max_ctx=2048 + 64)
        bpt = e.info.decode_bytes_per_token
        for ctx in (1, 576, 1900):
            best = 1e9
            for _ in range(3):
                ms, nl = e.time_decode(ctx, 48)
                best = min(best, ms)
            print(json.dumps({"variant": var, "ctx": ctx, "ms_per_token": round(best, 4), "launches": nl,
                              "hbm_frac_weights_only": round(bpt / best / 1e6 / peak, 4)}), flush=True)
        e.close()


if __name__ == "__main__":
    main()
