"""GPU micro-benchmarks of the decode GEMV through the C ABI (run on an H100).
Matrices are sized > 50 MB (the H100's L2) so back-to-back launches cannot be served from L2."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gguf_synth as S  # noqa: E402


def main():
    from gridllm_b200 import native as N
    tiny = "/tmp/mb_tiny.gguf"
    S.build_model(tiny, S.TINY, "q4_k_m", seed=1)
    peak = 3350.0                    # H100 SXM data sheet (HBM3); MEASURED_PEAKS.json replaces it
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    shapes = [(S.Q4_K, 65536, 4096), (S.Q4_K, 20480, 14336), (S.Q6_K, 49152, 4096), (S.Q6_K, 12288, 14336), (S.Q8_0, 36864, 4096)]
    rng = np.random.Generator(np.random.PCG64(1))
    mats = {}
    for t, r, c in shapes:
        mats[(t, r, c)] = S.random_blocks(rng, t, r, c)
    configs = [
        {},
        {"GL_WARPS": "8"},
        {"GL_WARPS": "8", "GL_RING_DEPTH": "3"},
        {"GL_WARPS": "16"},
        {"GL_ACT_BITS": "8"},
    ]
    for cfg in configs:
        for k in ("GL_ACT_BITS", "GL_PDL", "GL_RING_DEPTH", "GL_SMEM_KB", "GL_WARPS"):
            os.environ.pop(k, None)
        os.environ.update(cfg)
        e = N.Engine(tiny)
        for (t, r, c), blocks in mats.items():
            x = np.random.Generator(np.random.PCG64(42)).standard_normal(c).astype(np.float32)
            y, ms = e.gemv(t, blocks, r, c, x, iters=20)
            nbytes = blocks.nbytes + 4 * c + 4 * r
            gbs = nbytes / (ms * 1e-3) / 1e9
            print(json.dumps({"cfg": cfg, "type": S.TYPE_NAMES[t], "rows": r, "cols": c, "ms": round(ms, 4),
                              "GBps": round(gbs, 1), "frac_of_measured_peak": round(gbs / peak, 3)}), flush=True)
        e.close()


if __name__ == "__main__":
    main()
