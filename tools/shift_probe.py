"""Measurement driver: the context shift (gl_engine_opts context_shift) on the bench model (synthetic Llama-3-8B q4_K_M).
  * kv_shift alone at the Llama-3-8B KV shape (32 layers, 8 KV heads, head_dim 128), W = 8192, k = 4: device time per launch
    (CUDA events, through the launcher shim tests/shiftcheck) and the bytes it must move -- each moved row is read and written
    once, K and V -- over that time, against the H100 SXM data-sheet 3.35 TB/s;
  * per-token decode time (gl_gen_stats eval_duration / eval_count) of a greedy generation that crosses a 2 048 window once,
    against the same request on an engine with a 4 096 window (no crossing);
  * a batched step in which all 32 rows shift (every row at position W = 2 048), against the steps around it.
The card's name and power limit are printed with the numbers.  usage: shift_probe.py  -- one JSON line per measurement."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_TBPS = 3.35


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kv_shift_alone():
    from gridllm_b200 import native
    native.load_library()
    lib = ctypes.CDLL(os.path.join(ROOT, "tests", "shiftcheck", "libshiftcheck.so"))
    out = []
    for n_seq, W in ((1, 8192), (32, 2048)):
        n_layer, n_kv, hd, keep = 32, 8, 128, 4
        ms = ctypes.c_float(0)
        rc = lib.sc_time_kv_shift(n_layer, n_kv, hd, W, keep, n_seq, 20, ctypes.byref(ms))
        if rc != 0:
            raise RuntimeError(f"sc_time_kv_shift: cudaError {rc}")
        d = (W - keep + 1) // 2
        rows = W - keep - d
        nbytes = n_seq * rows * n_layer * n_kv * hd * 2 * 2 * 2      # fp16, K and V, read and written
        out.append({"what": "kv_shift", "n_seq": n_seq, "W": W, "keep": keep, "discard": d, "rows": rows, "ms": round(ms.value, 4),
                    "bytes": nbytes, "TB_per_s": round(nbytes / (ms.value * 1e-3) / 1e12, 3),
                    "of_hbm_peak": round(nbytes / (ms.value * 1e-3) / 1e12 / HBM_TBPS, 3)})
    return out


def decode_crossing(path):
    from gridllm_b200 import native as N
    rng = np.random.Generator(np.random.PCG64(3))
    out = []
    for W, tag in ((2048, "crosses the window once"), (4096, "no crossing")):
        e = N.Engine(path, max_ctx=W, context_shift=True)
        prompt = rng.integers(0, e.info.n_vocab - 3, size=2000)
        e.generate(prompt[:64], num_predict=64, ignore_eos=True)                # warm-up
        per = []
        for _ in range(3):
            g = e.generate(prompt, num_predict=128, ignore_eos=True, num_keep=4)
            per.append(g.stats.eval_duration_ns / g.stats.eval_count / 1e6)
        out.append({"what": "decode", "W": W, "case": tag, "n_prompt": 2000, "num_predict": 128, "ms_per_token": [round(x, 4) for x in per]})
        e.close()
    return out


def batch_all_shift(path):
    from gridllm_b200 import native as N
    W, B = 2048, 32
    e = N.Engine(path, max_ctx=W, max_batch=B, batch_weights=2, context_shift=True)
    rng = np.random.Generator(np.random.PCG64(5))
    lead = 8
    prompts = [rng.integers(0, e.info.n_vocab - 3, size=W - lead) for _ in range(B)]
    slots = e.seq_open_many(prompts, [dict(num_predict=2 * lead, ignore_eos=True, num_keep=4)] * B)
    assert min(slots) >= 0
    times = []
    for _ in range(2 * lead - 1):
        before = e.batch_counters()["step_ns"]
        e.batch_step()
        times.append((e.batch_counters()["step_ns"] - before) / 1e6)
    e.close()
    return [{"what": "batch_step", "B": B, "W": W, "step_ms": [round(t, 4) for t in times],
             "note": f"entry 0 is the opens' first tokens (no device step); entry {lead + 1} is the step in which every row shifts"}]


def main():
    import bench
    path = bench.build_model_once("llama3_8b_q4km", 0, lambda: None)
    info = {"card": card()}
    for rec in kv_shift_alone() + decode_crossing(path) + batch_all_shift(path):
        rec.update(info)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
