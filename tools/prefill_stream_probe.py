"""The streamed prompt pass (GL_PREFILL_WEIGHTS=2, gridllm_b200/csrc/prefill_weights.h) against the resident 16-bit copy, and a
full 80-layer Llama-3-70B-shaped q4_K_M model on one card:
  - Llama-3-8B q4_K_M synthetic: prompt-pass device time (prompt_eval_duration) of gl_generate at 512 / 2 048 / 4 096 tokens,
    resident vs streamed engines alternating, best of 3; and, from a torch.profiler (CUPTI) trace of one streamed 4 096-token
    pass, the dequant kernel's device time per operand and its read + write bytes/s (bytes from the tensor shapes and types);
  - 70B-shaped random q4_K_M, 80 layers (about 42.5 GB, built in a temporary directory when shutil.disk_usage shows room, deleted
    at exit): load time, the launches of one prompt pass (from one packed gl_embed pass: 1 + 11 launches per layer streamed, 1 + 7 resident), prompt
    pass at 512 / 2 048 / 4 096 tokens (best of 3), decode ms per token at context 600 with its weight bytes/s, and a 256-token
    prompt streamed vs a prefill_mode=1 engine (every prompt token a decode step).
The first line names the card, its power limit and its maximum SM clock."""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPS = ("qkv", "attn_output", "gate_up", "ffn_down")
BLOCK_BYTES = {12: 144, 14: 210, 8: 272}       # bytes per 256 columns: Q4_K, Q6_K, Q8_0


def _print(**kw):
    print(json.dumps(kw), flush=True)


def _prompt(n, seed):
    return np.random.Generator(np.random.PCG64(seed)).integers(0, 128000, size=n)


def _engine(path, weights, **kw):
    from gridllm_b200 import native as N
    os.environ["GL_PREFILL_WEIGHTS"] = str(weights)
    try:
        return N.Engine(path, **kw)
    finally:
        del os.environ["GL_PREFILL_WEIGHTS"]


def _pass_ms(e, n, seed):
    e.kv_reset()
    g = e.generate(_prompt(n, seed), num_predict=1, ignore_eos=True)
    assert g.stats.prompt_eval_count == n
    return g.stats.prompt_eval_duration_ns / 1e6, int(g.stats.kernel_launches)


def _operand_bytes(shape, recipe):
    """per layer and operand: (bytes read from the engine layout, bytes written as fp16), averaged over the layers"""
    from oracle import gguf_synth as S
    rd = {op: 0 for op in OPS}
    wr = {op: 0 for op in OPS}
    kind_op = {"attn_q": "qkv", "attn_k": "qkv", "attn_v": "qkv", "attn_output": "attn_output", "ffn_gate": "gate_up", "ffn_up": "gate_up",
               "ffn_down": "ffn_down"}
    for name, t, (rows, cols) in S.tensor_plan(shape, recipe):
        kind = name.split(".")[2] if name.startswith("blk.") else None
        if kind not in kind_op:
            continue
        rd[kind_op[kind]] += rows * cols // 256 * BLOCK_BYTES[t]
        wr[kind_op[kind]] += rows * cols * 2
    return {op: (rd[op] / shape.n_layer, wr[op] / shape.n_layer) for op in OPS}


def _dequant_kernel_times(e, shape):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    e.kv_reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.generate(_prompt(4096, 4096), num_predict=1, ignore_eos=True)
    evs = sorted((ev for ev in prof.events() if "dequant_operand_kernel" in ev.name), key=lambda ev: ev.time_range.start)
    assert len(evs) == 4 * shape.n_layer, len(evs)
    nbytes = _operand_bytes(shape, "q4_k_m")
    total_us = 0.0
    for i, op in enumerate(OPS):
        us = [getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0) for ev in evs[i::4]]
        rd, wr = nbytes[op]
        mean = float(np.mean(us))
        total_us += float(np.sum(us))
        _print(dequant_operand=op, launches=len(us), mean_us=round(mean, 1), read_MB=round(rd / 1e6, 1), write_MB=round(wr / 1e6, 1),
               read_plus_write_TB_per_s=round((rd + wr) / (mean * 1e-6) / 1e12, 3))
    _print(dequant_ms_per_pass=round(total_us / 1e3, 2))


def _probe_8b():
    import bench
    from oracle import gguf_synth as S
    path = bench.build_model_once("llama3_8b_q4km", 0, lambda: None)
    res = _engine(path, 1, max_ctx=4096 + 16)
    st = _engine(path, 2, max_ctx=4096 + 16)
    launches = {}
    for n in (512, 2048, 4096):
        best = {}
        for _ in range(3):
            for name, e in (("resident", res), ("streamed", st)):
                ms, kl = _pass_ms(e, n, n)
                best[name] = min(best.get(name, ms), ms)
                launches[name] = kl
        _print(model="llama3-8b q4_K_M", prompt_tokens=n, resident_ms_best_of_3=round(best["resident"], 2),
               streamed_ms_best_of_3=round(best["streamed"], 2), streamed_over_resident=round(best["streamed"] / best["resident"], 3))
    _print(model="llama3-8b q4_K_M", generate_launches=launches, n_layer=res.info.n_layer)
    res.close()
    try:
        _dequant_kernel_times(st, S.LLAMA3_8B)
    except Exception as ex:                                   # the numbers above stand without it
        _print(dequant_kernel_time=f"unavailable ({ex})")
    st.close()


def _source(e):
    """which weights the prompt pass read: one packed gl_embed pass launches 1 + 7 kernels per layer on the resident copy, 1 + 11
    streamed, then 3 for the pooling"""
    _, st = e.embed([_prompt(512, 5)])
    n = int(st.kernel_launches) - 3
    L = e.info.n_layer
    return {1 + 7 * L: "resident", 1 + 11 * L: "streamed"}.get(n, f"unknown ({n} launches)")


def _probe_70b():
    from gridllm_b200 import native as N
    from oracle import gguf_synth as S
    tmp = tempfile.gettempdir()
    free = shutil.disk_usage(tmp).free
    if free < 50e9:
        _print(model="llama3-70b-shape q4_K_M", skipped=f"{free / 1e9:.1f} GB free under {tmp}, 50 GB needed")
        return
    mem = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if mem < 60e9:                                            # gguf_synth holds every tensor in memory until it writes the file
        _print(model="llama3-70b-shape q4_K_M", skipped=f"{mem / 1e9:.1f} GB of host memory available, 60 GB needed")
        return
    shape = S.LlamaShape("llama3-70b-synth", 80, 8192, 64, 8, 28672, 128256, 500000.0, 1e-5, 8192)
    d = tempfile.mkdtemp(dir=tmp)
    path = os.path.join(d, "llama3_70b_q4km_synth.gguf")
    try:
        t0 = time.time()
        info = S.build_model(path, shape, "q4_k_m", seed=1234, mode="random", with_vocab=False,
                             rope_freqs=S.llama3_rope_factors(128, 500000.0))
        _print(model="llama3-70b-shape q4_K_M", file_GB=round(info["bytes"] / 1e9, 2), build_s=round(time.time() - t0, 1))
        t0 = time.time()
        e = N.Engine(path)                                    # auto: the copy (136.9 GB) cannot fit
        _print(load_s=round(time.time() - t0, 1), n_ctx=int(e.info.n_ctx), prompt_pass_source=_source(e))
        best = {}
        for n in (512, 2048, 4096):
            for _ in range(3):
                ms, _ = _pass_ms(e, n, n)
                best[n] = min(best.get(n, ms), ms)
            _print(prompt_tokens=n, prompt_pass_ms_best_of_3=round(best[n], 2))
        e.kv_reset()
        ms, _ = e.time_decode(600, iters=32)
        wb = int(e.info.decode_bytes_per_token)
        _print(decode_ctx=600, decode_ms_per_token=round(ms, 3), decode_weight_GB=round(wb / 1e9, 2),
               decode_weight_TB_per_s=round(wb / (ms * 1e-3) / 1e12, 3))
        t256, _ = _pass_ms(e, 256, 256)
        e.close()
        es = N.Engine(path, prefill_mode=1)
        es.kv_reset()
        g = es.generate(_prompt(256, 256), num_predict=1, ignore_eos=True)
        es.close()
        _print(prompt_tokens=256, streamed_ms=round(t256, 2), prefill_mode_1_ms=round(g.stats.prompt_eval_duration_ns / 1e6, 1))
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:
        card = f"nvidia-smi unavailable ({ex})"
    _print(card=card)
    if "--only-70b" not in sys.argv:
        _probe_8b()
    if "--skip-70b" not in sys.argv:
        _probe_70b()


if __name__ == "__main__":
    main()
