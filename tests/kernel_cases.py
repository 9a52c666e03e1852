"""Inputs of the kernel-level GPU checks (tests/test_gpu_kernels.py), shared with tests/test_kernel_ref_cpu.py so that the
mutant checks run on exactly the inputs the GPU tests use.  Everything is generated from a seed."""
import numpy as np

import kernel_ref as R

F32, ADD, T16, SILU = R.GEMM_EPI_F32, R.GEMM_EPI_ADD_F32, R.GEMM_EPI_T16, R.GEMM_EPI_SILU

# (m, n, k, epilogue, ldc kind): "vec" takes the 16-byte stores of gemm_tc5's epilogue, "scalar" the element path
GEMM_CASES = [
    (1, 32, 64, F32, "vec"),
    (7, 96, 200, T16, "vec"),
    (7, 96, 200, T16, "scalar"),
    (128, 200, 4096, F32, "scalar"),
    (129, 1000, 200, ADD, "vec"),
    (300, 4096, 64, T16, "vec"),
    (2048, 4096, 4096, F32, "vec"),          # 512 output tiles: the persistent loop and the TMA ring cross tiles
    (2048, 1000, 200, T16, "scalar"),        # 128 tiles
    (300, 96, 14336, ADD, "scalar"),
    (7, 4096, 14336, T16, "scalar"),
    (129, 32, 4096, SILU, "vec"),
    (300, 4096, 200, SILU, "vec"),
    (1, 96, 14336, SILU, "vec"),
]


def gemm_case_id(c):
    m, n, k, epi, kind = c
    return f"{m}x{n}x{k}-{['f32', 'add', 't16', 'silu'][epi]}-{kind}"


def ldc_of(n, epi, kind):
    w = n // 2 if epi == SILU else n
    if kind == "vec":
        return (w + 7) // 8 * 8 + 8
    return w + 1 if epi != SILU else w + 8


def operand(rng, rows, k, bf16, scale=1.0):
    """(16-bit bits as stored, float64 values) of a [rows, k] operand ~ N(0, scale^2)"""
    x = (rng.standard_normal((rows, k), dtype=np.float32) * np.float32(scale))
    if bf16:
        bits = R.to_bf16_bits(x)
        return bits, R.bf16_bits_to_f64(bits)
    h = x.astype(np.float16)
    return h.view(np.uint16), h.astype(np.float64)


def gemm_inputs(case, bf16, seed=0):
    m, n, k, epi, _kind = case
    rng = np.random.Generator(np.random.PCG64(hash((m, n, k, epi, bf16, seed)) & 0xFFFFFFFF))
    a_bits, a = operand(rng, m, k, bf16)
    b_bits, b = operand(rng, n, k, bf16, 1.0 / np.sqrt(k))
    old = rng.standard_normal((m, n)) if epi == ADD else None
    if old is not None:
        old = old.astype(np.float32).astype(np.float64)
    return a_bits, a, b_bits, b, old


# ---- RoPE / split ---------------------------------------------------------------------------------------------------
ROPE_HEADS = (4, 2)          # n_head, n_kv
ROPE_M = 640                 # rows of the pack: [512, 640) belong to no segment


def rope_segs(pos0):
    """(start, len, pos0) of a pack of three segments (the second and third continue sequences at other positions)"""
    return [(0, 100, pos0), (128, 129, pos0 + 3), (384, 1, 7)]


def rope_tables(hd, n_pos):
    from oracle import llama_oracle as O
    return O.rope_table(n_pos, hd, 500000.0)


def page_tables(rng, segs, n_pages):
    """shuffled physical pages for every segment (pages of the pool are handed out without repetition)"""
    perm = rng.permutation(n_pages)
    tabs, used = [], 0
    for _s0, ln, p0 in segs:
        need = (p0 + ln + 15) // 16
        tabs.append(perm[used:used + need].astype(np.int32))
        used += need
    assert used <= n_pages
    return tabs


# ---- prompt attention ------------------------------------------------------------------------------------------------
ATTN_HEADS = [(4, 4), (8, 2), (8, 1), (32, 8)]
ATTN_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 300, 1000]
PAGED_POS0 = [1, 15, 16, 17, 63, 64, 100, 128, 4096]
PAGED_LENS = [1, 7, 64, 129, 300]


def qkv_values(rng, kv_len, n_q, n_head, n_kv, hd, peaked):
    """fp16 q [n_q, n_head hd] and k / v [kv_len, n_kv hd].  peaked: logit standard deviation ~6 and key norms growing along
    the sequence, so the running maximum of the online softmax keeps moving (the rescale path runs)"""
    if peaked:
        q = rng.standard_normal((n_q, n_head * hd)) * (6.0 / hd ** 0.25)
        growth = 0.5 + 1.5 * np.arange(kv_len)[:, None] / max(kv_len, 1)
        k = rng.standard_normal((kv_len, n_kv * hd)) * (1.0 / hd ** 0.25) * growth
    else:
        q = rng.standard_normal((n_q, n_head * hd))
        k = rng.standard_normal((kv_len, n_kv * hd))
    v = rng.standard_normal((kv_len, n_kv * hd))
    return q.astype(np.float16), k.astype(np.float16), v.astype(np.float16)


# ---- qgemm -------------------------------------------------------------------------------------------------------------
Q4, Q6 = R.Q4_K, R.Q6_K
# name -> ([(rows, type)], mode, k, epilogue, weights from "random" blocks or "quant"ised normals)
QG_SHAPES = {
    "nkb1": ([(1024, Q4)], 0, 256, F32, "quant"),
    "nkb3": ([(512, Q6)], 0, 768, ADD, "quant"),
    "nkb5": ([(384, Q4)], 0, 1280, F32, "quant"),
    "three_src": ([(128, Q4), (256, Q6), (128, Q4)], 0, 1024, ADD, "quant"),
    "silu_small": ([(256, Q4), (256, Q4)], 1, 1024, SILU, "quant"),
    "qkv_8b": ([(4096, Q4), (1024, Q4), (1024, Q6)], 0, 4096, F32, "random"),
    "o_8b": ([(4096, Q4)], 0, 4096, ADD, "random"),
    "gate_up_8b": ([(14336, Q4), (14336, Q4)], 1, 4096, SILU, "random"),
    "down_8b": ([(4096, Q6)], 0, 14336, ADD, "random"),
    "lm_head_8b": ([(128256, Q6)], 0, 4096, F32, "random"),
}


def qg_sources(name):
    from oracle import gguf_synth as S
    specs, mode, k, _epi, how = QG_SHAPES[name]
    rng = np.random.Generator(np.random.PCG64(sum(map(ord, name))))
    srcs = []
    for rows, t in specs:
        if how == "random":
            blk = S.random_blocks(rng, t, rows, k)
        else:
            blk = S.quantize(rng.standard_normal((rows, k), dtype=np.float32) / np.float32(np.sqrt(k)), t)
        srcs.append((np.ascontiguousarray(blk).view(np.uint8).reshape(rows, k // 256, R.BLOCK_BYTES[t]), t))
    return srcs, mode


def qg_act(name, k, rows=128):
    """fp16 activations [128, k]; the tests put NaN in the rows at and beyond the batch"""
    rng = np.random.Generator(np.random.PCG64(sum(map(ord, name)) + 1))
    return rng.standard_normal((rows, k)).astype(np.float16)
