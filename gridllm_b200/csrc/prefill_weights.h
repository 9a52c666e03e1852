// Where the tensor-core prompt pass reads its 16-bit layer matrices from (rule in include/gridllm_native.h, prefill_mode).
// Host only and self-contained, so that the CPU suite can compile and test it on its own (tests/hostcheck/prefill_weights_shim.cpp).
//   resident : a 16-bit copy of every layer matrix, built once at load (2 bytes per weight); the only source continuous
//              batching can use
//   streamed : one staging buffer the size of the largest per-layer operand; before each of a layer's four linear GEMMs the
//              operand is dequantised into it from the decode layout, so a pass costs one extra HBM write + read of the
//              16-bit weights but a model whose copy cannot fit (70B-class at q4) still gets a tensor-core prompt pass
#pragma once
#include <stdint.h>

namespace gl {

enum PrefillWeights : int {
    PREFILL_W_NONE = 0,        // prefill_mode 1: prompts step through the decode kernels, nothing is built
    PREFILL_W_RESIDENT = 1,
    PREFILL_W_STREAMED = 2,
};

// the copy is built only when this much HBM stays free beside it (prompt scratch, batching state, the lm_head copy)
constexpr uint64_t PREFILL_COPY_MARGIN = (uint64_t)4 << 30;

// 16-bit elements of one layer's four GEMM operands: Q | K | V rows, attn_output, gate / up interleaved, ffn_down
inline uint64_t prefill_qkv_elems(int n_embd, int n_head, int n_kv, int hd) { return (uint64_t)(n_head + 2 * n_kv) * hd * n_embd; }
inline uint64_t prefill_o_elems(int n_embd, int n_head, int hd) { return (uint64_t)n_embd * n_head * hd; }
inline uint64_t prefill_gu_elems(int n_embd, int n_ff) { return (uint64_t)2 * n_ff * n_embd; }
inline uint64_t prefill_down_elems(int n_embd, int n_ff) { return (uint64_t)n_embd * n_ff; }

// bytes of the resident copy of every layer matrix
inline uint64_t prefill_copy_bytes(int n_layer, int n_embd, int n_head, int n_kv, int hd, int n_ff) {
    const uint64_t per_layer = prefill_qkv_elems(n_embd, n_head, n_kv, hd) + prefill_o_elems(n_embd, n_head, hd) + prefill_gu_elems(n_embd, n_ff) +
                               prefill_down_elems(n_embd, n_ff);
    return per_layer * 2 * (uint64_t)n_layer;
}

// bytes of the streamed pass's one staging buffer: the largest operand (gate / up for every Llama shape)
inline uint64_t prefill_stage_bytes(int n_embd, int n_head, int n_kv, int hd, int n_ff) {
    uint64_t m = prefill_qkv_elems(n_embd, n_head, n_kv, hd);
    const uint64_t o = prefill_o_elems(n_embd, n_head, hd), gu = prefill_gu_elems(n_embd, n_ff), d = prefill_down_elems(n_embd, n_ff);
    if (o > m) m = o;
    if (gu > m) m = gu;
    if (d > m) m = d;
    return m * 2;
}

// The source of a model's prompt pass.  request: GL_PREFILL_WEIGHTS (0 auto, 1 resident, 2 streamed; anything else is auto).
// Auto keeps the resident copy whenever copy_bytes + PREFILL_COPY_MARGIN <= free_bytes and streams otherwise.  Returns -1 when
// the resident copy is requested and does not fit (the load fails with GL_ERR_NOMEM).
inline int prefill_weights_source(int prefill_mode, int request, uint64_t copy_bytes, uint64_t free_bytes) {
    if (prefill_mode == 1) return PREFILL_W_NONE;
    if (request == PREFILL_W_STREAMED) return PREFILL_W_STREAMED;
    const bool fits = copy_bytes + PREFILL_COPY_MARGIN <= free_bytes;
    if (request == PREFILL_W_RESIDENT) return fits ? PREFILL_W_RESIDENT : -1;
    return fits ? PREFILL_W_RESIDENT : PREFILL_W_STREAMED;
}

}  // namespace gl
