// Launchers of the batched-prefill kernels (prefill.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gl {

enum GemmEpilogue : int {
    GEMM_EPI_F32 = 0,      // C fp32 = acc
    GEMM_EPI_ADD_F32 = 1,  // C fp32 += acc                 (residual add in place)
    GEMM_EPI_T16 = 2,      // C 16-bit = acc
    GEMM_EPI_SILU = 3,     // B rows interleaved [8 gate | 8 up]: C16[m][col] = silu(gate) * up
    GEMM_EPI_ROPE_SPLIT = 4,  // the QKV projection: RoPE on the q / k columns, 16-bit Q / K rows, V^T columns, fp16 cache pages (prefill_tc5.cu only)
};

// The sequences of one prompt pass: sequence i owns rows [start[i], start[i] + len[i]) of the packed activation matrix (starts at
// 128-row boundaries); table[i] = its KV page table on the device (null: nothing is cached).  pos0[i] = the absolute position
// of its first row (0 for a whole prompt; > 0 for a chunk that continues a sequence whose earlier positions are in its pages).
constexpr int PF_MAX_SEGS = 32;
struct PrefillSegs {
    int n;
    int start[PF_MAX_SEGS];
    int len[PF_MAX_SEGS];
    const int* table[PF_MAX_SEGS];
    int pos0[PF_MAX_SEGS];
};
// what GEMM_EPI_ROPE_SPLIT writes instead of C (the arguments of rope_split_segs_launch, which it replaces)
struct RopeSplitArgs {
    const float* cos_t;
    const float* sin_t;
    __half* q;          // [rows][n_head * hd]
    __half* k;          // [rows][n_kv * hd]
    __half* vt;         // [n_kv * hd][vt_ld]
    __half* k_cache;    // this layer's pages, or null
    __half* v_cache;
    int n_head, n_kv, hd, vt_ld;
    PrefillSegs segs;
};

// C[M x N] = A[M x K] * B[N x K]^T, 16-bit inputs (fp16 or bf16), fp32 accumulate; strides in ELEMENTS.
struct GemmParams {
    const void* a;
    const void* b;
    void* c;
    int m, n, k;
    int lda, ldb, ldc;
    int batch;                 // blockIdx.z
    long long a_batch_stride;  // elements of A per batch
    long long b_batch_stride;  // elements of B per (batch / b_batch_div)   (GQA: several query heads share one KV head)
    long long c_batch_stride;
    int b_batch_div;
    int epi;
    int causal_skip;           // 1: skip tiles entirely above the diagonal (S = Q K^T)
    int causal_k;              // 1: limit K to the last row of the tile + 1 (O = P V, P lower-triangular)
    const RopeSplitArgs* rope; // GEMM_EPI_ROPE_SPLIT: where the rotated / split rows go (host pointer, copied into the launch)
};

cudaError_t prefill_configure();   // per device: opt in to the GEMM's dynamic shared memory
cudaError_t gemm_tn_launch(const GemmParams& p, bool bf16, cudaStream_t s);      // mma.sync path (batched attention GEMMs)
// wgmma / TMA path (prefill_tc5.cu) for the plain linear layers; a_rows_alloc = rows of A that exist in memory
cudaError_t gemm_tc5_configure();
bool gemm_tc5_supported(const GemmParams& p);
cudaError_t gemm_tc5_launch(const GemmParams& p, int a_rows_alloc, bool bf16, cudaStream_t s);
// One source matrix of a 16-bit GEMM operand: engine layout (rowdot.h) for Q4_K / Q6_K / Q8_0, plain rows of row_stride bytes
// (a multiple of 16) for F32 / F16 / BF16.  Its rows land at dst_row0 + r, or interleaved in groups of 8 as GEMM_EPI_SILU reads them.
struct DequantSrc {
    const uint8_t* w;
    int type, rows, row_stride, tile_rows;
    int dst_row0;
    int interleave;     // 0: plain; 1: gate rows, 2: up rows of a [8 gate | 8 up] matrix (row r -> (r / 8) * 16 + (0 | 8) + r % 8)
};
constexpr int DEQUANT_MAX_SRCS = 3;
struct DequantOp {
    DequantSrc src[DEQUANT_MAX_SRCS];
    int n_src;
    int cols;           // columns of every source = row length of dst (a multiple of 8)
    void* dst;          // [rows][cols] fp16 or bf16
};
// one launch dequantises every source of op (Q | K | V, gate / up, or a single matrix)
cudaError_t dequant_launch(const DequantOp& op, bool bf16, cudaStream_t s);
cudaError_t rmsnorm_rows_launch(const float* x, const float* w, int rows, int rows_pad, int n, float eps, void* y, bool bf16, cudaStream_t s);
cudaError_t rope_split_launch(const float* qkv, int t_rows, int t_pad, int pos0, int n_head, int n_kv, int hd, const float* cos_t,
                              const float* sin_t, __half* qo, __half* ko, __half* vt, __half* k_cache, __half* v_cache,
                              const int* page_table, int vt_ld /* row stride of vt; k_cache may be null (nothing cached) */, cudaStream_t s);
// ---- fused prompt attention (prefill_attn.cu) --------------------------------------------------------------------
cudaError_t flash_prefill_configure();
bool flash_prefill_supported(int hd);
// out[rows][n_head * hd] = causal softmax(q k^T * scale) v per sequence and head; q / k rows, vt = V^T [n_kv * hd][vt_ld].
// When some segment has pos0 > 0, its query rows attend to keys 0 .. pos0 + len - 1 read from this layer's fp16 pages
// (k_cache / v_cache through segs.table; the segment's own rows must already be appended) and k / vt are not read.
cudaError_t flash_prefill_launch(const __half* q, const __half* k, const __half* vt, __half* out, const PrefillSegs& segs, int n_head, int n_kv,
                                 int hd, int vt_ld, float scale, const __half* k_cache, const __half* v_cache, cudaStream_t s);
// rope_split for every sequence of a pack in one launch (rows_pad = rows of the pack, padding rows are zeroed)
cudaError_t rope_split_segs_launch(const float* qkv, int rows_pad, int n_head, int n_kv, int hd, const float* cos_t, const float* sin_t, __half* qo,
                                   __half* ko, __half* vt, __half* k_cache, __half* v_cache, int vt_ld, const PrefillSegs& segs, cudaStream_t s);
cudaError_t softmax_causal_launch(const float* sc, int n_head, int t_rows, int t_pad, float scale, __half* p, cudaStream_t s);
cudaError_t embed_rows_launch(const uint8_t* w, int type, int cols, int row_bytes, const int* ids, int t_rows, float* x, cudaStream_t s);

}  // namespace gl
