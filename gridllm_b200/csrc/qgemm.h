// Launcher interface of the batched decode GEMM on quantised weights (qgemm.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "prefill.h"

namespace gl {

// One weight matrix (or a row-wise concatenation / interleave of several) in the QG layout (qgemm_layout.h):
// tiles of 128 output rows, each tile = nkb consecutive qtiles (one per 256-column block), tiles in order.
struct QGemmWeights {
    uint8_t* w = nullptr;             // qtile stream
    uint64_t* tile_off = nullptr;     // device [n_tiles]: byte offset of a tile's first qtile
    uint8_t* tile_type = nullptr;     // device [n_tiles]: ggml type of the tile's rows (12 Q4_K / 14 Q6_K)
    unsigned* counters = nullptr;     // device [n_tiles]: parts of a split tile stored so far, zero between launches
    int n = 0;                        // output features (rows of the matrix), multiple of 128
    int k = 0;                        // input features, multiple of 256
    int n_tiles = 0, nkb = 0;
    uint64_t bytes = 0;               // bytes of the stream = the GGUF bytes of the matrix
    // "tiles [0, tile_split) are type0, the rest type1": lets the kernel compute a tile's type and offset instead of loading them
    bool two_segment = false, has_q6k = false;
    int type0 = 0, type1 = 0, tile_split = 0;
    uint64_t off_split = 0;
    void describe(const uint64_t* toff_host, const uint8_t* ttype_host) {
        type0 = ttype_host[0];
        tile_split = n_tiles;
        type1 = type0;
        off_split = 0;
        has_q6k = false;
        two_segment = true;
        for (int t = 0; t < n_tiles; ++t) {
            if (ttype_host[t] == 14) has_q6k = true;
            if (tile_split == n_tiles && ttype_host[t] != type0) { tile_split = t; type1 = ttype_host[t]; off_split = toff_host[t]; }
            else if (tile_split != n_tiles && ttype_host[t] != type1) two_segment = false;
        }
    }
};

// source of rows for the load-time packer: a matrix in NATIVE GGUF row layout on the device
struct QGemmSource { const uint8_t* w; int type; int rows; };

constexpr int QGEMM_MAX_GRID = 132;       // one CTA per SM of an H100 SXM

// RMSNorm folded into the GEMMs around it (no separate kernel, no launch boundary):
//   the residual-add GEMM in front of a norm (attn_output, ffn_down) also writes xg[b][n] = fp16(x_new[b][n] * gamma[n] / 16) -- the
//   NEXT GEMM's activation rows, scaled by the norm's weights but not yet by 1 / rms -- and, per (32-row slice, token), the sum
//   of x_new^2 (`ssq_out`, [parts][64]);  the GEMM behind the norm (QKV, gate/up, lm_head) multiplies its accumulator by
//   16 / sqrt(sum of the parts / n_norm + eps) per token: W (g x / rms) = (W (g x)) / rms.  The parts are summed in a fixed order.
//   Producer side needs the cluster mode of the kernel (qgemm_uses_cluster); otherwise the engine keeps the stand-alone kernel.
struct QGemmNorm {
    const float* gamma_next = nullptr;   // producer: weights of the norm BEHIND this GEMM's output, [n]
    __half* xg_out = nullptr;            // producer: [>= nb rows][ldxg] fp16
    int ldxg = 0;
    float* ssq_out = nullptr;            // producer: [n_tiles * 4][64]
    const float* ssq_in = nullptr;       // consumer: the parts written by the GEMM before; null = activations are already normalised
    int ssq_parts = 0;
    int n_norm = 0;                      // consumer: width of the normalised vector (n_embd)
    float eps = 0.f;
};
constexpr float QGEMM_NORM_PRESCALE = 1.0f / 16.0f;

size_t qgemm_partial_floats(int nb);          // floats of split-tile scratch a launch with nb batch columns may use
cudaError_t qgemm_configure();                // opt in to the kernel's dynamic shared memory (once per device)
bool qgemm_batch_ok(int nb);                  // nb in {16, 32, 64}
// Pack nsrc native matrices (all with k columns) into one QG stream.  mode 0: rows concatenated (Q | K | V);
// mode 1: two sources interleaved in groups of 8 rows (8 gate | 8 up), the order the SiLU*mul epilogue expects.
// dst must hold the sum of the sources' GGUF bytes; tile_off / tile_type get n_tiles entries (host arrays).
cudaError_t qgemm_pack_launch(const QGemmSource* src, int nsrc, int mode, int k, uint8_t* dst, uint64_t* tile_off_host, uint8_t* tile_type_host,
                              cudaStream_t s);
// C[b][n] (+)= sum_k act[b][k] * W[n][k] for b < nb batch rows.  act: fp16 [>= 128 rows][k] (rows beyond the batch are
// read but their results never stored); epi as GemmEpilogue (F32, ADD_F32, SILU with C fp16 [.. x n/2]).
cudaError_t qgemm_launch(const QGemmWeights& wt, const __half* act, int act_rows_alloc, int nb, void* c, int ldc, int epi, float* partial,
                         int n_sm, cudaStream_t s, const QGemmNorm* norm = nullptr);
// will qgemm_launch run this GEMM in cluster mode (tile-aligned split-K inside clusters of four)?
bool qgemm_uses_cluster(const QGemmWeights& wt, int nb, int epi, int n_sm);

}  // namespace gl
