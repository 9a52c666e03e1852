// Launcher interface of the sm_90a kernels (implemented in gemv.cu, attention.cu, misc.cu,
// prefill.cu).  Host code (engine.cu) only sees plain structs and cudaStream_t.
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gl {

struct StepState;

// consumer warps per CTA: a launch-time choice among the compiled variants {8, 12, 16}
inline int gemv_threads(int consumer_warps) { return (consumer_warps + 1) * 32; }
constexpr int RING_MAX_SLOTS = 36;
constexpr int GEMV_MIN_SLOT_BYTES = 9216;   // four Q4_K row segments of 16 blocks
constexpr int KV_PAGE_TOKENS = 16;

enum GemvEpilogue : int {
    EPI_STORE = 0,   // out[r] = y[r]
    EPI_ADD = 1,     // out[r] = resid[r] + y[r]                (attn_output / ffn_down + residual)
    EPI_QKV = 2,     // seg0 -> RoPE -> q fp32; seg1 -> RoPE -> K page (fp16); seg2 -> V page (fp16)
    EPI_SILU = 3,    // pair mode: out[r] = silu(gate[r]) * up[r]
};

// Geometry of one GEMV phase: what the producer lane needs to stream it and the consumers need to walk it
// (gemv_core.cuh).  64 bytes, so that the persistent kernel can keep one per phase in its parameter constant bank.
struct ProdSeg {
    const uint8_t* w;      // engine layout (rowdot.h): [tile][K-segment][row in tile][seg_bytes]
    int rows;
    int n_items;           // ceil(rows / rows-per-item)   (pair mode: gate rows / (rpi/2))
};
struct alignas(16) ProdDesc {
    ProdSeg seg[3];
    unsigned short seg_bytes[3];   // bytes of one K-segment of one row
    unsigned char rpi[3];          // rows per item (4 or 2); pair mode: rpi/2 gate rows + rpi/2 up rows
    unsigned char type[3];         // ggml type id
    unsigned char nseg;
    unsigned char pair;            // 1: seg[0] / seg[1] are gate / up, staged together, EPI_SILU
    unsigned char nks;             // K-segments per row
    unsigned char seg_nb;          // 256-column blocks per K-segment (<= 16)
};
static_assert(sizeof(ProdDesc) == 64, "ProdDesc must stay 64 bytes");

struct GemvParams {
    ProdDesc pd;           // filled by gemv_plan()
    int cols;              // K, multiple of 256, <= 32768
    const float* x;        // [cols] fp32 activations (produced by the previous kernel)
    const float* norm_w;   // fused RMSNorm prologue when non-null
    float eps;
    int epi;
    float* out;            // STORE / ADD / SILU: [rows]; QKV: q fp32 [seg0.rows]
    const float* resid;    // ADD
    // EPI_QKV
    const float* rope_cos; // [n_ctx][head_dim/2]
    const float* rope_sin;
    int head_dim;
    int n_kv_heads;
    __half* k_cache;       // this layer: [n_pages][n_kv][KV_PAGE_TOKENS][head_dim]
    __half* v_cache;
    const int* page_table; // logical page -> physical page
    const StepState* st;   // position (EPI_QKV) / done flag
    // ring (stand-alone kernel; the persistent kernel has one ring for all phases)
    unsigned long long* trace;   // optional (GL_TRACE=1): [2 CTAs][8] %globaltimer stamps of this launch (first / last CTA)
    int hb256;             // stand-alone kernel: half-block prologue with 256-bit loads straight from global memory (gemv_core.cuh)
    int xraw_bytes;        // > 0: stand-alone kernel stages x raw (bulk copies) in a buffer of this size after the planes
    int xraw_nseg;         // pieces x is staged in: 1 (narrow rows) or the K-segments, two buffers deep (wide rows)
    int polite_tracks;     // > 0: only the first polite_tracks producer lanes prefetch before griddepcontrol.wait (see gemv.cu)
    int n_tracks;          // consumer warps that take items; each owns `depth` ring slots (gemv_core.cuh)
    int depth;
    int slot_bytes;
};

constexpr int GEMV_XRAW_MAX_COLS = 4096;    // x rows up to this width are staged raw (16 KB) for the half-block prologue

// a weight matrix as the planner sees it
struct GemvMat { const uint8_t* w; int type; int rows; int tile_rows; };   // tile_rows: what the matrix was stored with (rowdot.h)

// host helpers
size_t gemv_smem_bytes(int cols, int n_slots, int slot_bytes);
// Fills p.pd (K-segmentation, rows per item, item counts) for nmat matrices sharing cols; slot_bytes is the ring's
// slot size the items must fit.  Returns false if the shape is outside the kernel's envelope.
bool gemv_plan(GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, int slot_bytes);
cudaError_t gemv_configure();   // opt-in to large dynamic shared memory (once per process)
bool gemv_prologue_variants(int consumer_warps);   // are the specialised prologues (raw staging, 256-bit loads) compiled for this width?
cudaError_t gemv_launch(const GemvParams& p, int abits, int consumer_warps, int n_ctas, bool pdl, cudaStream_t s);
// (abits, consumer_warps) combinations that are compiled: abits in {16, 8} x warps in {8, 12, 16}
bool gemv_variant_ok(int abits, int consumer_warps);

// plain fp weights (F32/F16/BF16): y = W x, fp32 accumulate, no fusion
cudaError_t gemv_fp_launch(const void* w, int type, int rows, int cols, const float* x, float* y, cudaStream_t s);

// ---- small kernels ---------------------------------------------------------------------------
// x[n_embd] = dequant(token_embd[row token]); also publishes the token for this step.
struct EmbedParams {
    const uint8_t* w;       // token_embd in NATIVE GGUF layout (row gather)
    int type;
    int cols;
    int row_bytes;
    StepState* st;
    const int* prompt_ids;  // sequential prefill: token = prompt_ids[pos] while pos < n_prompt
    float* x;
};
cudaError_t embed_launch(const EmbedParams& p, bool pdl, cudaStream_t s);

struct AttnParams {
    const float* q;         // [n_head][head_dim] (already rotated)
    const __half* k_cache;  // layer base
    const __half* v_cache;
    const int* page_table;
    int n_table;            // entries in page_table
    const StepState* st;    // attends to positions 0..st->pos
    float* out;             // [n_head][head_dim]
    float* part_o;          // [n_head][n_splits][head_dim]
    float* part_ml;         // [n_head][n_splits][2]
    unsigned* counters;     // [n_kv_heads], zero between launches
    int n_head, n_kv_heads, head_dim, n_splits;
    float scale;
    unsigned long long* trace;   // optional (GL_TRACE=1): [2 CTAs][8] %globaltimer stamps
    int cluster;            // 1: the splits of a KV head form one thread-block cluster and merge through distributed shared memory
};
cudaError_t attn_decode_launch(const AttnParams& p, bool pdl, cudaStream_t s);
cudaError_t attn_decode_configure();
bool attn_cluster_ok(int n_head, int n_kv_heads, int head_dim, int n_splits);

struct SampleParams {
    const float* logits;
    int n_vocab;
    StepState* st;
    int* out_ids;
    float* out_logprobs;
    float* logits_keep;     // optional [max_steps][n_vocab] copy for parity tests
    int max_out;
    float* scratch;         // SAMPLE_SCRATCH_FLOATS floats, zeroed once: per-CTA (max, argmax, sum exp) + ticket
    unsigned long long* topk_scratch;   // TOPK_SCRATCH_BYTES, zeroed once: two-stage top-k sampler (sampler.cu); may be null
};
constexpr int SAMPLE_CTAS = 64;
constexpr int SAMPLE_SCRATCH_FLOATS = 3 * SAMPLE_CTAS + 1;
// greedy: argmax + log-softmax of the winner; advances StepState (pos+1, token=argmax, out_idx+1).
cudaError_t sample_greedy_launch(const SampleParams& p, bool pdl, cudaStream_t s);
// temperature / top-k / top-p draw with a counter-based generator (sampler.cu); same state update as the greedy sampler.
// Candidates are the top_k best logits, at most SAMPLE_MAX_K (top_k <= 0 "off" means SAMPLE_MAX_K, not the whole vocabulary).
constexpr int SAMPLE_MAX_K = 1024;
constexpr int TOPK_FAST_K = 64;              // top_k up to this takes the two-stage path ...
constexpr int TOPK_FAST_MAX_CTAS = 64;       // ... for vocabularies up to 64 x 2048 entries
constexpr size_t TOPK_SCRATCH_BYTES = (size_t)TOPK_FAST_MAX_CTAS * TOPK_FAST_K * 8 + TOPK_FAST_MAX_CTAS * 8 + 16;
bool sample_topk_fast_applies(int top_k, int n_vocab);
cudaError_t sample_topk_launch(const SampleParams& p, bool fast, bool pdl, cudaStream_t s);
// sequential-prefill step without sampling: pos += 1
cudaError_t advance_launch(StepState* st, bool pdl, cudaStream_t s);

// standalone pieces (used for fp-weight models and as unfused cross-checks)
cudaError_t rmsnorm_launch(const float* x, const float* w, int n, float eps, float* y, cudaStream_t s);
cudaError_t rope_kv_launch(float* q, const float* k, const float* v, int n_head, int n_kv, int head_dim,
                           const float* cos_t, const float* sin_t, const StepState* st, __half* k_cache,
                           __half* v_cache, const int* page_table, cudaStream_t s);
cudaError_t silu_mul_launch(const float* g, const float* u, int n, float* out, cudaStream_t s);
cudaError_t add_launch(const float* a, const float* b, int n, float* out, cudaStream_t s);
// generateEmbedding: out[n] = L2-normalised mean over rows of RMSNorm(h_t) * norm_w;  scratch: rstd [rows], pooled [n]
cudaError_t pool_embedding_launch(const float* h, int rows, int n, const float* norm_w, float eps, float* rstd_scratch, float* pooled_scratch,
                                  float* out, cudaStream_t s);
cudaError_t l2_flush_launch(float* buf, size_t n, cudaStream_t s);

}  // namespace gl
