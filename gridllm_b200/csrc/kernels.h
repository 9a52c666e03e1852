// Launcher interface of the sm_90a kernels (implemented in gemv.cu, attention.cu, misc.cu,
// prefill.cu).  Host code (engine.cu) only sees plain structs and cudaStream_t.
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "schema_fsm.h"

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

// The switches a stand-alone GEMV launch is staged by (engine.h members; GL_WARPS, GL_SMEM_KB, GL_RING_DEPTH_MAX, GL_HB256,
// GL_XRAW, GL_XRAW_WIDE, GL_LEAN_RINGS).  The defaults are the engine's when no variable overrides them.
struct GemvGeomOpts {
    int nw = 12;               // consumer warps
    int smem_kb = 227;         // dynamic shared memory a CTA may take
    int ring_depth_max = 3;    // slots per track
    bool hb256 = true;         // half-block prologue with 256-bit loads, every width it fits
    bool xraw = false;         // narrow rows staged raw by one bulk copy
    bool xraw_wide = false;    // wide rows staged raw by K-segment pieces
    bool lean_rings = true;    // one slot per track for single-round, single-K-segment launches
};
enum GemvGeomResult : int { GEMV_GEOM_OK = 0, GEMV_GEOM_SHAPE = 1, GEMV_GEOM_SMEM = 2 };
// Plans one launch (gemv_plan) and decides its ring geometry over n_ctas CTAs: slot bytes, the prologue variant (hb256,
// xraw_bytes, xraw_nseg), n_tracks x depth and the lean ring.  GEMV_GEOM_SHAPE: the shape is outside the kernel's envelope;
// GEMV_GEOM_SMEM: the staging does not fit shared memory.
int gemv_geometry(GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, const GemvGeomOpts& o, int n_ctas);
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
    const int* prompt_ids;  // sequential prefill: token = prompt_ids[pos] while pos < n_prompt and nothing was drawn yet
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
    int n_head, n_kv_heads, head_dim;
    int n_splits;           // 8 or 16: the CTAs of one KV head, one thread-block cluster (attn_splits_ok)
    float scale;
    unsigned long long* trace;   // optional (GL_TRACE=1): [2 CTAs][8] %globaltimer stamps
};
cudaError_t attn_decode_launch(const AttnParams& p, bool pdl, cudaStream_t s);
cudaError_t attn_decode_configure();
bool attn_splits_ok(int n_head, int n_kv_heads, int head_dim, int n_splits);

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

// Repetition / presence / frequency penalties in place on the logits, before the sampler (penalty.cu; semantics in
// include/gridllm_native.h).  One CTA per row.  History of a row's sequence: prompt[0..st.n_prompt) then out_ids[0..st.out_idx).
struct BatchCtl;
struct PenaltyParams {
    float* logits;          // row r at logits + r * n_vocab
    int n_vocab;
    StepState* st;          // ctl == null: the one sequence's state; else [slots]
    const BatchCtl* ctl;    // batched step: row -> slot, rows >= n_rows leave at once; null: one row, slot 0
    const int* prompt;      // [slot][prompt_stride]
    int prompt_stride;
    const int* out_ids;     // [slot][out_stride]
    int out_stride;
    int* counts;            // [slot][n_vocab] int32, zero between launches (each launch leaves it zero)
};
cudaError_t penalty_launch(const PenaltyParams& p, int rows, bool pdl, cudaStream_t s);

// JSON grammar mask in place on the logits, after the penalties and before the sampler (schema_mask.cu; language in
// schema_fsm.h over json_fsm.h, semantics in include/gridllm_native.h: format json and gl_format_schema).  Grid: vocabulary
// chunks x rows, one thread per token.  Rows with StepState.json = 1 follow the schema their SchemaSlot points at (format json:
// the built-in any-object schema); other rows and finished rows leave at once.
struct SchemaSlot {
    const uint8_t* tab;         // the row's compiled schema (schema_compile.cpp blob), set by the host when the request starts
    uint32_t pad[2];
    SchemaState st[2];          // st[i & 1]: the automaton state after the output's first i tokens (written by the mask kernel
                                // of output i, read by that of output i + 1)
};
struct SchemaMaskParams {
    float* logits;              // row r at logits + r * n_vocab
    int n_vocab;
    StepState* st;              // ctl == null: the one sequence's state; else [slots]
    const BatchCtl* ctl;        // batched step: row -> slot, rows >= n_rows leave at once; null: one row
    SchemaSlot* ss;             // ctl == null: the one sequence's entry; else [slots]
    const uint32_t* offsets;    // [n_vocab + 1] byte offsets of the token pieces
    const uint8_t* bytes;       // the pieces, back to back
    const uint8_t* cls;         // [n_vocab] class bits (JSON_CLS_*)
};
cudaError_t schema_mask_launch(const SchemaMaskParams& p, int rows, bool pdl, cudaStream_t s);
// one thread: e's automaton from the initial state through the pieces of ids[0..n-1), stored as entry (n - 1) & 1 (the mask
// kernel of output n advances by ids[n-1] itself).  gl_constrain_logits.
cudaError_t schema_replay_launch(SchemaSlot* e, const int* ids, int n, const uint32_t* offsets, const uint8_t* bytes, cudaStream_t s);

// Context shift (kv_shift.cu; rule in include/gridllm_native.h): for each sequence of the list, the rows [keep + discard,
// keep + discard + n_rows) of every layer and KV head move to [keep, keep + n_rows) of its paged cache, K rotated by -discard
// positions (fp32 pair rotation with the cos / sin table row `discard`, rounded to fp16), V copied bit for bit; then
// st->pos -= discard (st may be null).  HBM-bound: 16-byte loads and stores.
// ORDERING: the batch-1 decode attention reads the position before its griddepcontrol.wait, on the promise that the position
// only grows within a step; a shift makes it go down.  So the shift is launched WITHOUT programmatic dependent launch and never
// executes griddepcontrol.launch_dependents: nothing of the next step starts before it completes.
struct KvShiftSeq {
    const int* table;       // the sequence's page table (logical -> physical page)
    int keep, discard, n_rows;
    StepState* st;
};
struct KvShiftParams {
    __half* k_cache;        // layer 0 base, [layer][page][kv][16][head_dim]
    __half* v_cache;
    size_t layer_elems;     // elements of one layer of the pool
    const KvShiftSeq* seqs; // device, [n_seq]
    int n_seq;
    int n_layer, n_kv, head_dim;
    const float* cos_t;     // [n_ctx][head_dim / 2]
    const float* sin_t;
};
// max_rows: the largest n_rows of the list.  A sequence whose discard is smaller than its n_rows (source and destination
// overlap) moves its rows in launches of at most `discard` rows each, in increasing order: n_rounds = the largest
// ceil(n_rows / discard) of the list (at least 1; one launch when no ranges overlap, the case of the rule's discard).
int kv_shift_rounds(int n_rows, int discard);
cudaError_t kv_shift_launch(const KvShiftParams& p, int max_rows, int n_rounds, cudaStream_t s);

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
// the same pooling over a sequence that arrives in several prompt passes: each pass adds the column sums of its rows' RMSNorm(h_t)
// (without norm_w) to sum [n] (accumulate = 0: the first pass overwrites it); the finish scales by norm_w / total_rows in place
// and L2-normalises into out
cudaError_t pool_embedding_sum_launch(const float* h, int rows, int n, float eps, float* rstd_scratch, float* sum, bool accumulate, cudaStream_t s);
cudaError_t pool_embedding_finish_launch(float* sum, int total_rows, int n, const float* norm_w, float* out, cudaStream_t s);
cudaError_t l2_flush_launch(float* buf, size_t n, cudaStream_t s);

}  // namespace gl
