// Engine: one loaded GGUF model on one H100.  Owns the weights in HBM (engine row layouts), the
// paged KV pool, the device-resident step state and the captured decode-step CUDA graphs.
// This is the native replacement for what sits behind OllamaService in the reference
// (/root/reference/client/src/services/OllamaService.ts) -- see include/gridllm_native.h.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <string>
#include <vector>

#include "../../include/gridllm_native.h"
#include "gguf_file.h"
#include "kernels.h"
#include "prefill.h"
#include "batch.h"
#include "qgemm.h"
#include "decode_mega.h"
#include "tokenizer.h"

namespace gl {

struct DevMatrix {
    uint8_t* w = nullptr;      // device
    int type = 0;
    int rows = 0, cols = 0;
    int row_stride = 0;        // row stride (bytes) of native / fp layouts; 0 for the tiled engine layout
    int tile_rows = 1;         // engine layout: rows per tile (rowdot.h)
    size_t gguf_bytes = 0;     // algorithmic bytes (GGUF payload)
    bool quantized() const { return type == T_Q4_K || type == T_Q6_K || type == T_Q8_0; }
};

struct LayerWeights {
    float* attn_norm = nullptr;
    float* ffn_norm = nullptr;
    DevMatrix wq, wk, wv, wo, wgate, wup, wdown;
    // resident 16-bit copies for the batched tensor-core prefill (built on the GPU at load)
    void* wqkv16 = nullptr;   // [(qd + 2 kvd) x n_embd]
    void* wo16 = nullptr;     // [n_embd x qd]
    void* wgu16 = nullptr;    // [2 n_ff x n_embd], rows interleaved 8 gate / 8 up
    void* wd16 = nullptr;     // [n_embd x n_ff]
};

struct Status {
    int code = GL_OK;
    std::string msg;
    bool ok() const { return code == GL_OK; }
};

class Engine {
public:
    static Status create(const std::string& path, int device, const gl_engine_opts* opts, Engine** out);
    ~Engine();

    Status info(gl_model_info* out) const;
    Status generate(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, gl_token_cb cb, void* user,
                    int32_t* out_ids, float* out_lp, gl_gen_stats* stats);
    Status embed(const int32_t* ids, const int32_t* offs, int n_seq, float* out, gl_gen_stats* stats);
    Status last_logits(int step, float* out, int n_vocab);
    // continuous batching (engine_batch.cu): B open sequences share one decode step
    Status seq_open(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, int* slot);
    Status seq_open_many(const int32_t* ids, const int32_t* offs, int n_seq, const gl_sample_opts* opts, int32_t* slots, int* n_opened);
    Status batch_step(int32_t* slots, int32_t* ids, float* logprobs, int32_t* done, int cap, int* n);
    Status seq_close(int slot);
    Status seq_logits(int slot, float* out, int n_vocab);
    Status seq_stats(int slot, gl_gen_stats* out) const;
    void batch_counters(uint64_t out[8], bool reset) {
        for (int i = 0; i < 8; ++i) { out[i] = bc_[i]; if (reset) bc_[i] = 0; }
        out[7] = have_qg_ ? 2 : 1;                    // which weights the batched step reads (2: quantised, 1: 16-bit copy)
    }
    Status time_batch_step(int batch, int ctx_len, int iters, float* ms, int* launches, uint64_t* wbytes);
    Status sample_logits(const float* logits, int n_vocab, const gl_sample_opts& so, int out_index, int* id, float* logprob);
    Status gemv_host(int type, const void* w_host, int rows, int cols, const float* x, float* y, int iters, float* ms);
    Status gemv_tensor(const std::string& name, const float* x, float* y, int iters, int flush, float* ms, uint64_t* wbytes);
    Status rmsnorm(const float* x, const float* w, int n, float eps, float* y);
    Status decode_step(int token, float* logits, int* argmax, float* logprob);
    Status kv_reset();
    Status prefill(const int32_t* ids, int n, float* last_logits);
    Status time_decode(int ctx_len, int iters, float* ms, int* launches);
    Status mega_trace(unsigned long long* out, int cap, int* n_ctas, int* n_phases);
    Status perop_trace(unsigned long long* out, int cap, int* n_launches);
    int position() const { return host_pos_; }
    const Tokenizer& tokenizer() const { return tok_; }

private:
    Engine() = default;
    Status load(const std::string& path, int device, const gl_engine_opts* opts);
    Status upload_matrix(const GGUFTensor& t, DevMatrix& m, bool native_layout, bool paired = false);
    Status upload_f32(const GGUFTensor& t, float** out, int expect);
    Status ensure_pages(int n_tokens);
    Status enqueue_step(cudaStream_t s, bool with_head, bool keep_logits, int* n_launch);
    Status enqueue_gemv(cudaStream_t s, GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, int* n_launch);
    Status plain_gemv(cudaStream_t s, const DevMatrix& m, const float* x, float* y, int* n_launch);
    Status build_graphs();
    Status set_state(int pos, int token, int n_prompt, int out_idx, const gl_sample_opts* so);
    StepState make_state(int pos, int token, int n_prompt, int out_idx, const gl_sample_opts* so, int* sampler) const;
    Status run_steps(int n_nohead, int n_head, bool keep_logits);
    Status enqueue_head(cudaStream_t s, bool keep_logits, int* n_launch);
    Status build_prefill_weights();
    Status build_mega();
    Status launch_mega(int n_steps, bool with_head, bool keep_logits);
    Status ensure_prefill_scratch(int t_pad);
    Status prefill_batched(int n, int* n_launch);     // tokens already in prompt_ids_[0..n)
    // embeddings: several sequences in ONE prompt pass (block-diagonal causal attention); seq s = rows [starts[s], starts[s] + lens[s])
    // tables: per sequence, the device page table its K / V rows are cached through (null: nothing is cached -- embeddings)
    Status prefill_packed(const std::vector<int>& starts, const std::vector<int>& lens, int t_rows, int* n_launch,
                          const std::vector<const int*>* tables = nullptr);
    static constexpr int EMB_PACK_TOKENS = 2048;      // rows of one packed pass (each sequence starts on a 128-row boundary)
    int* pk_ids_ = nullptr;                           // [EMB_PACK_TOKENS] token ids of a pack (pad rows: token 0)
    float *emb_out_ = nullptr, *emb_rstd_ = nullptr, *emb_pooled_ = nullptr;
    int emb_out_cap_ = 0;
    bool can_batch_prefill(int n) const { return have_w16_ && prefill_mode_ != 1 && host_pos_ == 0 && n >= prefill_min_ && n <= 4096; }
    const DevMatrix* find_matrix(const std::string& name) const;

    // model
    GGUFFile gguf_;
    Tokenizer tok_;
    gl_model_info info_{};
    int n_layer_ = 0, n_embd_ = 0, n_head_ = 0, n_kv_ = 0, hd_ = 0, n_ff_ = 0, n_vocab_ = 0, n_ctx_ = 0;
    float eps_ = 1e-5f, rope_base_ = 10000.f;
    std::vector<LayerWeights> layers_;
    DevMatrix tok_embd_;       // native layout (row gather)
    DevMatrix output_;         // engine layout (GEMV)
    float* output_norm_ = nullptr;
    bool all_quant_ = true;

    // options
    int device_ = 0, sm_count_ = 132;
    int abits_ = 16;
    int nw_ = 12;              // consumer warps per CTA of the GEMV / persistent kernels
    int ring_depth_ = 2;       // ring slots per consumer warp (track depth, gemv_core.cuh)
    int ring_depth_max_ = 3;
    int polite_tracks_ = 3;    // attn_output: producer lanes that may prefetch before the attention kernel is done (0: all)
    bool xraw_wide_ = false;   // wide rows: the same through two K-segment buffers (opt-in: GL_XRAW_WIDE=1)
    // GEMV prologue variant.  Every GEMV launch of a step should be the SAME kernel: two variants alternating (61 + 68 KB of
    // code, plus 30 KB of attention) overflow the SM's instruction cache and cost 0.5 us per launch (runs 52 / 53).
    bool hb256_ = true;        // half-block prologue with 256-bit global loads, all widths (default)
    bool xraw_ = false;        // narrow rows: raw x staging by bulk copy + half-block prologue (opt-in, GL_XRAW=1)
    bool lean_rings_ = true;   // one ring slot per warp for single-round kernels (room for the next kernel's CTAs)
    bool use_graph_ = true, use_pdl_ = true, fused_ = true;
    int smem_kb_ = 224, attn_splits_ = 16;
    bool attn_cluster_ = false;
    int prefill_mode_ = 0, prefill_min_ = 8;
    bool have_w16_ = false, prefill_bf16_ = false, prefill_tc5_ = true;
    bool prefill_fuse_rope_ = true;  // RoPE / split / cache append in the QKV GEMM's epilogue (GL_PREFILL_FUSE_ROPE=0: the stand-alone kernel)
    bool prefill_flash_ = true;     // fused prompt attention (prefill_attn.cu); GL_PREFILL_FLASH=0: the three-launch path, for A/B runs
    // prefill scratch (grown on demand)
    int pf_cap_ = 0;
    float *pf_x_ = nullptr, *pf_qkv_ = nullptr, *pf_s_ = nullptr;
    void *pf_xn_ = nullptr, *pf_attn_ = nullptr, *pf_h_ = nullptr;
    __half *pf_q_ = nullptr, *pf_k_ = nullptr, *pf_vt_ = nullptr, *pf_p_ = nullptr;
    std::vector<void*> pf_allocs_;
    int last_prefill_launches_ = 0;
    // persistent decode kernel
    bool use_mega_ = false;
    MegaPhase *mega_head_ = nullptr, *mega_nohead_ = nullptr;
    int mega_n_head_ = 0, mega_n_nohead_ = 0, mega_tracks_ = 0, mega_depth_ = 2, mega_slot_bytes_ = 0, mega_max_cols_ = 0;
    unsigned* bar_counter_ = nullptr;
    float* head_part_ = nullptr;
    int mega_launches_ = 0;
    int mega_splits_ = 16;
    unsigned long long* mega_trace_ = nullptr;
    static constexpr int PEROP_TRACE_LAUNCHES = 512;
    unsigned long long* perop_trace_ = nullptr;    // GL_TRACE=1: [launch of the step][first / last CTA][4] %globaltimer stamps
    std::vector<ProdDesc> mega_prod_;

    // device state
    cudaStream_t stream_ = nullptr;
    std::vector<void*> allocs_;
    float *x_ = nullptr, *xn_ = nullptr, *q_ = nullptr, *ktmp_ = nullptr, *vtmp_ = nullptr, *attn_ = nullptr, *h_ = nullptr,
          *gate_ = nullptr, *up_ = nullptr, *ytmp_ = nullptr, *logits_ = nullptr;
    float *rope_cos_ = nullptr, *rope_sin_ = nullptr;
    float *part_o_ = nullptr, *part_ml_ = nullptr;
    unsigned* counters_ = nullptr;
    float* sample_scratch_ = nullptr;
    unsigned long long* topk_scratch_ = nullptr;
    __half *kcache_ = nullptr, *vcache_ = nullptr;    // [layer][page][kv][16][hd]
    size_t kv_layer_elems_ = 0;
    int n_pages_ = 0;                                // entries of ONE sequence's page table (n_ctx / 16)
    int pool_pages_ = 0;                             // physical pages of the pool all sequences share
    int* page_table_ = nullptr;                      // device
    std::vector<int> free_pages_;
    std::vector<int> seq_pages_;
    StepState* st_ = nullptr;
    int* prompt_ids_ = nullptr;
    int* out_ids_ = nullptr;
    float* out_lp_ = nullptr;
    float* logits_keep_ = nullptr;
    int keep_cap_ = 0;
    float* flush_buf_ = nullptr;
    size_t flush_elems_ = 0;
    int max_out_ = 0;
    int host_pos_ = 0;

    // ---- continuous batching (engine_batch.cu) ----
    struct SeqSlot {
        bool open = false, done = false, first_pending = false;
        std::vector<int> pages;
        int n_prompt = 0, n_pred = 0, produced = 0, sampler = 0;
        int32_t last_token = 0;
        float first_lp = 0.f;
        int last_row = -1;                            // row of the last batched step this sequence took part in
        int64_t prefill_ns = 0, eval_ns = 0, t_open_ns = 0;      // device time of its prefill / of the steps it took part in; host clock at open
        int launches = 0;
        bool stopped = false;                         // ended on a stop token
    };
    static constexpr int N_BUCKETS = 5;               // batch-size buckets of the captured step: 8, 16, 32, 64, 128 rows
    int max_batch_ = 0;                               // gl_engine_opts.max_batch (0: batching off)
    bool batch_ready_ = false;
    int batch_weights_ = 0;                           // 1: resident 16-bit copy, 2: quantised weights (engine_batch.cu picks for 0)
    std::vector<SeqSlot> slots_;
    std::vector<int> last_rows_;                      // composition the device-resident BatchCtl currently describes
    int last_bucket_ = 0;
    BatchCtl* bctl_ = nullptr;
    StepState* bst_ = nullptr;                        // [MAX_BATCH]
    int* btables_ = nullptr;                          // [MAX_BATCH][n_pages_]
    int *bids_ = nullptr, *bout_ids_ = nullptr;
    static constexpr int BSSQ_PARTS = 512;       // 32-row slices of the residual stream the folded RMSNorm can sum (n_embd <= 16 384)
    float* bssq_[2] = {nullptr, nullptr};
    float *bx_ = nullptr, *bqkv_ = nullptr, *bq_ = nullptr, *blogits_ = nullptr, *bfirst_logits_ = nullptr, *bout_lp_ = nullptr, *bpart_o_ = nullptr, *bpart_ml_ = nullptr, *bsample_scratch_ = nullptr;
    __half *bxn16_ = nullptr, *battn16_ = nullptr, *bh16_ = nullptr;
    unsigned* bcounters_ = nullptr;
    BatchOut* bout_ = nullptr;
    void* head16_ = nullptr;                          // [n_vocab x n_embd] fp16 copy of the lm_head (16-bit batched path)
    // batched step on the QUANTISED weights (qgemm.cu): a second copy of the matrices in the QG qtile layout, same bytes as the GGUF
    struct QLayer { QGemmWeights qkv, o, gu, down; };
    std::vector<QLayer> qlayers_;
    QGemmWeights qhead_;
    float* qpartial_ = nullptr;
    bool have_qg_ = false;
    std::string qg_why_not_;                          // why the quantised path is unavailable for this model (message for batch_weights = 2)
    Status build_qgemm_weights();
    Status pack_qgemm(const std::vector<const GGUFTensor*>& src, int mode, QGemmWeights& out, uint8_t*& tmp, size_t& tmp_cap);
    cudaGraphExec_t g_batch_[N_BUCKETS] = {};
    int batch_launches_ = 0;                          // kernels of one batched step
    uint64_t bc_[8] = {};                             // gl_batch_counters
    Status ensure_batch_state();
    Status seq_open_single(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, int* slot);
    Status enqueue_batch_step(cudaStream_t s, int bucket, int* n_launch);
    Status run_batch_graph(int bucket);
    static int bucket_of(int rows) { int b = 8; while (b < rows) b <<= 1; return b; }
    static int bucket_index(int bucket) { int i = 0; while ((8 << i) < bucket) ++i; return i; }

    cudaGraphExec_t g_nohead_ = nullptr;
    cudaGraphExec_t g_head_var_[3][2] = {};   // [sampler of the running request][logits kept]
    // The top-k samplers are launched WITHOUT programmatic dependent launch: their CTAs (33 KB of shared memory each) resident
    // beside the lm_head CTAs cost the step 60 us (run 67: 1.537 -> 1.478 ms/token at top_k 40); the greedy sampler keeps it.
    bool sampler_pdl_ = false;
    bool greedy_pdl_ = false;                 // the greedy sampler likewise (64 small CTAs: 3 us per token, run 68)
    int sampler_ = 0;                          // 0 greedy (argmax), 1 / 2: the two kernels of sampler.cu (temperature > 0)
    int launches_nohead_ = 0, launches_head_ = 0;
    cudaEvent_t ev_[4] = {nullptr, nullptr, nullptr, nullptr};
    int64_t load_ns_ = 0;
    uint64_t weight_bytes_ = 0, decode_bytes_ = 0, n_params_ = 0;
};

void set_last_error(const std::string& s);
const char* get_last_error();

}  // namespace gl
