// Engine: continuous batching (SURVEY.md section 8f.1; include/gridllm_native.h gl_seq_open / gl_batch_step / gl_seq_close).
//
// The reference worker holds one job at a time (/root/reference/client/src/services/WorkerClientService.ts:500-505;
// MAX_CONCURRENT_JOBS_PER_WORKER, server/src/config/index.ts:31).  With that limit raised, every job the worker holds is an
// open SEQUENCE here: its own KV pages out of the shared pool, its own device-resident StepState (position, last token,
// sampling options), its own page-table row.  One batched decode step then serves all of them:
//     gather tokens -> embedding rows -> per layer { RMSNorm rows -> QKV GEMM -> RoPE + KV append per row -> paged attention per
//     row -> O GEMM (+residual) -> RMSNorm rows -> gate/up GEMM (SiLU*mul) -> down GEMM (+residual) } -> final norm -> lm_head
//     GEMM -> sampler per row -> collect
// The GEMMs are tensor-core GEMMs with M = rows of the step: the weights are read ONCE per step for all sequences.  The step
// is captured as a CUDA graph per batch-size bucket (8 / 16 / 32 / 64 / 128 rows); which sequences form the rows is device
// state (BatchCtl), so joining and leaving costs one small copy, not a re-capture.
// A sequence's arithmetic never looks at another row: its tokens do not depend on who shares the batch.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "engine.h"
#include "context_shift.h"

namespace gl {

namespace {
Status failb(int code, const std::string& m) { return Status{code, m}; }
#define CU(expr)                                                                                  \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) return failb(GL_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
#define ST(expr)                 \
    do {                         \
        Status _s = (expr);      \
        if (!_s.ok()) return _s; \
    } while (0)

int attn_splits_for(int bucket, int n_kv, int n_sm) {
    // ONE wave of CTAs: the tensor-core kernel keeps two CTAs per SM resident (96 KB of page buffers each), and a second,
    // mostly empty wave costs as much as the first (B = 32 with 2 splits: 512 CTAs on 444 slots took 28.8 us against 11 us of
    // KV traffic).  Within one wave, as many splits as fit: every split shortens the per-warp chain of dependent page loads.
    const int slots = 2 * n_sm;
    int s = slots / std::max(1, n_kv * bucket);
    return std::max(1, std::min(16, s));
}
}  // namespace

// One GEMM's weights -> QG qtile stream: the sources' native GGUF bytes go to the device as they are (mmap -> staging buffer),
// the packer kernel (qgemm.cu) regroups the bits of every super-block into the qtile planes.
Status Engine::pack_qgemm(const std::vector<const GGUFTensor*>& src, int mode, QGemmWeights& out, uint8_t*& tmp, size_t& tmp_cap) {
    size_t total = 0;
    int rows = 0;
    for (const GGUFTensor* t : src) { total += t->nbytes; rows += (int)t->rows(); }
    if (total + 256 > tmp_cap) {
        if (tmp) cudaFree(tmp);
        tmp = nullptr;
        CU(cudaMalloc((void**)&tmp, total + 256));
        tmp_cap = total + 256;
    }
    QGemmSource qs[3];
    size_t off = 0;
    for (size_t i = 0; i < src.size(); ++i) {
        CU(cudaMemcpyAsync(tmp + off, src[i]->data, src[i]->nbytes, cudaMemcpyHostToDevice, stream_));
        qs[i] = QGemmSource{tmp + off, (int)src[i]->type, (int)src[i]->rows()};
        off += (src[i]->nbytes + 255) & ~(size_t)255;
        if (off > tmp_cap) return failb(GL_ERR_NOMEM, "qgemm staging overflow");
    }
    const int k = (int)src[0]->cols();
    out.n = rows; out.k = k; out.nkb = k / 256; out.n_tiles = rows / 128; out.bytes = total;
    CU(cudaMalloc((void**)&out.w, total + 256));
    allocs_.push_back(out.w);
    std::vector<uint64_t> toff(out.n_tiles);
    std::vector<uint8_t> ttype(out.n_tiles);
    CU(qgemm_pack_launch(qs, (int)src.size(), mode, k, out.w, toff.data(), ttype.data(), stream_));
    CU(cudaMalloc((void**)&out.tile_off, (size_t)out.n_tiles * 8));
    allocs_.push_back(out.tile_off);
    CU(cudaMalloc((void**)&out.tile_type, (size_t)out.n_tiles + 16));
    allocs_.push_back(out.tile_type);
    CU(cudaMalloc((void**)&out.counters, (size_t)out.n_tiles * 4));
    allocs_.push_back(out.counters);
    CU(cudaMemcpy(out.tile_off, toff.data(), (size_t)out.n_tiles * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(out.tile_type, ttype.data(), (size_t)out.n_tiles, cudaMemcpyHostToDevice));
    CU(cudaMemset(out.counters, 0, (size_t)out.n_tiles * 4));
    out.describe(toff.data(), ttype.data());
    return {};
}

// The second copy of the weights for the batched step on quantised weights: same bytes as the GGUF (4.6 GB for Llama-3-8B
// q4_K_M), QG layout.  Only for models whose matrices are all Q4_K / Q6_K with 128-row / 256-column granularity; anything else
// keeps the 16-bit path (have_qg_ stays false, qg_why_not_ says why).
Status Engine::build_qgemm_weights() {
    have_qg_ = false;
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_;
    auto ok_t = [](const GGUFTensor* t) { return t && (t->type == T_Q4_K || t->type == T_Q6_K); };
    if (n_embd_ % 256 || n_ff_ % 256 || qd % 256) { qg_why_not_ = "widths must be multiples of 256"; return {}; }
    if (qd % 128 || kvd % 128 || n_embd_ % 128 || n_ff_ % 64 || n_vocab_ % 128) { qg_why_not_ = "matrix heights must be multiples of 128"; return {}; }
    const GGUFTensor* tout = gguf_.tensor("output.weight");
    if (!tout) tout = gguf_.tensor("token_embd.weight");
    if (!ok_t(tout)) { qg_why_not_ = "output.weight is not Q4_K / Q6_K"; return {}; }
    std::vector<std::vector<const GGUFTensor*>> per_layer;
    for (int il = 0; il < n_layer_; ++il) {
        const std::string p = "blk." + std::to_string(il) + ".";
        std::vector<const GGUFTensor*> t;
        for (const char* n : {"attn_q.weight", "attn_k.weight", "attn_v.weight", "attn_output.weight", "ffn_gate.weight", "ffn_up.weight", "ffn_down.weight"}) {
            const GGUFTensor* x = gguf_.tensor(p + n);
            if (!ok_t(x)) { qg_why_not_ = "tensor " + p + n + " is not Q4_K / Q6_K"; return {}; }
            t.push_back(x);
        }
        if (t[4]->type != t[5]->type) { qg_why_not_ = "ffn_gate / ffn_up of different types"; return {}; }
        per_layer.push_back(t);
    }
    CU(qgemm_configure());
    uint8_t* tmp = nullptr;
    size_t tmp_cap = 0;
    qlayers_.assign(n_layer_, QLayer{});
    Status st;
    for (int il = 0; il < n_layer_ && st.ok(); ++il) {
        const auto& t = per_layer[il];
        st = pack_qgemm({t[0], t[1], t[2]}, 0, qlayers_[il].qkv, tmp, tmp_cap);
        if (st.ok()) st = pack_qgemm({t[3]}, 0, qlayers_[il].o, tmp, tmp_cap);
        if (st.ok()) st = pack_qgemm({t[4], t[5]}, 1, qlayers_[il].gu, tmp, tmp_cap);
        if (st.ok()) st = pack_qgemm({t[6]}, 0, qlayers_[il].down, tmp, tmp_cap);
    }
    if (st.ok()) st = pack_qgemm({tout}, 0, qhead_, tmp, tmp_cap);
    if (tmp) cudaFree(tmp);
    ST(st);
    CU(cudaMalloc((void**)&qpartial_, qgemm_partial_floats(64) * 4));
    allocs_.push_back(qpartial_);
    have_qg_ = true;
    return {};
}

Status Engine::ensure_batch_state() {
    if (batch_ready_) return {};
    if (bst_) return failb(GL_ERR_CUDA, "continuous batching: an earlier initialisation failed on this engine");
    if (max_batch_ < 2) return failb(GL_ERR_UNSUPPORTED, "continuous batching is off: create the engine with gl_engine_opts.max_batch >= 2");
    if (prefill_w_ != PREFILL_W_RESIDENT) return failb(GL_ERR_UNSUPPORTED, "continuous batching needs the resident 16-bit weights (not enough HBM at load, or prefill_mode 1)");
    if (n_ff_ % 8) return failb(GL_ERR_UNSUPPORTED, "continuous batching: n_ff must be a multiple of 8");
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_, ldq = qd + 2 * kvd;
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess) { allocs_.push_back(*p); e = cudaMemsetAsync(*p, 0, bytes, stream_); }
        return e;
    };
    const size_t R = MAX_BATCH;
    CU(batch_attn_configure());
    CU(dalloc((void**)&bctl_, sizeof(BatchCtl)));
    CU(dalloc((void**)&btables_, R * n_pages_ * 4));
    CU(dalloc((void**)&bids_, R * 4));
    CU(dalloc((void**)&bout_ids_, R * max_out_ * 4));
    CU(dalloc((void**)&bout_lp_, R * max_out_ * 4));
    CU(dalloc((void**)&bout_, R * sizeof(BatchOut)));
    CU(dalloc((void**)&bx_, R * n_embd_ * 4));
    CU(dalloc((void**)&bxn16_, R * n_embd_ * 2));
    CU(dalloc((void**)&bqkv_, R * ldq * 4));
    CU(dalloc((void**)&bq_, R * qd * 4));
    CU(dalloc((void**)&battn16_, R * qd * 2));
    CU(dalloc((void**)&bh16_, R * n_ff_ * 2));
    CU(dalloc((void**)&blogits_, R * n_vocab_ * 4));
    CU(dalloc((void**)&bfirst_logits_, (size_t)max_batch_ * n_vocab_ * 4));      // logits each sequence's FIRST token was drawn from (gl_seq_logits)
    CU(dalloc((void**)&bpart_o_, R * n_head_ * 16 * hd_ * 4));
    CU(dalloc((void**)&bpart_ml_, R * n_head_ * 16 * 2 * 4));
    CU(dalloc((void**)&bcounters_, R * n_kv_ * 4));
    for (int i = 0; i < 2; ++i) CU(dalloc((void**)&bssq_[i], (size_t)BSSQ_PARTS * 64 * 4));      // folded RMSNorm: per-slice sums of squares
    CU(dalloc((void**)&bsample_scratch_, R * BATCH_SAMPLE_ROW_FLOATS * 4));
    // the lm_head as a 16-bit matrix (the layer matrices already have their copy: build_prefill_weights)
    CU(dalloc(&head16_, (size_t)n_vocab_ * n_embd_ * 2));
    {
        DequantOp op{};
        op.src[0] = {output_.w, output_.type, output_.rows, output_.row_stride, output_.tile_rows, 0, 0};
        op.n_src = 1; op.cols = n_embd_; op.dst = head16_;
        CU(dequant_launch(op, false, stream_));
    }
    CU(dalloc((void**)&bst_, sizeof(StepState) * R));
    CU(cudaStreamSynchronize(stream_));
    if (batch_weights_ != 1) {
        ST(build_qgemm_weights());
        if (!have_qg_ && batch_weights_ == 2)
            return failb(GL_ERR_UNSUPPORTED, "batch_weights = 2 (quantised weights) is not available for this model: " + qg_why_not_);
    }
    slots_.assign(MAX_BATCH, SeqSlot{});
    last_rows_.clear();
    last_bucket_ = 0;
    // one un-captured pass with an empty batch (n_rows = 0: the per-row kernels leave at once, the GEMMs run on zero rows): every
    // launch configuration is validated -- and every lazily initialised driver entry point touched -- OUTSIDE stream capture,
    // where an error has a name
    int nl = 0;
    ST(enqueue_batch_step(stream_, 8, false, false, &nl));
    CU(cudaStreamSynchronize(stream_));
    batch_launches_ = nl;
    batch_ready_ = true;
    return {};
}

Status Engine::ensure_batch_penalty() {
    if (bpen_counts_) return {};
    int* pr = nullptr;
    int* cnt = nullptr;
    CU(cudaMalloc((void**)&pr, (size_t)max_batch_ * n_ctx_ * 4));
    allocs_.push_back(pr);
    CU(cudaMalloc((void**)&cnt, (size_t)max_batch_ * n_vocab_ * 4));
    allocs_.push_back(cnt);
    CU(cudaMemsetAsync(cnt, 0, (size_t)max_batch_ * n_vocab_ * 4, stream_));
    bprompt_ = pr;
    bpen_counts_ = cnt;
    return {};
}

Status Engine::keep_prompt(int slot, const int32_t* prompt, int n_prompt) {
    ST(ensure_batch_penalty());
    CU(cudaMemcpyAsync(bprompt_ + (size_t)slot * n_ctx_, prompt, (size_t)n_prompt * 4, cudaMemcpyHostToDevice, stream_));
    return {};
}

bool Engine::take_pages(const int32_t* prompt, int n_prompt, int n_pred, bool share, std::vector<int>* pages, int* r) {
    pages->clear();
    *r = 0;
    if (share) {
        const int l = pages_.match(prompt, n_prompt, pages);
        *r = shared_prefix_reuse(l, n_prompt, prefill_min_);
        pages->resize(*r / KV_PAGE_TOKENS);
        for (int p : *pages) pages_.ref(p);            // before the allocation below, which may evict retained pages
    }
    const int own = (n_prompt + n_pred + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS - *r / KV_PAGE_TOKENS;
    if (!pages_.alloc(own, *pages)) {
        release_pages(*pages);
        *r = 0;
        return false;
    }
    return true;
}

void Engine::release_pages(std::vector<int>& pages) {
    for (int p : pages) pages_.release(p);
    pages.clear();
}

void Engine::index_prompt_pages(const int32_t* prompt, int n_prompt, const std::vector<int>& pages, int from, std::vector<int>* added) {
    for (int j = from; j < n_prompt / KV_PAGE_TOKENS; ++j) {
        if (!pages_.insert(j > 0 ? pages[j - 1] : -1, prompt + (size_t)j * KV_PAGE_TOKENS, pages[j])) break;      // already indexed
        if (added) added->push_back(pages[j]);
    }
}

// Prefill a prompt into a free slot's own pages and draw its first token.  The single-sequence code runs unchanged on the
// slot's state: the members it reads (page table, step state, output buffers) point at the slot's rows for the duration.
// One prompt.  It takes the SAME path as a prompt opened together with others (gl_seq_open_many with one entry: packed prompt
// pass, lm_head GEMM on the 16-bit matrix), so a sequence's first token does not depend on how it was admitted; only prompts the
// packed pass does not take (shorter than 8 tokens, longer than a pack, no 16-bit weights) go through seq_open_single.
Status Engine::seq_open(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, int* slot_out) {
    if (!prompt || n_prompt <= 0 || !slot_out) return failb(GL_ERR_INVALID, "seq_open: empty prompt");
    int n_eval = n_prompt;                            // what the prompt pass evaluates: a prompt of W ids or more is cut first
    if (context_shift_ && n_prompt >= n_ctx_ && so.num_keep >= -1) n_eval = n_ctx_ - shift_discard(n_ctx_, shift_keep(so.num_keep, n_prompt, n_ctx_));
    if (prefill_w_ == PREFILL_W_RESIDENT && n_eval >= prefill_min_ && n_eval <= EMB_PACK_TOKENS) {
        const int32_t offs[2] = {0, n_prompt};
        int32_t slot = -1;
        int n = 0;
        ST(seq_open_many(prompt, offs, 1, &so, &slot, &n));
        *slot_out = slot;
        return {};
    }
    return seq_open_single(prompt, n_prompt, so, slot_out);
}

Status Engine::seq_open_single(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, int* slot_out, bool was_cut) {
    CU(cudaSetDevice(device_));
    if (!prompt || n_prompt <= 0 || !slot_out) return failb(GL_ERR_INVALID, "seq_open: empty prompt");
    for (int i = 0; i < n_prompt; ++i)
        if (prompt[i] < 0 || prompt[i] >= n_vocab_) return failb(GL_ERR_INVALID, "prompt token id out of range");
    DrawPlan plan;
    ST(plan_draw(so, false, &plan));
    ST(ensure_batch_state());
    const int n_pred = so.num_predict > 0 ? so.num_predict : 128;
    // context shift: cut an over-long prompt; a sequence that may shift reserves pages for W positions at most and shares none
    int keep = 0, page_pred = n_pred;                 // pages for n_prompt + page_pred positions
    bool shifting = false;
    std::vector<int32_t> cut_ids;
    if (context_shift_) {
        ST(shift_plan(so, n_prompt, n_pred, &keep));
        shifting = was_cut || n_prompt + n_pred > n_ctx_;
        if (n_prompt >= n_ctx_) {
            cut_ids.resize(n_ctx_);
            n_prompt = cut_prompt(prompt, n_prompt, n_ctx_, keep, shift_discard(n_ctx_, keep), cut_ids.data());
            prompt = cut_ids.data();
        }
        page_pred = std::min(n_pred, n_ctx_ - n_prompt);
    } else if (n_prompt + n_pred > n_ctx_) {
        return failb(GL_ERR_CONTEXT, "prompt + num_predict exceeds the engine context");
    }
    int slot = -1;
    for (int i = 0; i < max_batch_; ++i)
        if (!slots_[i].open) { slot = i; break; }
    if (slot < 0) return failb(GL_ERR_NOMEM, "no free sequence slot (max_batch " + std::to_string(max_batch_) + ")");
    // pages for every position it will hold, reserved up front: a step can never run out.  Only a prompt that takes the prompt
    // pass shares a prefix (and indexes its pages afterwards); short prompts step through the decode kernels.
    const bool share = share_prefixes() && can_batch_prefill(0, n_prompt) && !shifting;
    SeqSlot& S = slots_[slot];
    S = SeqSlot{};
    int r = 0;
    if (!take_pages(prompt, n_prompt, page_pred, share, &S.pages, &r)) return failb(GL_ERR_NOMEM, "KV page pool exhausted");
    int* table = btables_ + (size_t)slot * n_pages_;
    CU(cudaMemcpyAsync(table, S.pages.data(), S.pages.size() * 4, cudaMemcpyHostToDevice, stream_));
    if (plan.penalised) {                                 // the head of the history the batched steps penalise with
        Status ks = keep_prompt(slot, prompt, n_prompt);
        if (!ks.ok()) {
            release_pages(S.pages);
            S = SeqSlot{};
            return ks;
        }
    }

    struct Saved { int* pt; StepState* st; int* oi; float* ol; int hp; } sv{page_table_, st_, out_ids_, out_lp_, host_pos_};
    page_table_ = table; st_ = bst_ + slot; out_ids_ = bout_ids_ + (size_t)slot * max_out_; out_lp_ = bout_lp_ + (size_t)slot * max_out_; host_pos_ = 0;
    Status rs;
    int prefill_launches = 0;
    const int64_t t_open = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
    do {
        int& dummy = prefill_launches;
        cudaError_t ce = cudaMemcpyAsync(prompt_ids_, prompt, (size_t)n_prompt * 4, cudaMemcpyHostToDevice, stream_);
        if (ce == cudaSuccess) ce = cudaEventRecord(ev_[2], stream_);
        if (ce != cudaSuccess) { rs = failb(GL_ERR_CUDA, cudaGetErrorString(ce)); break; }
        if (can_batch_prefill(0, n_prompt)) {      // any length: passes of PF_CHUNK rows, the later ones over the slot's pages
            rs = set_state(n_prompt - 1, prompt[n_prompt - 1], n_prompt, 0, &so, plan);
            if (rs.ok()) rs = prefill_batched(r, n_prompt - r, &dummy);      // positions [0, r) are in the shared pages
            if (rs.ok()) rs = enqueue_head(stream_, false, &dummy);
        } else {      // short prompts: plain launches of the decode step (the captured graphs hold the engine's own pointers)
            rs = set_state(0, prompt[0], n_prompt, 0, &so, plan);
            for (int i = 0; rs.ok() && i < n_prompt; ++i) rs = enqueue_step(stream_, i == n_prompt - 1, false, &dummy);
        }
        if (!rs.ok()) break;
        StepState hs{};
        float lp = 0.f;
        ce = cudaEventRecord(ev_[3], stream_);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(bfirst_logits_ + (size_t)slot * n_vocab_, logits_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToDevice, stream_);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&hs, st_, sizeof(hs), cudaMemcpyDeviceToHost, stream_);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(&lp, out_lp_, 4, cudaMemcpyDeviceToHost, stream_);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(stream_);
        if (ce != cudaSuccess) { rs = failb(GL_ERR_CUDA, cudaGetErrorString(ce)); break; }
        float pms = 0.f;
        cudaEventElapsedTime(&pms, ev_[2], ev_[3]);
        S.prefill_ns = (int64_t)(pms * 1e6);
        S.pos = hs.pos;
        S.last_token = hs.token;
        S.first_lp = lp;
        S.done = hs.done != 0;
    } while (false);
    page_table_ = sv.pt; st_ = sv.st; out_ids_ = sv.oi; out_lp_ = sv.ol; host_pos_ = sv.hp;
    if (!rs.ok()) {
        release_pages(S.pages);
        S = SeqSlot{};
        return rs;
    }
    if (share) index_prompt_pages(prompt, n_prompt, S.pages, r / KV_PAGE_TOKENS, nullptr);
    S.open = true;
    S.n_shared = r;
    S.n_prompt = n_prompt; S.n_pred = n_pred; S.produced = 0; S.plan = plan; S.first_pending = true;
    S.keep = keep; S.shift_on = shifting;
    S.t_open_ns = t_open; S.launches = prefill_launches; S.stopped = S.done;
    bc_[3] += (uint64_t)S.prefill_ns; bc_[4] += (uint64_t)(n_prompt - r); bc_[5] += 1; bc_[6] += (uint64_t)prefill_launches;
    bc_[7] += (uint64_t)r;
    *slot_out = slot;
    return {};
}

// Several prompts at once: they share ONE packed prompt pass per <= EMB_PACK_TOKENS rows (engine_prefill.cu prompt_pass: the
// linear layers see all their tokens as one [T x n_embd] matrix, each sequence attends only to itself and caches its K / V rows
// through its own page table), then one lm_head GEMM over the last hidden row of every sequence and one sampler pass draw all the
// first tokens.  32 prompts of 512 tokens: 8 passes with M = 2048 instead of 32 passes with M = 512, and one 1 GB lm_head read
// instead of 32.  Sequences are opened in order until slots or KV pages run out: slots[i] = -1 for those that did not fit.
Status Engine::seq_open_many(const int32_t* ids, const int32_t* offs, int n_seq, const gl_sample_opts* opts, int32_t* slots_out, int* n_opened) {
    CU(cudaSetDevice(device_));
    if (!ids || !offs || !opts || !slots_out || !n_opened || n_seq <= 0) return failb(GL_ERR_INVALID, "seq_open_many: bad argument");
    *n_opened = 0;
    ST(ensure_batch_state());
    std::vector<DrawPlan> plans(n_seq);
    // context shift: per prompt its keep count and whether it may shift (or was cut); over-long prompts are cut into a copy
    std::vector<int> keeps(n_seq, 0);
    std::vector<char> shifting(n_seq, 0);
    std::vector<int32_t> cut_ids;
    std::vector<int32_t> cut_offs;
    for (int i = 0; i < n_seq; ++i) {
        slots_out[i] = -1;
        const int n = offs[i + 1] - offs[i];
        if (n <= 0) return failb(GL_ERR_INVALID, "seq_open_many: empty prompt");
        for (int k = 0; k < n; ++k)
            if (ids[offs[i] + k] < 0 || ids[offs[i] + k] >= n_vocab_) return failb(GL_ERR_INVALID, "prompt token id out of range");
        ST(plan_draw(opts[i], false, &plans[i]));
        const int n_pred = opts[i].num_predict > 0 ? opts[i].num_predict : 128;
        if (context_shift_) {
            ST(shift_plan(opts[i], n, n_pred, &keeps[i]));
            shifting[i] = n + n_pred > n_ctx_;
        } else if (n + n_pred > n_ctx_) {
            return failb(GL_ERR_CONTEXT, "prompt + num_predict exceeds the engine context");
        }
    }
    if (context_shift_) {
        cut_offs.assign(1, 0);
        for (int i = 0; i < n_seq; ++i) {
            const int n = offs[i + 1] - offs[i];
            const size_t at = cut_ids.size();
            cut_ids.resize(at + n);
            const int m = cut_prompt(ids + offs[i], n, n_ctx_, keeps[i], shift_discard(n_ctx_, keeps[i]), cut_ids.data() + at);
            cut_ids.resize(at + m);
            cut_offs.push_back((int32_t)cut_ids.size());
        }
        ids = cut_ids.data();
        offs = cut_offs.data();
    }
    ST(ensure_pack_buffers());
    const bool packable = prefill_w_ == PREFILL_W_RESIDENT;
    const bool share = packable && share_prefixes();
    const int64_t t_open = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
    int next = 0;
    std::vector<int32_t> h_ids(EMB_PACK_TOKENS);
    while (next < n_seq) {
        // ---- one pack: as many of the next prompts as fit EMB_PACK_TOKENS rows, free slots and free pages ----
        std::vector<PromptSeq> seqs;
        std::vector<int> which, pslots;
        std::vector<int> indexed;                    // pages this pack added to the prefix index (taken out again if its pass fails)
        int rows = 0;
        bool out_of_room = false;
        std::fill(h_ids.begin(), h_ids.end(), 0);
        while (next < n_seq && (int)which.size() < MAX_BATCH) {
            const int32_t* prompt = ids + offs[next];
            const int n = offs[next + 1] - offs[next];
            if (!packable || n > EMB_PACK_TOKENS || n < prefill_min_) break;              // this one goes through gl_seq_open's own path
            // the positions a shared prefix covers are not evaluated: only the suffix takes rows of the pack
            const bool share_i = share && !shifting[next];
            const int r_max = share_i ? shared_prefix_reuse(pages_.match(prompt, n, nullptr), n, prefill_min_) : 0;
            if (rows + (n - r_max + 127) / 128 * 128 > EMB_PACK_TOKENS) break;
            int n_pred = opts[next].num_predict > 0 ? opts[next].num_predict : 128;
            if (shifting[next]) n_pred = std::min(n_pred, n_ctx_ - n);         // pages for min(n_prompt + num_predict, W) positions
            int slot = -1;
            for (int k = 0; k < max_batch_; ++k)
                if (!slots_[k].open && std::find(pslots.begin(), pslots.end(), k) == pslots.end()) { slot = k; break; }
            if (slot < 0) { out_of_room = true; break; }
            SeqSlot& S = slots_[slot];
            S = SeqSlot{};
            int r = 0;
            if (!take_pages(prompt, n, n_pred, share_i, &S.pages, &r)) { out_of_room = true; break; }
            CU(cudaMemcpyAsync(btables_ + (size_t)slot * n_pages_, S.pages.data(), S.pages.size() * 4, cudaMemcpyHostToDevice, stream_));
            // its prompt pages go into the index now, so that later prompts of this pack share them: the QKV projection of every
            // layer writes this sequence's K / V rows to its pages before that layer's attention reads them through a sharer's
            // table (a sharer comes after its owner in the pack)
            if (share_i) index_prompt_pages(prompt, n, S.pages, r / KV_PAGE_TOKENS, &indexed);
            const int len = n - r;
            std::memcpy(h_ids.data() + rows, prompt + r, (size_t)len * 4);
            seqs.push_back({rows, len, r, btables_ + (size_t)slot * n_pages_});
            which.push_back(next); pslots.push_back(slot);
            rows += (len + 127) / 128 * 128;
            ++next;
        }
        if (which.empty()) {
            if (out_of_room) break;
            // a prompt the packed pass does not take (too short / too long / no 16-bit weights): the single-sequence open
            int slot = -1;
            Status st = seq_open_single(ids + offs[next], offs[next + 1] - offs[next], opts[next], &slot, shifting[next] != 0);
            if (!st.ok()) {
                if (st.code == GL_ERR_NOMEM || *n_opened > 0) break;      // what was opened so far stays open and is reported
                return st;
            }
            slots_out[next] = slot;
            ++*n_opened;
            ++next;
            continue;
        }
        const int P = (int)which.size();
        Status rs;
        int launches = 0;
        float pack_ms = 0.f;
        std::vector<BatchOut> ho(P);
        do {
            cudaError_t ce = cudaMemcpyAsync(pk_ids_, h_ids.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, stream_);
            if (ce == cudaSuccess) ce = cudaEventRecord(ev_[2], stream_);
            if (ce != cudaSuccess) { rs = failb(GL_ERR_CUDA, cudaGetErrorString(ce)); break; }
            rs = prompt_pass(seqs, rows, pk_ids_, &launches);
            if (!rs.ok()) break;
            // first tokens: last hidden row of each sequence -> rows 0..P-1 of the batched-step buffers -> final norm -> lm_head GEMM
            for (int i = 0; i < P && ce == cudaSuccess; ++i)
                ce = cudaMemcpyAsync(bx_ + (size_t)i * n_embd_, pf_x_ + (size_t)(seqs[i].start + seqs[i].len - 1) * n_embd_, (size_t)n_embd_ * 4,
                                     cudaMemcpyDeviceToDevice, stream_);
            if (ce == cudaSuccess) ce = batch_rmsnorm_launch(bx_, output_norm_, P, n_embd_, eps_, bxn16_, stream_);
            if (ce == cudaSuccess) {
                GemmParams g{};
                g.a = bxn16_; g.b = head16_; g.c = blogits_; g.m = P; g.n = n_vocab_; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = n_vocab_;
                g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_F32;
                ce = gemm_tc5_supported(g) ? gemm_tc5_launch(g, MAX_BATCH, false, stream_) : gemm_tn_launch(g, false, stream_);
            }
            launches += P + 2;
            // the sequences' step states and a temporary row map (the next gl_batch_step uploads its own)
            std::vector<StepState> hst(P);
            BatchCtl hc{};
            hc.n_rows = P;
            bool any_pen = false, any_mask = false;
            for (int i = 0; i < P && ce == cudaSuccess; ++i) {
                const int w = which[i], n = seqs[i].len + seqs[i].pos0;
                const DrawPlan& plan = plans[w];
                hst[i] = make_state(n - 1, ids[offs[w] + n - 1], n, 0, &opts[w]);
                slots_[pslots[i]].plan = plan;
                if (plan.masked) {
                    Status bs = schema_bind(sch_ + 1 + pslots[i], plan.format);
                    if (!bs.ok()) { rs = bs; break; }
                    any_mask = true;
                }
                if (plan.penalised) {                        // the head of the history the penalty kernel reads
                    Status ks = keep_prompt(pslots[i], ids + offs[w], n);
                    if (!ks.ok()) { rs = ks; break; }
                    any_pen = true;
                }
                hc.row_slot[i] = pslots[i];
                ce = cudaMemcpyAsync(bst_ + pslots[i], &hst[i], sizeof(StepState), cudaMemcpyHostToDevice, stream_);
            }
            if (!rs.ok()) break;
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(bctl_, &hc, sizeof(hc), cudaMemcpyHostToDevice, stream_);
            last_rows_.clear();
            const int bucket = bucket_of(P);
            if (ce == cudaSuccess) ce = enqueue_pre_draw(stream_, bucket, any_pen, any_mask, nullptr, &launches);      // before every first-token draw of the pack
            if (ce == cudaSuccess) ce = batch_sample_greedy_launch(blogits_, n_vocab_, bucket, bctl_, bst_, bout_ids_, bout_lp_, max_out_, bsample_scratch_, stream_);
            for (int i = 0; i < P && ce == cudaSuccess; ++i) {
                const int slot = pslots[i];
                if (slots_[slot].plan.sampler != 0) {
                    SampleParams sp{blogits_ + (size_t)i * n_vocab_, n_vocab_, bst_ + slot, bout_ids_ + (size_t)slot * max_out_,
                                    bout_lp_ + (size_t)slot * max_out_, nullptr, max_out_, sample_scratch_, topk_scratch_};
                    ce = sample_topk_launch(sp, slots_[slot].plan.sampler == 1, false, stream_);
                }
                if (ce == cudaSuccess)
                    ce = cudaMemcpyAsync(bfirst_logits_ + (size_t)slot * n_vocab_, blogits_ + (size_t)i * n_vocab_, (size_t)n_vocab_ * 4,
                                         cudaMemcpyDeviceToDevice, stream_);
            }
            if (ce == cudaSuccess) ce = batch_collect_launch(bctl_, bst_, bout_lp_, max_out_, bout_, bucket, stream_);
            if (ce == cudaSuccess) ce = cudaEventRecord(ev_[3], stream_);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(ho.data(), bout_, sizeof(BatchOut) * P, cudaMemcpyDeviceToHost, stream_);
            if (ce == cudaSuccess) ce = cudaStreamSynchronize(stream_);
            if (ce != cudaSuccess) { rs = failb(GL_ERR_CUDA, cudaGetErrorString(ce)); break; }
            cudaEventElapsedTime(&pack_ms, ev_[2], ev_[3]);
            launches += 3;
        } while (false);
        if (!rs.ok()) {
            for (size_t k = indexed.size(); k-- > 0;) pages_.forget(indexed[k]);
            for (int i = 0; i < P; ++i) {
                release_pages(slots_[pslots[i]].pages);
                slots_[pslots[i]] = SeqSlot{};
            }
            if (*n_opened > 0) break;                // earlier packs are open and reported; the caller sees -1 for the rest
            return rs;
        }
        int64_t pack_tokens = 0;
        for (int i = 0; i < P; ++i) pack_tokens += seqs[i].len;
        for (int i = 0; i < P; ++i) {
            SeqSlot& S = slots_[pslots[i]];
            const int w = which[i];
            S.open = true;
            S.n_prompt = seqs[i].len + seqs[i].pos0;
            S.n_shared = seqs[i].pos0;
            S.n_pred = opts[w].num_predict > 0 ? opts[w].num_predict : 128;
            S.produced = 0;
            S.first_pending = true;
            S.last_token = ho[i].token;
            S.pos = ho[i].pos;
            S.keep = keeps[w];
            S.shift_on = shifting[w] != 0;
            S.first_lp = ho[i].logprob;
            S.done = ho[i].done != 0;
            S.stopped = S.done;
            S.t_open_ns = t_open;
            S.prefill_ns = (int64_t)(pack_ms * 1e6 * (double)seqs[i].len / (double)pack_tokens);      // its share of the pass
            S.launches = launches / P;
            slots_out[w] = pslots[i];
            bc_[4] += (uint64_t)seqs[i].len;
            bc_[5] += 1;
            bc_[7] += (uint64_t)seqs[i].pos0;
        }
        bc_[3] += (uint64_t)(pack_ms * 1e6);
        bc_[6] += (uint64_t)launches;
        *n_opened += P;
        if (out_of_room) break;
    }
    if (*n_opened == 0) return failb(GL_ERR_NOMEM, "no free sequence slot / KV pages for any of the prompts");
    return {};
}

Status Engine::seq_close(int slot) {
    if (slot < 0 || slot >= (int)slots_.size() || !slots_[slot].open) return failb(GL_ERR_INVALID, "seq_close: no such open sequence");
    release_pages(slots_[slot].pages);           // indexed prompt pages stay retained for later prompts
    slots_[slot] = SeqSlot{};
    return {};
}

Status Engine::seq_stats(int slot, gl_gen_stats* out) const {
    if (slot < 0 || slot >= (int)slots_.size() || !slots_[slot].open || !out) return failb(GL_ERR_INVALID, "seq_stats: no such open sequence");
    const SeqSlot& S = slots_[slot];
    std::memset(out, 0, sizeof(*out));
    out->prompt_eval_count = S.n_prompt - S.n_shared;      // the evaluated tokens
    out->eval_count = S.produced;
    out->prompt_eval_duration_ns = S.prefill_ns;
    out->eval_duration_ns = S.eval_ns;
    out->total_duration_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count() - S.t_open_ns;
    out->load_duration_ns = load_ns_;
    out->done_reason = S.stopped ? 0 : 1;
    out->kernel_launches = S.launches;
    return {};
}

Status Engine::seq_logits(int slot, float* out, int n_vocab) {
    CU(cudaSetDevice(device_));
    if (slot < 0 || slot >= (int)slots_.size() || !slots_[slot].open || n_vocab != n_vocab_ || !out) return failb(GL_ERR_INVALID, "seq_logits: bad argument");
    const SeqSlot& S = slots_[slot];
    // the first token is drawn at gl_seq_open (its logits are kept per slot); later ones from the sequence's row of the last step
    const float* src = S.last_row < 0 ? bfirst_logits_ + (size_t)slot * n_vocab_ : blogits_ + (size_t)S.last_row * n_vocab_;
    CU(cudaMemcpy(out, src, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost));
    return {};
}

// every launch of one batched step, for `bucket` rows; all pointers are fixed, the composition is read from bctl_ / bst_
Status Engine::enqueue_batch_step(cudaStream_t s, int bucket, bool penalised, bool masked, int* n_launch) {
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_, ldq = qd + 2 * kvd;
    const float scale = 1.0f / std::sqrt((float)hd_);
    int nl = 0;
    // the GEMMs read the QUANTISED weights (4.5 / 6.56 bits per weight, unpacked inside the kernel) for up to 64 rows; the
    // resident 16-bit copy otherwise (models with other tensor types, or 65..128 rows, where the step is tensor-bound anyway)
    const bool use_q = have_qg_ && bucket <= 64;
    const int nb = std::max(16, bucket);
    auto linear = [&](const void* a, const void* w, void* c, int n, int k, int ldc, int epi, const QGemmWeights* qw,
                      const QGemmNorm* norm = nullptr) -> cudaError_t {
        if (use_q) {
            ++nl;
            return qgemm_launch(*qw, (const __half*)a, MAX_BATCH, nb, c, ldc, epi, qpartial_, sm_count_, s, norm);
        }
        GemmParams g{};
        g.a = a; g.b = w; g.c = c; g.m = bucket; g.n = n; g.k = k; g.lda = k; g.ldb = k; g.ldc = ldc;
        g.batch = 1; g.b_batch_div = 1; g.epi = epi;
        ++nl;
        return gemm_tc5_supported(g) ? gemm_tc5_launch(g, MAX_BATCH, false, s) : gemm_tn_launch(g, false, s);
    };
    // RMSNorm folded into the GEMMs around it (qgemm.h, QGemmNorm): the residual-add GEMMs write the next GEMM's activation rows
    // (x * gamma / 16, fp16) and the per-slice sums of squares; the GEMM behind the norm scales its accumulator by 16 / rms.
    // Only the first norm of the step (behind the embedding gather) is still a kernel.
    static const bool fold_env = []() { const char* e = getenv("GL_BATCH_FOLD_NORM"); return !(e && e[0] == '0'); }();
    const bool fold = use_q && fold_env && bssq_[0] != nullptr && qgemm_uses_cluster(qlayers_[0].o, nb, GEMM_EPI_ADD_F32, sm_count_) &&
                      qgemm_uses_cluster(qlayers_[0].down, nb, GEMM_EPI_ADD_F32, sm_count_) && n_embd_ / 128 * 4 <= BSSQ_PARTS;
    const int ssq_parts = n_embd_ / 128 * 4;
    auto produce = [&](const float* gamma, float* ssq) {
        QGemmNorm nm{};
        nm.gamma_next = gamma; nm.xg_out = bxn16_; nm.ldxg = n_embd_; nm.ssq_out = ssq;
        return nm;
    };
    auto consume = [&](const float* ssq) {
        QGemmNorm nm{};
        nm.ssq_in = ssq; nm.ssq_parts = ssq_parts; nm.n_norm = n_embd_; nm.eps = eps_;
        return nm;
    };
    CU(batch_gather_tokens_launch(bctl_, bst_, bids_, bucket, s)); ++nl;
    CU(embed_rows_launch(tok_embd_.w, tok_embd_.type, n_embd_, tok_embd_.row_stride, bids_, bucket, bx_, s)); ++nl;
    const int splits = attn_splits_for(bucket, n_kv_, sm_count_);
    const bool fuse_rope = batch_attn_fuses_rope(hd_);
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = kcache_ + (size_t)il * kv_layer_elems_;
        __half* vc = vcache_ + (size_t)il * kv_layer_elems_;
        const bool folded_in = fold && il > 0;                           // this layer's attn_norm came out of the ffn_down GEMM before
        if (!folded_in) { CU(batch_rmsnorm_launch(bx_, L.attn_norm, bucket, n_embd_, eps_, bxn16_, s)); ++nl; }
        {
            const QGemmNorm nm = consume(bssq_[1]);
            CU(linear(bxn16_, L.wqkv16, bqkv_, ldq, n_embd_, ldq, GEMM_EPI_F32, use_q ? &qlayers_[il].qkv : nullptr, folded_in ? &nm : nullptr));
        }
        BatchAttnParams a{};
        if (fuse_rope) {        // the attention kernel rotates q itself and appends the step's K / V rows (batch.h)
            a.q = nullptr; a.qkv = bqkv_; a.ld_qkv = ldq; a.cos_t = rope_cos_; a.sin_t = rope_sin_;
        } else {
            CU(batch_rope_kv_launch(bqkv_, bucket, bctl_, bst_, btables_, n_pages_, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, bq_, kc, vc, s)); ++nl;
            a.q = bq_;
        }
        a.k_cache = kc; a.v_cache = vc; a.tables = btables_; a.table_stride = n_pages_; a.st = bst_; a.ctl = bctl_;
        a.out16 = battn16_; a.part_o = bpart_o_; a.part_ml = bpart_ml_; a.counters = bcounters_;
        a.n_head = n_head_; a.n_kv_heads = n_kv_; a.head_dim = hd_; a.n_splits = splits; a.scale = scale;
        CU(batch_attn_launch(a, bucket, s)); ++nl;
        {
            const QGemmNorm nm = produce(L.ffn_norm, bssq_[0]);
            CU(linear(battn16_, L.wo16, bx_, n_embd_, qd, n_embd_, GEMM_EPI_ADD_F32, use_q ? &qlayers_[il].o : nullptr, fold ? &nm : nullptr));
        }
        if (!fold) { CU(batch_rmsnorm_launch(bx_, L.ffn_norm, bucket, n_embd_, eps_, bxn16_, s)); ++nl; }
        {
            const QGemmNorm nm = consume(bssq_[0]);
            CU(linear(bxn16_, L.wgu16, bh16_, 2 * n_ff_, n_embd_, n_ff_, GEMM_EPI_SILU, use_q ? &qlayers_[il].gu : nullptr, fold ? &nm : nullptr));
        }
        {
            const QGemmNorm nm = produce(il + 1 < n_layer_ ? layers_[il + 1].attn_norm : output_norm_, bssq_[1]);
            CU(linear(bh16_, L.wd16, bx_, n_embd_, n_ff_, n_embd_, GEMM_EPI_ADD_F32, use_q ? &qlayers_[il].down : nullptr, fold ? &nm : nullptr));
        }
    }
    if (!fold) { CU(batch_rmsnorm_launch(bx_, output_norm_, bucket, n_embd_, eps_, bxn16_, s)); ++nl; }
    {
        const QGemmNorm nm = consume(bssq_[1]);
        CU(linear(bxn16_, head16_, blogits_, n_vocab_, n_embd_, n_vocab_, GEMM_EPI_F32, use_q ? &qhead_ : nullptr, fold ? &nm : nullptr));
    }
    // repetition penalties, then the grammar mask, of the rows that have them: each only in the variants used for steps in which
    // some row needs it
    CU(enqueue_pre_draw(s, bucket, penalised, masked, nullptr, &nl));
    CU(batch_sample_greedy_launch(blogits_, n_vocab_, bucket, bctl_, bst_, bout_ids_, bout_lp_, max_out_, bsample_scratch_, s)); ++nl;
    if (n_launch) *n_launch = nl;
    return {};
}

// One un-captured launch of the penalty / mask kernels a new variant adds, on a composition of no rows (every CTA leaves at once;
// a launch on the real rows would advance their automata), validates their configuration outside stream capture, where an
// error has a name; the step's composition is restored.
Status Engine::check_pre_draw(int variant) {
    const int todo = variant & ~batch_checked_;
    if (!todo) return {};
    BatchCtl none{};
    CU(cudaMemcpyAsync(bctl_, &none, sizeof(int), cudaMemcpyHostToDevice, stream_));
    cudaError_t e0 = enqueue_pre_draw(stream_, 8, todo & 1, todo & 2);
    if (e0 == cudaSuccess) e0 = cudaStreamSynchronize(stream_);
    BatchCtl h{};
    h.n_rows = (int)last_rows_.size();
    for (int r = 0; r < h.n_rows; ++r) h.row_slot[r] = last_rows_[r];
    CU(cudaMemcpyAsync(bctl_, &h, sizeof(h), cudaMemcpyHostToDevice, stream_));
    CU(cudaStreamSynchronize(stream_));                       // h is on the stack
    CU(e0);
    batch_checked_ |= todo;
    return {};
}

// penalised / masked: the variants with the penalty kernel / the mask kernel (up to four captured steps per bucket);
// batch_launches_ counts the plain one
Status Engine::run_batch_graph(int bucket, bool penalised, bool masked) {
    if (penalised && !bpen_counts_) return failb(GL_ERR_INVALID, "batched step: no penalty state");
    if (masked && !sch_) return failb(GL_ERR_INVALID, "batched step: no mask state");
    const int variant = (penalised ? 1 : 0) | (masked ? 2 : 0);
    const int extra = (penalised ? 1 : 0) + (masked ? 1 : 0);
    if (!use_graph_) {
        int nl = 0;
        ST(enqueue_batch_step(stream_, bucket, penalised, masked, &nl));
        batch_launches_ = nl - extra;
        return {};
    }
    cudaGraphExec_t& ge = g_batch_[bucket_index(bucket)][variant];
    if (!ge) {
        ST(check_pre_draw(variant));
        cudaGraph_t g = nullptr;
        int nl = 0;
        CU(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
        Status st = enqueue_batch_step(stream_, bucket, penalised, masked, &nl);
        cudaError_t e = cudaStreamEndCapture(stream_, &g);
        if (!st.ok()) { if (g) cudaGraphDestroy(g); return st; }
        if (e != cudaSuccess) return failb(GL_ERR_CUDA, std::string("batched step: graph capture: ") + cudaGetErrorString(e));
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return failb(GL_ERR_CUDA, std::string("batched step: graph instantiate: ") + cudaGetErrorString(e));
        batch_launches_ = nl - extra;
    }
    CU(cudaGraphLaunch(ge, stream_));
    return {};
}

// One token for every open, unfinished sequence.  Entries: (slot, id, logprob, done) -- see include/gridllm_native.h.
Status Engine::batch_step(int32_t* out_slots, int32_t* out_ids, float* out_lps, int32_t* out_done, int cap, int* n_out) {
    CU(cudaSetDevice(device_));
    if (!n_out) return failb(GL_ERR_INVALID, "batch_step: null argument");
    *n_out = 0;
    if (slots_.empty()) return {};
    int n = 0;
    auto emit = [&](int slot, int32_t id, float lp, int done) {
        if (out_slots) out_slots[n] = slot;
        if (out_ids) out_ids[n] = id;
        if (out_lps) out_lps[n] = lp;
        if (out_done) out_done[n] = done;
        ++n;
    };
    int n_first = 0, n_rows = 0;
    for (int s = 0; s < max_batch_; ++s) {
        const SeqSlot& S = slots_[s];
        if (!S.open) continue;
        if (S.first_pending) ++n_first;
        else if (!S.done) ++n_rows;
    }
    if (n_first + n_rows > cap) return failb(GL_ERR_INVALID, "batch_step: output capacity too small");
    std::vector<int> rows;
    for (int s = 0; s < max_batch_; ++s) {
        SeqSlot& S = slots_[s];
        if (!S.open || (S.done && !S.first_pending)) continue;
        if (S.first_pending) {                       // the token drawn at gl_seq_open
            S.first_pending = false;
            if (S.done) { emit(s, -1, 0.f, 1); continue; }
            S.produced = 1;
            if (S.produced >= S.n_pred) S.done = true;
            emit(s, S.last_token, S.first_lp, S.done ? 1 : 0);
            continue;
        }
        rows.push_back(s);
    }
    const int B = (int)rows.size();
    if (B == 0) { *n_out = n; return {}; }
    const int bucket = bucket_of(B);
    if (rows != last_rows_) {                        // composition changed: one small copy, the captured step is unchanged
        BatchCtl h{};
        h.n_rows = B;
        for (int r = 0; r < B; ++r) h.row_slot[r] = rows[r];
        CU(cudaMemcpyAsync(bctl_, &h, sizeof(h), cudaMemcpyHostToDevice, stream_));      // pageable source: staged before the call returns
        last_rows_ = rows;
    }
    last_bucket_ = bucket;
    bool penalised = false, masked = false;         // the step with the penalty / mask kernel only when some row needs it
    for (int r = 0; r < B; ++r) {
        penalised = penalised || slots_[rows[r]].plan.penalised;
        masked = masked || slots_[rows[r]].plan.masked;
    }
    CU(cudaEventRecord(ev_[2], stream_));
    // context shift: every row whose step would write position W first shifts its rows, all of them in one launch.  The
    // captured step, BatchCtl and the page tables stay as they are: the position is read on the device.
    std::vector<KvShiftSeq> shifts;
    for (int r = 0; r < B; ++r) {
        SeqSlot& S = slots_[rows[r]];
        if (!S.shift_on || S.pos < n_ctx_) continue;
        const int d = shift_discard(n_ctx_, S.keep);
        shifts.push_back(KvShiftSeq{btables_ + (size_t)rows[r] * n_pages_, S.keep, d, shift_rows(n_ctx_, S.keep, d), bst_ + rows[r]});
        S.pos -= d;
    }
    ST(launch_shift(shifts));
    ST(run_batch_graph(bucket, penalised, masked));
    const int step_launches = batch_launches_ + (penalised ? 1 : 0) + (masked ? 1 : 0) + 1 + (shifts.empty() ? 0 : 1);
    for (int r = 0; r < B; ++r) {                    // sampled rows: the seeded top-k / top-p sampler of the single-sequence path
        const int slot = rows[r];
        if (slots_[slot].plan.sampler == 0) continue;
        SampleParams sp{blogits_ + (size_t)r * n_vocab_, n_vocab_, bst_ + slot, bout_ids_ + (size_t)slot * max_out_, bout_lp_ + (size_t)slot * max_out_,
                        nullptr, max_out_, sample_scratch_, topk_scratch_};
        CU(sample_topk_launch(sp, slots_[slot].plan.sampler == 1, false, stream_));
    }
    CU(batch_collect_launch(bctl_, bst_, bout_lp_, max_out_, bout_, bucket, stream_));
    CU(cudaEventRecord(ev_[3], stream_));
    std::vector<BatchOut> ho(B);
    CU(cudaMemcpyAsync(ho.data(), bout_, sizeof(BatchOut) * B, cudaMemcpyDeviceToHost, stream_));
    CU(cudaStreamSynchronize(stream_));
    float step_ms = 0.f;
    cudaEventElapsedTime(&step_ms, ev_[2], ev_[3]);
    bc_[0] += 1; bc_[1] += (uint64_t)B; bc_[2] += (uint64_t)(step_ms * 1e6); bc_[6] += (uint64_t)step_launches;
    for (int r = 0; r < B; ++r) {
        SeqSlot& S = slots_[rows[r]];
        S.last_row = r;
        S.eval_ns += (int64_t)(step_ms * 1e6);
        S.launches += step_launches;
        if (ho[r].done) {                            // the token just drawn is a stop token: not part of the output
            S.done = true;
            S.stopped = true;
            emit(rows[r], -1, 0.f, 1);
            continue;
        }
        S.last_token = ho[r].token;
        S.pos = ho[r].pos;
        ++S.produced;
        if (S.produced >= S.n_pred) S.done = true;
        emit(rows[r], ho[r].token, ho[r].logprob, S.done ? 1 : 0);
    }
    *n_out = n;
    return {};
}

// Device time of one batched step with `batch` synthetic sequences at context ctx_len (bench roofline line).  The sequences are
// real slots whose KV pages hold whatever is resident (timing does not depend on the values); they are closed afterwards.
Status Engine::time_batch_step(int batch, int ctx_len, int iters, float* ms, int* launches, uint64_t* wbytes) {
    CU(cudaSetDevice(device_));
    ST(ensure_batch_state());
    if (batch < 1 || batch > max_batch_ || ctx_len < 1 || iters < 1) return failb(GL_ERR_INVALID, "time_batch_step: bad arguments");
    for (const SeqSlot& S : slots_)
        if (S.open) return failb(GL_ERR_INVALID, "time_batch_step: close the open sequences first");
    const int need_tokens = ctx_len + iters + 8;
    if (need_tokens > n_ctx_) return failb(GL_ERR_CONTEXT, "time_batch_step: context too long for this engine");
    const int need = (need_tokens + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    if ((size_t)need * batch > (size_t)pages_.available()) return failb(GL_ERR_NOMEM, "time_batch_step: KV page pool too small for this batch");
    std::vector<StepState> hst(batch);
    std::vector<int> rows(batch);
    for (int b = 0; b < batch; ++b) {
        SeqSlot& S = slots_[b];
        S = SeqSlot{};
        S.open = true;
        pages_.alloc(need, S.pages);                 // never indexed: the pages go back to the free list
        CU(cudaMemcpyAsync(btables_ + (size_t)b * n_pages_, S.pages.data(), S.pages.size() * 4, cudaMemcpyHostToDevice, stream_));
        StepState h{};
        h.pos = ctx_len - 1; h.token = (7 + 13 * b) % n_vocab_; h.ignore_eos = 1; h.top_p = 1.f;
        hst[b] = h;
        rows[b] = b;
    }
    const int bucket = bucket_of(batch);
    BatchCtl hc{};
    hc.n_rows = batch;
    for (int b = 0; b < batch; ++b) hc.row_slot[b] = b;
    CU(cudaMemcpyAsync(bctl_, &hc, sizeof(hc), cudaMemcpyHostToDevice, stream_));
    last_rows_ = rows;
    auto reset = [&]() -> cudaError_t { return cudaMemcpyAsync(bst_, hst.data(), sizeof(StepState) * batch, cudaMemcpyHostToDevice, stream_); };
    CU(reset());
    Status rs;
    for (int i = 0; i < 3 && rs.ok(); ++i) rs = run_batch_graph(bucket, false, false);  // warm-up (captures the bucket's graph)
    if (rs.ok()) {
        cudaError_t e = reset();
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream_);                 // hst must outlive the copy
        if (e == cudaSuccess) e = cudaEventRecord(ev_[0], stream_);
        for (int i = 0; i < iters && rs.ok() && e == cudaSuccess; ++i) rs = run_batch_graph(bucket, false, false);
        if (e == cudaSuccess) e = cudaEventRecord(ev_[1], stream_);
        if (e == cudaSuccess) e = cudaEventSynchronize(ev_[1]);
        if (rs.ok() && e != cudaSuccess) rs = failb(GL_ERR_CUDA, std::string("time_batch_step: ") + cudaGetErrorString(e));
    }
    cudaStreamSynchronize(stream_);
    for (int b = 0; b < batch; ++b) {
        release_pages(slots_[b].pages);
        slots_[b] = SeqSlot{};
    }
    last_rows_.clear();
    ST(rs);
    float t_ms = 0.f;
    cudaEventElapsedTime(&t_ms, ev_[0], ev_[1]);
    if (ms) *ms = t_ms / iters;
    if (launches) *launches = batch_launches_;
    if (wbytes) {
        // bytes of weights one batched step reads: the quantised matrices (= the GGUF bytes), or the resident 16-bit matrices of
        // every layer + the 16-bit lm_head + norms
        const uint64_t per_layer = ((uint64_t)(n_head_ * hd_ + 2 * n_kv_ * hd_) * n_embd_ + (uint64_t)n_embd_ * n_head_ * hd_ +
                                    (uint64_t)2 * n_ff_ * n_embd_ + (uint64_t)n_embd_ * n_ff_) * 2;
        *wbytes = (have_qg_ && bucket <= 64) ? decode_bytes_
                                             : per_layer * n_layer_ + (uint64_t)n_vocab_ * n_embd_ * 2 + (uint64_t)(2 * n_layer_ + 1) * n_embd_ * 4;
    }
    return {};
}

}  // namespace gl
