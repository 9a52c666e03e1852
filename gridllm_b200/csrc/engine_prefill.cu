// Engine: batched tensor-core prefill driver (kernels in prefill.cu).  One pass over the layers with
// a [T x n_embd] activation matrix; writes the fp16 KV pages the decode path then reads.
#include <algorithm>
#include <cmath>

#include "engine.h"

namespace gl {

namespace {
Status failp(int code, const std::string& m) { return Status{code, m}; }
#define CU(expr)                                                                                  \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) return failp(GL_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
#define ST(expr)                 \
    do {                         \
        Status _s = (expr);      \
        if (!_s.ok()) return _s; \
    } while (0)
}  // namespace

// The prompt pass's 16-bit layer matrices (prefill_weights.h).  Resident: a copy of every layer matrix, dequantised on the GPU
// from the engine layouts -- 2 bytes/weight (14 GB for Llama-3-8B) of the 80 GB HBM buys a prefill that never touches the 4-bit
// decode layout.  Streamed (the copy does not fit, e.g. 137 GB for a 70B): one staging buffer the size of the largest operand,
// filled before each GEMM by prompt_operand.  fp16 is used for every model type (what ggml's CUDA backend also does for
// batched matmuls [external]); bf16 weights convert to fp16 exactly within fp16's normal range.
Status Engine::build_prefill_weights(int request) {
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_;
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t copy = prefill_copy_bytes(n_layer_, n_embd_, n_head_, n_kv_, hd_, n_ff_);
    const int src = prefill_weights_source(prefill_mode_, request, copy, free_b);
    if (src < 0)
        return failp(GL_ERR_NOMEM, "GL_PREFILL_WEIGHTS=1: the resident 16-bit copy of the layer matrices needs " + std::to_string(copy >> 20) +
                                       " MiB + 4096 MiB spare, " + std::to_string(free_b >> 20) + " MiB of HBM are free");
    prefill_w_ = src;
    if (src == PREFILL_W_NONE) return {};
    if (n_ff_ % 8) return failp(GL_ERR_UNSUPPORTED, "n_ff must be a multiple of 8 for the batched prefill");
    auto alloc = [&](void** p, size_t elems) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, elems * 2);
        if (e == cudaSuccess) allocs_.push_back(*p);
        return e;
    };
    if (src == PREFILL_W_STREAMED) {
        CU(alloc(&w16_stage_, prefill_stage_bytes(n_embd_, n_head_, n_kv_, hd_, n_ff_) / 2));
        return {};
    }
    for (int il = 0; il < n_layer_; ++il) {
        LayerWeights& L = layers_[il];
        CU(alloc(&L.wqkv16, (size_t)(qd + 2 * kvd) * n_embd_));
        CU(alloc(&L.wo16, (size_t)n_embd_ * qd));
        CU(alloc(&L.wgu16, (size_t)2 * n_ff_ * n_embd_));
        CU(alloc(&L.wd16, (size_t)n_embd_ * n_ff_));
        ST(dequant_operand(L, OP_QKV, L.wqkv16));
        ST(dequant_operand(L, OP_O, L.wo16));
        ST(dequant_operand(L, OP_GU, L.wgu16));
        ST(dequant_operand(L, OP_DOWN, L.wd16));
    }
    CU(cudaStreamSynchronize(stream_));
    return {};
}

Status Engine::dequant_operand(const LayerWeights& L, PrefillOperand op, void* dst) {
    auto src = [](const DevMatrix& m, int row0, int interleave) {
        return DequantSrc{m.w, m.type, m.rows, m.row_stride, m.tile_rows, row0, interleave};
    };
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_;
    DequantOp d{};
    d.dst = dst;
    switch (op) {
        case OP_QKV: d.src[0] = src(L.wq, 0, 0); d.src[1] = src(L.wk, qd, 0); d.src[2] = src(L.wv, qd + kvd, 0); d.n_src = 3; d.cols = n_embd_; break;
        case OP_O: d.src[0] = src(L.wo, 0, 0); d.n_src = 1; d.cols = qd; break;
        case OP_GU: d.src[0] = src(L.wgate, 0, 1); d.src[1] = src(L.wup, 0, 2); d.n_src = 2; d.cols = n_embd_; break;
        case OP_DOWN: d.src[0] = src(L.wdown, 0, 0); d.n_src = 1; d.cols = n_ff_; break;
    }
    CU(dequant_launch(d, prefill_bf16_, stream_));
    return {};
}

Status Engine::prompt_operand(const LayerWeights& L, PrefillOperand op, const void** b, int* nl) {
    if (prefill_w_ == PREFILL_W_RESIDENT) {
        *b = op == OP_QKV ? L.wqkv16 : op == OP_O ? L.wo16 : op == OP_GU ? L.wgu16 : L.wd16;
        return {};
    }
    // stream order alone makes the reuse safe: the GEMM that read the previous operand precedes this launch on stream_
    ST(dequant_operand(L, op, w16_stage_));
    ++*nl;
    *b = w16_stage_;
    return {};
}

Status Engine::ensure_prefill_scratch(int t_pad) {
    if (t_pad <= pf_cap_) return {};
    CU(cudaStreamSynchronize(stream_));
    for (void* p : pf_allocs_) cudaFree(p);
    pf_allocs_.clear();
    pf_cap_ = 0;
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_;
    auto alloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess) { pf_allocs_.push_back(*p); e = cudaMemsetAsync(*p, 0, bytes, stream_); }
        return e;
    };
    const size_t T = (size_t)t_pad;
    CU(alloc((void**)&pf_x_, T * n_embd_ * 4));
    CU(alloc((void**)&pf_qkv_, T * (qd + 2 * kvd) * 4));
    if (!prefill_flash_) CU(alloc((void**)&pf_s_, (size_t)n_head_ * T * T * 4));      // scores exist in HBM on the three-launch path only
    CU(alloc((void**)&pf_xn_, T * n_embd_ * 2));
    CU(alloc((void**)&pf_attn_, T * qd * 2));
    CU(alloc((void**)&pf_h_, T * n_ff_ * 2));
    CU(alloc((void**)&pf_q_, T * qd * 2));
    CU(alloc((void**)&pf_k_, T * kvd * 2));
    CU(alloc((void**)&pf_vt_, (size_t)kvd * T * 2));
    if (!prefill_flash_) CU(alloc((void**)&pf_p_, (size_t)n_head_ * T * T * 2));
    pf_cap_ = t_pad;
    return {};
}

// Positions [pos0, pos0 + n) of the single sequence, in passes of at most PF_CHUNK rows: each pass is one segment
// {start 0, len, pos0 of the pass, page_table_}, so its K / V rows land in the pages before its attention reads them, and a
// pass that does not start at 0 attends to everything before it through the pages (the PAGED prompt attention).  A prompt of
// at most PF_CHUNK tokens from position 0 is the one pass it always was.
Status Engine::prefill_batched(int pos0, int n, int* n_launch) {
    int nl = 0;
    for (int c0 = 0; c0 < n; c0 += PF_CHUNK) {
        const int len = std::min(PF_CHUNK, n - c0);
        ST(prompt_pass({{0, len, pos0 + c0, page_table_}}, len, prompt_ids_ + pos0 + c0, &nl));
    }
    // hidden state of the last prompt token -> the decode path's x buffer (lm_head / sampler follow)
    const int last = (n - 1) % PF_CHUNK;
    CU(cudaMemcpyAsync(x_, pf_x_ + (size_t)last * n_embd_, (size_t)n_embd_ * 4, cudaMemcpyDeviceToDevice, stream_));
    if (n_launch) *n_launch += nl;
    last_prefill_launches_ = nl;
    return {};
}

// One pass over the layers for rows [0, t_rows) of the pf_* scratch.  The sequences share the linear layers -- one
// [t_rows x n_embd] activation matrix, every weight matrix read once per pass -- and each attends only to itself
// (block-diagonal causal attention), and to its positions before pos0 through its pages.  Two kinds of caller:
// prefill_batched and gl_embed's sequences longer than a pack run one sequence {0, n, pos0, page_table_} with t_rows = n <=
// PF_CHUNK; the packs of gl_embed and gl_seq_open_many start every sequence on a 128-row boundary and pass a 128-aligned
// t_rows.  Rows t_rows .. TP - 1 are padding that nothing reads back.
Status Engine::prompt_pass(const std::vector<PromptSeq>& seqs, int t_rows, const int* ids, int* n_launch) {
    if (!prefill_flash_)
        for (const PromptSeq& q : seqs)
            if (q.pos0 > 0) return failp(GL_ERR_UNSUPPORTED, "a prompt pass from a non-zero position needs the fused prompt attention");
    const int TP = (t_rows + 127) / 128 * 128;
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_, ldq = qd + 2 * kvd, grp = n_head_ / n_kv_;
    ST(ensure_prefill_scratch(TP));
    const int tp = pf_cap_;          // leading dimension of the [T_pad]-shaped scratch
    cudaStream_t s = stream_;
    const bool bf = prefill_bf16_;
    // gl_seq_open_many and the single sequence cache their K / V rows through their tables; embedding packs cache nothing
    const bool cached = std::any_of(seqs.begin(), seqs.end(), [](const PromptSeq& q) { return q.table != nullptr; });
    // one segment list per PF_MAX_SEGS sequences: one RoPE / split launch and one fused attention launch each
    std::vector<PrefillSegs> groups((seqs.size() + PF_MAX_SEGS - 1) / PF_MAX_SEGS, PrefillSegs{});
    for (size_t i = 0; i < seqs.size(); ++i) {
        PrefillSegs& g = groups[i / PF_MAX_SEGS];
        g.start[g.n] = seqs[i].start; g.len[g.n] = seqs[i].len; g.table[g.n] = seqs[i].table; g.pos0[g.n] = seqs[i].pos0;
        ++g.n;
    }
    int nl = 0;
    // linear layers: wgmma / TMA GEMM (prefill_tc5.cu); GL_PREFILL_TC5=0 keeps the mma.sync kernel for A/B runs
    auto linear = [&](const GemmParams& g) -> cudaError_t {
        if (prefill_tc5_ && gemm_tc5_supported(g)) return gemm_tc5_launch(g, tp, bf, s);
        return gemm_tn_launch(g, bf, s);
    };
    CU(embed_rows_launch(tok_embd_.w, tok_embd_.type, n_embd_, tok_embd_.row_stride, ids, t_rows, pf_x_, s)); ++nl;
    const float scale = 1.0f / std::sqrt((float)hd_);
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = cached ? kcache_ + (size_t)il * kv_layer_elems_ : nullptr;
        __half* vc = cached ? vcache_ + (size_t)il * kv_layer_elems_ : nullptr;
        CU(rmsnorm_rows_launch(pf_x_, L.attn_norm, t_rows, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        bool roped = false;
        {
            GemmParams g{};
            ST(prompt_operand(L, OP_QKV, &g.b, &nl));
            g.a = pf_xn_; g.c = pf_qkv_; g.m = t_rows; g.n = ldq; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = ldq;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_F32;
            if (prefill_flash_ && prefill_fuse_rope_ && prefill_tc5_ && groups.size() == 1) {
                // RoPE + split + cache append in the projection's own epilogue: the fp32 QKV matrix never exists (rows t_rows .. TP
                // of the normalised activations are zeros; the epilogue writes them as padding rows)
                RopeSplitArgs ra{rope_cos_, rope_sin_, pf_q_, pf_k_, pf_vt_, kc, vc, n_head_, n_kv_, hd_, tp, groups[0]};
                GemmParams gr = g;
                gr.epi = GEMM_EPI_ROPE_SPLIT; gr.rope = &ra; gr.m = TP;
                if (gemm_tc5_supported(gr)) { CU(gemm_tc5_launch(gr, tp, bf, s)); ++nl; roped = true; }
            }
            if (!roped) { CU(linear(g)); ++nl; }
        }
        if (prefill_flash_) {
            // (RoPE + split + cache append, then) ONE fused attention launch per segment list (prefill_attn.cu): scores stay on the SM
            for (size_t c = 0; c < groups.size(); ++c) {
                const PrefillSegs& segs = groups[c];
                if (!roped) {
                    // the kernel indexes rows of its list absolutely: shift the segment starts to the list's first row; the
                    // trailing rows of the pass are zeroed too
                    PrefillSegs rs = segs;
                    const int row_lo = segs.start[0];
                    int row_hi = c + 1 == groups.size() ? TP : row_lo;
                    for (int i = 0; i < rs.n; ++i) {
                        row_hi = std::max(row_hi, segs.start[i] + (segs.len[i] + 127) / 128 * 128);
                        rs.start[i] -= row_lo;
                    }
                    CU(rope_split_segs_launch(pf_qkv_ + (size_t)row_lo * ldq, row_hi - row_lo, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_ + (size_t)row_lo * qd,
                                              pf_k_ + (size_t)row_lo * kvd, pf_vt_ + row_lo, kc, vc, tp, rs, s)); ++nl;
                }
                CU(flash_prefill_launch(pf_q_, pf_k_, pf_vt_, (__half*)pf_attn_, segs, n_head_, n_kv_, hd_, tp, scale, kc, vc, s));
                ++nl;
            }
        } else {
            // the three-launch A/B path, per sequence (every pos0 is 0 here)
            for (const PromptSeq& q : seqs) {
                const int r0 = q.start, len = q.len, lp = (len + 127) / 128 * 128;
                // RoPE at positions 0..len-1 of THIS sequence; V^T columns r0.. of the pass-wide [kvd][tp] matrix
                CU(rope_split_launch(pf_qkv_ + (size_t)r0 * ldq, len, lp, 0, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_ + (size_t)r0 * qd,
                                     pf_k_ + (size_t)r0 * kvd, pf_vt_ + r0, kc, vc, q.table, tp, s)); ++nl;
                {   // S[h] = Q_h K_kvh^T, compact [n_head][lp][lp]
                    GemmParams g{};
                    g.a = pf_q_ + (size_t)r0 * qd; g.b = pf_k_ + (size_t)r0 * kvd; g.c = pf_s_; g.m = len; g.n = len; g.k = hd_; g.lda = qd; g.ldb = kvd; g.ldc = lp;
                    g.batch = n_head_; g.a_batch_stride = hd_; g.b_batch_stride = hd_; g.b_batch_div = grp; g.c_batch_stride = (long long)lp * lp;
                    g.epi = GEMM_EPI_F32; g.causal_skip = 1;
                    CU(gemm_tn_launch(g, false, s)); ++nl;
                }
                CU(softmax_causal_launch(pf_s_, n_head_, len, lp, scale, pf_p_, s)); ++nl;
                {   // O[:, h] = P[h] V_kvh   (B = V^T rows = head dims)
                    GemmParams g{};
                    g.a = pf_p_; g.b = pf_vt_ + r0; g.c = (__half*)pf_attn_ + (size_t)r0 * qd; g.m = len; g.n = hd_; g.k = lp; g.lda = lp; g.ldb = tp; g.ldc = qd;
                    g.batch = n_head_; g.a_batch_stride = (long long)lp * lp; g.b_batch_stride = (long long)hd_ * tp; g.b_batch_div = grp; g.c_batch_stride = hd_;
                    g.epi = GEMM_EPI_T16; g.causal_k = 1;
                    CU(gemm_tn_launch(g, false, s)); ++nl;
                }
            }
        }
        {
            GemmParams g{};
            ST(prompt_operand(L, OP_O, &g.b, &nl));
            g.a = pf_attn_; g.c = pf_x_; g.m = t_rows; g.n = n_embd_; g.k = qd; g.lda = qd; g.ldb = qd; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
        CU(rmsnorm_rows_launch(pf_x_, L.ffn_norm, t_rows, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        {
            GemmParams g{};
            ST(prompt_operand(L, OP_GU, &g.b, &nl));
            g.a = pf_xn_; g.c = pf_h_; g.m = t_rows; g.n = 2 * n_ff_; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = n_ff_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_SILU;
            CU(linear(g)); ++nl;
        }
        {
            GemmParams g{};
            ST(prompt_operand(L, OP_DOWN, &g.b, &nl));
            g.a = pf_h_; g.c = pf_x_; g.m = t_rows; g.n = n_embd_; g.k = n_ff_; g.lda = n_ff_; g.ldb = n_ff_; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
    }
    if (n_launch) *n_launch += nl;
    return {};
}

Status Engine::ensure_pack_buffers() {
    if (pk_ids_) return {};
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess) allocs_.push_back(*p);
        return e;
    };
    CU(dalloc((void**)&pk_ids_, (size_t)EMB_PACK_TOKENS * 4));
    CU(dalloc((void**)&emb_pooled_, (size_t)n_embd_ * 4));
    CU(dalloc((void**)&emb_rstd_, (size_t)std::max(EMB_PACK_TOKENS, n_ctx_) * 4));
    return {};
}

}  // namespace gl
