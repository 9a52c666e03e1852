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

// Resident 16-bit copy of every layer matrix, dequantised on the GPU from the engine layouts.
// 2 bytes/weight (16 GB for Llama-3-8B) of the 80 GB HBM buys a prefill that never touches the
// 4-bit decode layout.  fp16 is used for every model type (what ggml's CUDA backend also does for
// batched matmuls [external]); bf16 weights convert to fp16 exactly within fp16's normal range.
Status Engine::build_prefill_weights() {
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_;
    const size_t per_layer = ((size_t)(qd + 2 * kvd) * n_embd_ + (size_t)n_embd_ * qd + (size_t)2 * n_ff_ * n_embd_ + (size_t)n_embd_ * n_ff_) * 2;
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (per_layer * n_layer_ + ((size_t)4 << 30) > free_b) {
        have_w16_ = false;          // not enough HBM: prompts fall back to the sequential path (still on the GPU)
        return {};
    }
    auto alloc = [&](void** p, size_t elems) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, elems * 2);
        if (e == cudaSuccess) allocs_.push_back(*p);
        return e;
    };
    for (int il = 0; il < n_layer_; ++il) {
        LayerWeights& L = layers_[il];
        CU(alloc(&L.wqkv16, (size_t)(qd + 2 * kvd) * n_embd_));
        CU(alloc(&L.wo16, (size_t)n_embd_ * qd));
        CU(alloc(&L.wgu16, (size_t)2 * n_ff_ * n_embd_));
        CU(alloc(&L.wd16, (size_t)n_embd_ * n_ff_));
        if (n_ff_ % 8) return failp(GL_ERR_UNSUPPORTED, "n_ff must be a multiple of 8 for the batched prefill");
        CU(dequant_rows_launch(L.wq.w, L.wq.type, L.wq.rows, L.wq.cols, L.wq.row_stride, L.wq.tile_rows, L.wqkv16, n_embd_, 0, 0, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wk.w, L.wk.type, L.wk.rows, L.wk.cols, L.wk.row_stride, L.wk.tile_rows, L.wqkv16, n_embd_, qd, 0, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wv.w, L.wv.type, L.wv.rows, L.wv.cols, L.wv.row_stride, L.wv.tile_rows, L.wqkv16, n_embd_, qd + kvd, 0, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wo.w, L.wo.type, L.wo.rows, L.wo.cols, L.wo.row_stride, L.wo.tile_rows, L.wo16, qd, 0, 0, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wgate.w, L.wgate.type, L.wgate.rows, L.wgate.cols, L.wgate.row_stride, L.wgate.tile_rows, L.wgu16, n_embd_, 0, 1, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wup.w, L.wup.type, L.wup.rows, L.wup.cols, L.wup.row_stride, L.wup.tile_rows, L.wgu16, n_embd_, 0, 2, prefill_bf16_, stream_));
        CU(dequant_rows_launch(L.wdown.w, L.wdown.type, L.wdown.rows, L.wdown.cols, L.wdown.row_stride, L.wdown.tile_rows, L.wd16, n_ff_, 0, 0, prefill_bf16_, stream_));
    }
    CU(cudaStreamSynchronize(stream_));
    have_w16_ = true;
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

Status Engine::prefill_batched(int n, int* n_launch) {
    const int T = n, TP = (n + 127) / 128 * 128;
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_, ldq = qd + 2 * kvd, grp = n_head_ / n_kv_;
    ST(ensure_prefill_scratch(TP));
    const int tp = pf_cap_;          // leading dimension of the [T_pad]-shaped scratch
    cudaStream_t s = stream_;
    const bool bf = prefill_bf16_;
    int nl = 0;
    // linear layers: wgmma / TMA GEMM (prefill_tc5.cu); GL_PREFILL_TC5=0 keeps the mma.sync kernel for A/B runs
    auto linear = [&](const GemmParams& g) -> cudaError_t {
        if (prefill_tc5_ && gemm_tc5_supported(g)) return gemm_tc5_launch(g, tp, bf, s);
        return gemm_tn_launch(g, bf, s);
    };
    CU(embed_rows_launch(tok_embd_.w, tok_embd_.type, n_embd_, tok_embd_.row_stride, prompt_ids_, T, pf_x_, s)); ++nl;
    const float scale = 1.0f / std::sqrt((float)hd_);
    PrefillSegs segs{};
    segs.n = 1; segs.start[0] = 0; segs.len[0] = T; segs.table[0] = page_table_;
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = kcache_ + (size_t)il * kv_layer_elems_;
        __half* vc = vcache_ + (size_t)il * kv_layer_elems_;
        CU(rmsnorm_rows_launch(pf_x_, L.attn_norm, T, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        bool roped = false;
        {
            GemmParams g{};
            g.a = pf_xn_; g.b = L.wqkv16; g.c = pf_qkv_; g.m = T; g.n = ldq; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = ldq;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_F32;
            RopeSplitArgs ra{rope_cos_, rope_sin_, pf_q_, pf_k_, pf_vt_, kc, vc, n_head_, n_kv_, hd_, tp, segs};
            if (prefill_flash_ && prefill_fuse_rope_ && prefill_tc5_) {
                // RoPE + split + cache append in the projection's own epilogue: the fp32 QKV matrix never exists (rows T .. TP of
                // the normalised activations are zeros; the epilogue writes them as padding rows)
                GemmParams gr = g;
                gr.epi = GEMM_EPI_ROPE_SPLIT; gr.rope = &ra; gr.m = TP;
                if (gemm_tc5_supported(gr)) { CU(gemm_tc5_launch(gr, tp, bf, s)); ++nl; roped = true; }
            }
            if (!roped) { CU(linear(g)); ++nl; }
        }
        if (prefill_flash_) {
            // (RoPE + split + cache append, then) ONE fused attention launch (prefill_attn.cu): scores stay on the SM
            if (!roped) { CU(rope_split_segs_launch(pf_qkv_, TP, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_, pf_k_, pf_vt_, kc, vc, tp, segs, s)); ++nl; }
            CU(flash_prefill_launch(pf_q_, pf_k_, pf_vt_, (__half*)pf_attn_, segs, n_head_, n_kv_, hd_, tp, scale, s));
            ++nl;
        } else {
            CU(rope_split_launch(pf_qkv_, T, tp, 0, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_, pf_k_, pf_vt_, kc, vc, page_table_, tp, s)); ++nl;
            {   // S[h] = Q_h K_kvh^T
                GemmParams g{};
                g.a = pf_q_; g.b = pf_k_; g.c = pf_s_; g.m = T; g.n = T; g.k = hd_; g.lda = qd; g.ldb = kvd; g.ldc = tp;
                g.batch = n_head_; g.a_batch_stride = hd_; g.b_batch_stride = hd_; g.b_batch_div = grp; g.c_batch_stride = (long long)tp * tp;
                g.epi = GEMM_EPI_F32; g.causal_skip = 1;
                CU(gemm_tn_launch(g, false, s)); ++nl;
            }
            CU(softmax_causal_launch(pf_s_, n_head_, T, tp, scale, pf_p_, s)); ++nl;
            {   // O[:, h] = P[h] V_kvh   (B = V^T rows = head dims)
                GemmParams g{};
                g.a = pf_p_; g.b = pf_vt_; g.c = pf_attn_; g.m = T; g.n = hd_; g.k = TP; g.lda = tp; g.ldb = tp; g.ldc = qd;
                g.batch = n_head_; g.a_batch_stride = (long long)tp * tp; g.b_batch_stride = (long long)hd_ * tp; g.b_batch_div = grp; g.c_batch_stride = hd_;
                g.epi = GEMM_EPI_T16; g.causal_k = 1;
                CU(gemm_tn_launch(g, false, s)); ++nl;
            }
        }
        {
            GemmParams g{};
            g.a = pf_attn_; g.b = L.wo16; g.c = pf_x_; g.m = T; g.n = n_embd_; g.k = qd; g.lda = qd; g.ldb = qd; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
        CU(rmsnorm_rows_launch(pf_x_, L.ffn_norm, T, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        {
            GemmParams g{};
            g.a = pf_xn_; g.b = L.wgu16; g.c = pf_h_; g.m = T; g.n = 2 * n_ff_; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = n_ff_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_SILU;
            CU(linear(g)); ++nl;
        }
        {
            GemmParams g{};
            g.a = pf_h_; g.b = L.wd16; g.c = pf_x_; g.m = T; g.n = n_embd_; g.k = n_ff_; g.lda = n_ff_; g.ldb = n_ff_; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
    }
    // hidden state of the last prompt token -> the decode path's x buffer (lm_head / sampler follow)
    CU(cudaMemcpyAsync(x_, pf_x_ + (size_t)(T - 1) * n_embd_, (size_t)n_embd_ * 4, cudaMemcpyDeviceToDevice, s));
    if (n_launch) *n_launch += nl;
    last_prefill_launches_ = nl;
    return {};
}

// Packed prompt pass for embeddings (generateEmbedding with `input: string[]`, /root/reference/server/src/routes/ollama.ts:574-643 ->
// client/src/services/OllamaService.ts:619-636): the sequences of a call share the linear layers -- one [T x n_embd] activation
// matrix, T = all their tokens, every weight matrix read once per PACK instead of once per sequence -- and attend only inside
// themselves (block-diagonal causal attention: the three attention launches run per sequence on its own rows).  Nothing is
// cached: an embedding has no decode phase.  Hidden states end up in pf_x_ for pooling.
Status Engine::prefill_packed(const std::vector<int>& starts, const std::vector<int>& lens, int t_rows, int* n_launch,
                              const std::vector<const int*>* tables) {
    const int TP = (t_rows + 127) / 128 * 128;
    const int qd = n_head_ * hd_, kvd = n_kv_ * hd_, ldq = qd + 2 * kvd, grp = n_head_ / n_kv_;
    ST(ensure_prefill_scratch(std::max(TP, 128)));
    const int tp = pf_cap_;
    cudaStream_t s = stream_;
    const bool bf = prefill_bf16_;
    int nl = 0;
    auto linear = [&](const GemmParams& g) -> cudaError_t {
        if (prefill_tc5_ && gemm_tc5_supported(g)) return gemm_tc5_launch(g, tp, bf, s);
        return gemm_tn_launch(g, bf, s);
    };
    CU(embed_rows_launch(tok_embd_.w, tok_embd_.type, n_embd_, tok_embd_.row_stride, pk_ids_, TP, pf_x_, s)); ++nl;
    const float scale = 1.0f / std::sqrt((float)hd_);
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = tables ? kcache_ + (size_t)il * kv_layer_elems_ : nullptr;      // gl_seq_open_many: each sequence's K / V rows go
        __half* vc = tables ? vcache_ + (size_t)il * kv_layer_elems_ : nullptr;      // to its own pages; embeddings cache nothing
        CU(rmsnorm_rows_launch(pf_x_, L.attn_norm, TP, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        bool roped = false;
        {
            GemmParams g{};
            g.a = pf_xn_; g.b = L.wqkv16; g.c = pf_qkv_; g.m = TP; g.n = ldq; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = ldq;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_F32;
            RopeSplitArgs ra{rope_cos_, rope_sin_, pf_q_, pf_k_, pf_vt_, kc, vc, n_head_, n_kv_, hd_, tp, {}};
            if (prefill_flash_ && prefill_fuse_rope_ && prefill_tc5_ && starts.size() <= (size_t)PF_MAX_SEGS) {
                ra.segs.n = (int)starts.size();
                for (int i = 0; i < ra.segs.n; ++i) {
                    ra.segs.start[i] = starts[i];
                    ra.segs.len[i] = lens[i];
                    ra.segs.table[i] = tables ? (*tables)[i] : nullptr;
                }
                GemmParams gr = g;
                gr.epi = GEMM_EPI_ROPE_SPLIT; gr.rope = &ra;
                if (gemm_tc5_supported(gr)) { CU(gemm_tc5_launch(gr, tp, bf, s)); ++nl; roped = true; }
            }
            if (!roped) { CU(linear(g)); ++nl; }
        }
        if (prefill_flash_) {
            // the whole pack: one RoPE / split launch and one fused attention launch per PF_MAX_SEGS sequences
            for (size_t c0 = 0; c0 < starts.size(); c0 += PF_MAX_SEGS) {
                PrefillSegs segs{};
                segs.n = (int)std::min<size_t>(PF_MAX_SEGS, starts.size() - c0);
                int row_lo = starts[c0], row_hi = row_lo;
                for (int i = 0; i < segs.n; ++i) {
                    segs.start[i] = starts[c0 + i];
                    segs.len[i] = lens[c0 + i];
                    segs.table[i] = tables ? (*tables)[c0 + i] : nullptr;
                    row_hi = std::max(row_hi, segs.start[i] + (segs.len[i] + 127) / 128 * 128);
                }
                if (c0 + PF_MAX_SEGS >= starts.size()) row_hi = std::max(row_hi, TP);      // trailing rows of the pack are zeroed too
                // the kernel indexes rows of the pack absolutely: shift the segment starts to the chunk's first row
                if (!roped) {
                    PrefillSegs rs = segs;
                    for (int i = 0; i < rs.n; ++i) rs.start[i] -= row_lo;
                    CU(rope_split_segs_launch(pf_qkv_ + (size_t)row_lo * ldq, row_hi - row_lo, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_ + (size_t)row_lo * qd,
                                              pf_k_ + (size_t)row_lo * kvd, pf_vt_ + row_lo, kc, vc, tp, rs, s)); ++nl;
                }
                CU(flash_prefill_launch(pf_q_, pf_k_, pf_vt_, (__half*)pf_attn_, segs, n_head_, n_kv_, hd_, tp, scale, s));
                ++nl;
            }
        } else
        for (size_t i = 0; i < starts.size(); ++i) {
            const int r0 = starts[i], len = lens[i], lp = (len + 127) / 128 * 128;
            // RoPE at positions 0..len-1 of THIS sequence; V^T columns r0.. of the pack-wide [kvd][tp] matrix; no cache
            CU(rope_split_launch(pf_qkv_ + (size_t)r0 * ldq, len, lp, 0, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, pf_q_ + (size_t)r0 * qd,
                                 pf_k_ + (size_t)r0 * kvd, pf_vt_ + r0, kc, vc, tables ? (*tables)[i] : nullptr, tp, s)); ++nl;
            {   // S[h] = Q_h K_kvh^T, compact [n_head][lp][lp]
                GemmParams g{};
                g.a = pf_q_ + (size_t)r0 * qd; g.b = pf_k_ + (size_t)r0 * kvd; g.c = pf_s_; g.m = len; g.n = len; g.k = hd_; g.lda = qd; g.ldb = kvd; g.ldc = lp;
                g.batch = n_head_; g.a_batch_stride = hd_; g.b_batch_stride = hd_; g.b_batch_div = grp; g.c_batch_stride = (long long)lp * lp;
                g.epi = GEMM_EPI_F32; g.causal_skip = 1;
                CU(gemm_tn_launch(g, false, s)); ++nl;
            }
            CU(softmax_causal_launch(pf_s_, n_head_, len, lp, scale, pf_p_, s)); ++nl;
            {   // O[:, h] = P[h] V_kvh
                GemmParams g{};
                g.a = pf_p_; g.b = pf_vt_ + r0; g.c = (__half*)pf_attn_ + (size_t)r0 * qd; g.m = len; g.n = hd_; g.k = lp; g.lda = lp; g.ldb = tp; g.ldc = qd;
                g.batch = n_head_; g.a_batch_stride = (long long)lp * lp; g.b_batch_stride = (long long)hd_ * tp; g.b_batch_div = grp; g.c_batch_stride = hd_;
                g.epi = GEMM_EPI_T16; g.causal_k = 1;
                CU(gemm_tn_launch(g, false, s)); ++nl;
            }
        }
        {
            GemmParams g{};
            g.a = pf_attn_; g.b = L.wo16; g.c = pf_x_; g.m = TP; g.n = n_embd_; g.k = qd; g.lda = qd; g.ldb = qd; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
        CU(rmsnorm_rows_launch(pf_x_, L.ffn_norm, TP, TP, n_embd_, eps_, pf_xn_, bf, s)); ++nl;
        {
            GemmParams g{};
            g.a = pf_xn_; g.b = L.wgu16; g.c = pf_h_; g.m = TP; g.n = 2 * n_ff_; g.k = n_embd_; g.lda = n_embd_; g.ldb = n_embd_; g.ldc = n_ff_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_SILU;
            CU(linear(g)); ++nl;
        }
        {
            GemmParams g{};
            g.a = pf_h_; g.b = L.wd16; g.c = pf_x_; g.m = TP; g.n = n_embd_; g.k = n_ff_; g.lda = n_ff_; g.ldb = n_ff_; g.ldc = n_embd_;
            g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ADD_F32;
            CU(linear(g)); ++nl;
        }
    }
    if (n_launch) *n_launch += nl;
    return {};
}

}  // namespace gl
