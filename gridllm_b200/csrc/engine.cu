// Engine implementation: GGUF -> HBM upload (engine row layouts), paged KV pool, decode-step
// construction (fused sm_90a kernels, PDL, CUDA graph) and the generate / embed drivers.
// See engine.h / include/gridllm_native.h for the reference call sites this replaces.
#include "engine.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>

#include "common.cuh"
#include "json_fsm.h"
#include "prefix_reuse.h"
#include "rowdot.h"

namespace gl {

static thread_local std::string g_last_error;
void set_last_error(const std::string& s) { g_last_error = s; }
const char* get_last_error() { return g_last_error.c_str(); }

namespace {

Status fail(int code, const std::string& m) { return Status{code, m}; }

#define CU(expr)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(GL_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
    } while (0)

#define ST(expr)                          \
    do {                                  \
        Status _s = (expr);               \
        if (!_s.ok()) return _s;          \
    } while (0)

int64_t now_ns() {
    return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

int env_int(const char* name, int dflt) {
    const char* v = std::getenv(name);
    return (v && *v) ? std::atoi(v) : dflt;
}

const char* ftype_name(uint64_t ft) {
    switch (ft) {
        case 0: return "F32";
        case 1: return "F16";
        case 7: return "Q8_0";
        case 14: return "Q4_K_S";
        case 15: return "Q4_K_M";
        case 18: return "Q6_K";
        case 32: return "BF16";
        default: return "unknown";
    }
}

}  // namespace

Status Engine::create(const std::string& path, int device, const gl_engine_opts* opts, Engine** out) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        return fail(GL_ERR_NO_DEVICE, std::string("no CUDA device (") + cudaGetErrorString(e) +
                                          "): the native worker has no CPU fallback");
    if (device < 0 || device >= n) return fail(GL_ERR_INVALID, "device index out of range");
    Engine* eng = new Engine();
    Status s = eng->load(path, device, opts);
    if (!s.ok()) { delete eng; return s; }
    *out = eng;
    return {};
}

Engine::~Engine() {
    cudaSetDevice(device_);
    if (stream_) cudaStreamSynchronize(stream_);
    if (g_nohead_) cudaGraphExecDestroy(g_nohead_);
    for (auto& v : g_head_var_)
        for (auto& k : v)
            for (auto& j : k)
                for (auto& g : j)
                    if (g) cudaGraphExecDestroy(g);
    for (auto& v : g_batch_)
        for (auto& g : v)
            if (g) cudaGraphExecDestroy(g);
    for (auto& ev : ev_) if (ev) cudaEventDestroy(ev);
    for (auto& kv : schemas_) cudaFree(kv.second.dev);
    for (void* p : allocs_) cudaFree(p);
    for (void* p : pf_allocs_) cudaFree(p);
    if (stream_) cudaStreamDestroy(stream_);
}

Status Engine::upload_f32(const GGUFTensor& t, float** out, int expect) {
    if (t.type != T_F32 || t.cols() * t.rows() != expect) return fail(GL_ERR_FORMAT, "tensor '" + t.name + "': expected F32[" + std::to_string(expect) + "]");
    CU(cudaMalloc((void**)out, (size_t)expect * 4));
    allocs_.push_back(*out);
    CU(cudaMemcpy(*out, t.data, (size_t)expect * 4, cudaMemcpyHostToDevice));
    return {};
}

Status Engine::upload_matrix(const GGUFTensor& t, DevMatrix& m, bool native_layout, bool paired) {
    BlockGeom g = block_geom(t.type);
    if (!g.weights) return fail(GL_ERR_UNSUPPORTED, "tensor '" + t.name + "': ggml type " + std::to_string(t.type) + " is outside the hot path (F32/F16/BF16/Q8_0/Q4_K/Q6_K)");
    m.type = (int)t.type;
    m.rows = (int)t.rows();
    m.cols = (int)t.cols();
    m.gguf_bytes = t.nbytes;
    const size_t rb = row_bytes(t.type, t.cols());
    const bool engine_layout = !native_layout && m.quantized();
    if (engine_layout && !ksplit(m.cols).nks) return fail(GL_ERR_UNSUPPORTED, "tensor '" + t.name + "': cols must be a multiple of 256 (and cut into <= 8 K-segments) for the quantised GEMV");
    size_t total;
    if (engine_layout) {
        // tile = the rows of one GEMV item of this matrix (half an item for the gate / up pair); rowdot.h
        m.tile_rows = paired ? item_rows(m.type) / 2 : item_rows(m.type);
        total = engine_matrix_bytes(m.type, m.rows, m.cols, m.tile_rows);
        m.row_stride = 0;
    } else {
        m.tile_rows = 1;
        m.row_stride = (int)(native_layout ? rb : align16(rb));
        total = (size_t)m.row_stride * m.rows;
    }
    CU(cudaMalloc((void**)&m.w, total + 256));
    allocs_.push_back(m.w);
    if (!engine_layout && (size_t)m.row_stride == rb) {
        CU(cudaMemcpy(m.w, t.data, total, cudaMemcpyHostToDevice));
        return {};
    }
    // repack on the host (parallel over rows), in slabs of whole tiles through one staging buffer
    const size_t slab_row_bytes = engine_layout ? total / ((m.rows + m.tile_rows - 1) / m.tile_rows * (size_t)m.tile_rows) : (size_t)m.row_stride;
    size_t slab_rows = std::max<size_t>(1, (size_t)(64u << 20) / slab_row_bytes);
    slab_rows = std::max<size_t>(m.tile_rows, slab_rows / m.tile_rows * m.tile_rows);
    std::vector<uint8_t> stage;
    for (size_t r0 = 0; r0 < (size_t)m.rows; r0 += slab_rows) {
        const size_t nr = std::min(slab_rows, (size_t)m.rows - r0);
        const size_t nr_pad = (nr + m.tile_rows - 1) / m.tile_rows * m.tile_rows;
        stage.assign(nr_pad * slab_row_bytes, 0);
        const int nthreads = (int)std::min<size_t>(8, std::max<size_t>(1, nr / 64));
        std::vector<std::thread> th;
        for (int ti = 0; ti < nthreads; ++ti) {
            th.emplace_back([&, ti]() {
                for (size_t r = ti; r < nr; r += nthreads) {
                    const uint8_t* src = t.data + (r0 + r) * rb;
                    if (engine_layout) repack_row(m.type, src, stage.data(), m.cols, m.tile_rows, (int)r);     // r0 is a tile boundary
                    else memcpy(stage.data() + r * m.row_stride, src, rb);
                }
            });
        }
        for (auto& x : th) x.join();
        CU(cudaMemcpy(m.w + r0 * slab_row_bytes, stage.data(), stage.size(), cudaMemcpyHostToDevice));
    }
    return {};
}

Status Engine::load(const std::string& path, int device, const gl_engine_opts* opts) {
    const int64_t t0 = now_ns();
    device_ = device;
    CU(cudaSetDevice(device));
    cudaDeviceProp prop{};
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) return fail(GL_ERR_UNSUPPORTED, std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major * 10 + prop.minor) + "; this library is built for sm_90a (H100) only");
    sm_count_ = prop.multiProcessorCount;

    abits_ = (opts && opts->act_bits == 8) ? 8 : 16;
    use_graph_ = !(opts && opts->use_graph == 0) && env_int("GL_GRAPH", 1) != 0;
    use_pdl_ = !(opts && opts->use_pdl == 0) && env_int("GL_PDL", 1) != 0;
    fused_ = env_int("GL_FUSE", 1) != 0;
    abits_ = env_int("GL_ACT_BITS", abits_) == 8 ? 8 : 16;
    nw_ = env_int("GL_WARPS", 12);
    if (!gemv_variant_ok(abits_, nw_)) nw_ = 12;
    ring_depth_ = std::max(2, std::min(4, env_int("GL_RING_DEPTH", 2)));          // persistent kernel
    ring_depth_max_ = std::max(2, std::min(4, env_int("GL_RING_DEPTH_MAX", 3)));   // stand-alone kernels: up to this many slots per warp
    smem_kb_ = std::min(227, env_int("GL_SMEM_KB", 227));
    lean_rings_ = env_int("GL_LEAN_RINGS", 1) != 0;
    xraw_ = env_int("GL_XRAW", 0) != 0;       // opt-in: a second prologue variant = a second kernel in the step (see hb256_)
    hb256_ = env_int("GL_HB256", 1) != 0;
    xraw_wide_ = env_int("GL_XRAW_WIDE", 0) != 0;        // measured (run 49): no gain -- each 14 KB piece waits ~1 us for its bulk copy
    polite_tracks_ = std::max(0, env_int("GL_POLITE_TRACKS", 3));
    sampler_pdl_ = env_int("GL_SAMPLER_PDL", 0) != 0;
    greedy_pdl_ = env_int("GL_GREEDY_PDL", 0) != 0;
    attn_splits_ = env_int("GL_ATTN_SPLITS", 16) == 8 ? 8 : 16;      // the splits of a KV head = one thread-block cluster (attention.cu)
    prefill_mode_ = env_int("GL_PREFILL", opts ? opts->prefill_mode : 0);
    prefill_min_ = env_int("GL_PREFILL_MIN", 8);
    prefill_tc5_ = env_int("GL_PREFILL_TC5", 1) != 0;
    prefill_flash_ = env_int("GL_PREFILL_FLASH", 1) != 0;
    prefill_fuse_rope_ = env_int("GL_PREFILL_FUSE_ROPE", 1) != 0;
    prefix_cache_ = opts && opts->prefix_cache != 0;

    std::string err = gguf_.open(path);
    if (!err.empty()) return fail(err.find("cannot open") == 0 ? GL_ERR_IO : GL_ERR_FORMAT, err);
    const std::string arch = gguf_.get_s("general.architecture", "");
    if (arch != "llama") return fail(GL_ERR_UNSUPPORTED, "architecture '" + arch + "' is outside the hot path (llama-family GGUF only)");
    auto key = [&](const char* k) { return arch + "." + k; };
    n_layer_ = (int)gguf_.get_u(key("block_count"), 0);
    n_embd_ = (int)gguf_.get_u(key("embedding_length"), 0);
    n_head_ = (int)gguf_.get_u(key("attention.head_count"), 0);
    n_kv_ = (int)gguf_.get_u(key("attention.head_count_kv"), n_head_);
    n_ff_ = (int)gguf_.get_u(key("feed_forward_length"), 0);
    eps_ = (float)gguf_.get_f(key("attention.layer_norm_rms_epsilon"), 1e-5);
    rope_base_ = (float)gguf_.get_f(key("rope.freq_base"), 10000.0);
    const int n_ctx_train = (int)gguf_.get_u(key("context_length"), 2048);
    if (!n_layer_ || !n_embd_ || !n_head_ || !n_ff_) return fail(GL_ERR_FORMAT, "missing llama hyper-parameters in GGUF metadata");
    hd_ = (int)gguf_.get_u(key("rope.dimension_count"), n_embd_ / n_head_);
    if (hd_ * n_head_ != n_embd_ || (hd_ != 64 && hd_ != 128)) return fail(GL_ERR_UNSUPPORTED, "head_dim must be 64 or 128 and n_head*head_dim == n_embd");
    if (n_kv_ <= 0 || n_head_ % n_kv_ || n_head_ / n_kv_ > 8) return fail(GL_ERR_UNSUPPORTED, "GQA group must divide n_head and be <= 8");
    // RoPE variants that are also general.architecture == llama: Llama-3.1 / 3.2 carry per-frequency factors in
    // rope_freqs.weight, some long-context fine-tunes a linear position scale; YaRN / longrope change the attention scale and
    // the interpolation ramp as well and are outside the path -- refused loudly rather than decoded with the wrong angles
    const std::string rs_type = gguf_.get_s(key("rope.scaling.type"), "");
    float rope_lin = 1.f;
    if (rs_type == "linear") {
        rope_lin = (float)gguf_.get_f(key("rope.scaling.factor"), 1.0);
        if (!(rope_lin > 0.f) || !std::isfinite(rope_lin)) return fail(GL_ERR_FORMAT, "rope.scaling.factor must be a positive number");
    } else if (!rs_type.empty() && rs_type != "none") {
        return fail(GL_ERR_UNSUPPORTED, "rope.scaling.type '" + rs_type + "' is outside the hot path (none / linear only)");
    }
    std::vector<float> rope_ff;                       // frequency factors (Llama-3.1+), one per rotated pair
    if (const GGUFTensor* tf = gguf_.tensor("rope_freqs.weight")) {
        if (tf->type != T_F32 || tf->cols() * tf->rows() != hd_ / 2) return fail(GL_ERR_FORMAT, "rope_freqs.weight: expected F32[head_dim/2]");
        rope_ff.assign(reinterpret_cast<const float*>(tf->data), reinterpret_cast<const float*>(tf->data) + hd_ / 2);
        for (float f : rope_ff)
            if (!(f > 0.f) || !std::isfinite(f)) return fail(GL_ERR_FORMAT, "rope_freqs.weight holds a non-positive factor");
    }
    n_ctx_ = (opts && opts->max_ctx > 0) ? opts->max_ctx : std::min(n_ctx_train, 8192);
    n_ctx_ = (n_ctx_ + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS * KV_PAGE_TOKENS;

    const GGUFTensor* te = gguf_.tensor("token_embd.weight");
    if (!te) return fail(GL_ERR_FORMAT, "missing token_embd.weight");
    n_vocab_ = (int)te->rows();
    if (te->cols() != n_embd_) return fail(GL_ERR_FORMAT, "token_embd.weight has wrong width");

    CU(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    for (auto& ev : ev_) CU(cudaEventCreate(&ev));
    CU(gemv_configure());
    CU(prefill_configure());
    CU(gemm_tc5_configure());
    CU(flash_prefill_configure());
    CU(attn_decode_configure());
    if (!attn_splits_ok(n_head_, n_kv_, hd_, attn_splits_)) return fail(GL_ERR_UNSUPPORTED, "decode attention: no cluster split of this head layout");

    // ---- weights -> HBM -------------------------------------------------------------------------
    ST(upload_matrix(*te, tok_embd_, /*native=*/true));
    const GGUFTensor* tout = gguf_.tensor("output.weight");
    ST(upload_matrix(tout ? *tout : *te, output_, false));
    const GGUFTensor* ton = gguf_.tensor("output_norm.weight");
    if (!ton) return fail(GL_ERR_FORMAT, "missing output_norm.weight");
    ST(upload_f32(*ton, &output_norm_, n_embd_));
    layers_.resize(n_layer_);
    uint64_t layer_bytes = 0;
    n_params_ = (uint64_t)te->rows() * te->cols() + (tout ? (uint64_t)tout->rows() * tout->cols() : 0);
    for (int il = 0; il < n_layer_; ++il) {
        LayerWeights& L = layers_[il];
        const std::string p = "blk." + std::to_string(il) + ".";
        struct Item { const char* n; DevMatrix* m; int rows, cols; bool paired; };
        Item items[] = {{"attn_q.weight", &L.wq, n_head_ * hd_, n_embd_, false},  {"attn_k.weight", &L.wk, n_kv_ * hd_, n_embd_, false},
                        {"attn_v.weight", &L.wv, n_kv_ * hd_, n_embd_, false},    {"attn_output.weight", &L.wo, n_embd_, n_head_ * hd_, false},
                        {"ffn_gate.weight", &L.wgate, n_ff_, n_embd_, true},      {"ffn_up.weight", &L.wup, n_ff_, n_embd_, true},
                        {"ffn_down.weight", &L.wdown, n_embd_, n_ff_, false}};
        for (auto& it : items) {
            const GGUFTensor* t = gguf_.tensor(p + it.n);
            if (!t) return fail(GL_ERR_FORMAT, "missing tensor " + p + it.n);
            if (t->rows() != it.rows || t->cols() != it.cols) return fail(GL_ERR_FORMAT, "tensor " + p + it.n + " has unexpected shape");
            ST(upload_matrix(*t, *it.m, false, it.paired));
            layer_bytes += t->nbytes;
            n_params_ += (uint64_t)t->rows() * t->cols();
            if (!it.m->quantized()) all_quant_ = false;
        }
        const GGUFTensor* an = gguf_.tensor(p + "attn_norm.weight");
        const GGUFTensor* fn = gguf_.tensor(p + "ffn_norm.weight");
        if (!an || !fn) return fail(GL_ERR_FORMAT, "missing norm weights in layer " + std::to_string(il));
        ST(upload_f32(*an, &L.attn_norm, n_embd_));
        ST(upload_f32(*fn, &L.ffn_norm, n_embd_));
    }
    if (!output_.quantized()) all_quant_ = false;
    if (!all_quant_) fused_ = false;
    weight_bytes_ = layer_bytes + output_.gguf_bytes + tok_embd_.gguf_bytes;
    decode_bytes_ = layer_bytes + output_.gguf_bytes + (uint64_t)(2 * n_layer_ + 1) * n_embd_ * 4 + row_bytes(tok_embd_.type, n_embd_);

    // ---- activations, KV pool, state ------------------------------------------------------------
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess) { allocs_.push_back(*p); e = cudaMemset(*p, 0, bytes); }
        return e;
    };
    const int qdim = n_head_ * hd_, kvdim = n_kv_ * hd_;
    CU(dalloc((void**)&x_, (size_t)n_embd_ * 4));
    CU(dalloc((void**)&xn_, (size_t)std::max(n_embd_, n_ff_) * 4));
    CU(dalloc((void**)&q_, (size_t)qdim * 4));
    CU(dalloc((void**)&ktmp_, (size_t)kvdim * 4));
    CU(dalloc((void**)&vtmp_, (size_t)kvdim * 4));
    CU(dalloc((void**)&attn_, (size_t)qdim * 4));
    CU(dalloc((void**)&h_, (size_t)n_ff_ * 4));
    CU(dalloc((void**)&gate_, (size_t)n_ff_ * 4));
    CU(dalloc((void**)&up_, (size_t)n_ff_ * 4));
    CU(dalloc((void**)&ytmp_, (size_t)std::max(n_embd_, n_ff_) * 4));
    CU(dalloc((void**)&logits_, (size_t)n_vocab_ * 4));
    CU(dalloc((void**)&part_o_, (size_t)n_head_ * std::max(attn_splits_, 32) * hd_ * 4));
    if (env_int("GL_TRACE", 0)) {
        CU(dalloc((void**)&perop_trace_, (size_t)PEROP_TRACE_LAUNCHES * 16 * 8));
        CU(cudaMemset(perop_trace_, 0, (size_t)PEROP_TRACE_LAUNCHES * 16 * 8));
    }
    CU(dalloc((void**)&part_ml_, (size_t)n_head_ * std::max(attn_splits_, 32) * 2 * 4));
    CU(dalloc((void**)&counters_, (size_t)n_kv_ * 4));
    CU(dalloc((void**)&sample_scratch_, (size_t)SAMPLE_SCRATCH_FLOATS * 4));
    CU(dalloc((void**)&topk_scratch_, TOPK_SCRATCH_BYTES));
    CU(dalloc((void**)&pen_counts_, (size_t)n_vocab_ * 4));
    n_pages_ = n_ctx_ / KV_PAGE_TOKENS;
    // the page pool is shared by every open sequence (gl_generate's one sequence and the gl_seq_open slots)
    max_batch_ = std::max(0, std::min(MAX_BATCH, env_int("GL_MAX_BATCH", opts ? opts->max_batch : 0)));
    if (max_batch_ == 1) max_batch_ = 0;
    batch_weights_ = env_int("GL_BATCH_WEIGHTS", opts ? opts->batch_weights : 0);
    {
        long long pool_tokens = (opts && opts->kv_pool_tokens > 0) ? opts->kv_pool_tokens : (long long)n_ctx_ * std::max(1, max_batch_);
        pool_tokens = std::max<long long>(pool_tokens, n_ctx_);
        // never more than 60 % of what is free right now (the 16-bit prefill copy and the scratch come after this)
        size_t free_b = 0, total_b = 0;
        CU(cudaMemGetInfo(&free_b, &total_b));
        const size_t per_token = (size_t)2 * n_layer_ * n_kv_ * hd_ * sizeof(__half);
        const long long cap_tokens = (long long)(free_b * 6 / 10 / per_token);
        if (pool_tokens > cap_tokens) pool_tokens = std::max<long long>(cap_tokens, n_ctx_);
        pool_pages_ = (int)((pool_tokens + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS);
    }
    kv_layer_elems_ = (size_t)pool_pages_ * n_kv_ * KV_PAGE_TOKENS * hd_;
    CU(dalloc((void**)&kcache_, kv_layer_elems_ * n_layer_ * sizeof(__half)));
    CU(dalloc((void**)&vcache_, kv_layer_elems_ * n_layer_ * sizeof(__half)));
    CU(dalloc((void**)&page_table_, (size_t)n_pages_ * 4));
    CU(dalloc((void**)&st_, sizeof(StepState)));
    CU(dalloc((void**)&prompt_ids_, (size_t)n_ctx_ * 4));
    max_out_ = n_ctx_;
    CU(dalloc((void**)&out_ids_, (size_t)max_out_ * 4));
    CU(dalloc((void**)&out_lp_, (size_t)max_out_ * 4));
    // physical pages are handed out in reverse order so that the page table is a real indirection
    free_pages_.resize(pool_pages_);
    for (int i = 0; i < pool_pages_; ++i) free_pages_[i] = i;

    // RoPE tables (oracle/llama_oracle.py rope_table): inv_freq rounded to fp32, angle formed in fp32,
    // cos/sin evaluated in double, rounded to fp32.
    {
        std::vector<float> c((size_t)n_ctx_ * hd_ / 2), s((size_t)n_ctx_ * hd_ / 2);
        std::vector<float> inv(hd_ / 2);
        for (int i = 0; i < hd_ / 2; ++i) {
            inv[i] = (float)std::pow((double)rope_base_, -2.0 * i / hd_);
            if (!rope_ff.empty()) inv[i] = inv[i] / rope_ff[i];       // fp32 division, like the oracle
        }
        for (int pos = 0; pos < n_ctx_; ++pos)
            for (int i = 0; i < hd_ / 2; ++i) {
                const float ang = ((float)pos / rope_lin) * inv[i];
                c[(size_t)pos * hd_ / 2 + i] = (float)std::cos((double)ang);
                s[(size_t)pos * hd_ / 2 + i] = (float)std::sin((double)ang);
            }
        CU(dalloc((void**)&rope_cos_, c.size() * 4));
        CU(dalloc((void**)&rope_sin_, s.size() * 4));
        CU(cudaMemcpy(rope_cos_, c.data(), c.size() * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(rope_sin_, s.data(), s.size() * 4, cudaMemcpyHostToDevice));
    }
    tok_.load(gguf_);

    // ---- info -----------------------------------------------------------------------------------
    std::memset(&info_, 0, sizeof(info_));
    std::snprintf(info_.arch, sizeof(info_.arch), "%s", arch.c_str());
    std::snprintf(info_.name, sizeof(info_.name), "%s", gguf_.get_s("general.name", "unnamed").c_str());
    std::snprintf(info_.quantization, sizeof(info_.quantization), "%s", ftype_name(gguf_.get_u("general.file_type", 9999)));
    info_.n_layer = n_layer_; info_.n_embd = n_embd_; info_.n_head = n_head_; info_.n_head_kv = n_kv_; info_.head_dim = hd_;
    info_.n_ff = n_ff_; info_.n_vocab = n_vocab_; info_.n_ctx_train = n_ctx_train; info_.n_ctx = n_ctx_;
    info_.rope_base = rope_base_; info_.rms_eps = eps_;
    info_.bos_id = tok_.bos; info_.eos_id = tok_.eos; info_.eot_id = tok_.eot; info_.has_tokenizer = tok_.ok() ? 1 : 0;
    info_.n_params = n_params_; info_.file_bytes = gguf_.file_bytes; info_.weight_bytes = weight_bytes_;
    info_.decode_bytes_per_token = decode_bytes_; info_.device = device_; info_.sm_count = sm_count_;

    ST(kv_reset());
    if (prefill_mode_ != 1) ST(build_prefill_weights());
    // the persistent single-launch decode kernel is opt-in: it is correct (same tests) but, as of round 1, slower than
    // the per-op graph path
    if (fused_ && all_quant_ && env_int("GL_MEGA", 0) != 0) ST(build_mega());
    if (use_graph_ && !use_mega_) ST(build_graphs());
    CU(cudaStreamSynchronize(stream_));
    load_ns_ = now_ns() - t0;
    return {};
}

Status Engine::info(gl_model_info* out) const {
    *out = info_;
    return {};
}

const DevMatrix* Engine::find_matrix(const std::string& name) const {
    if (name == "output.weight") return &output_;
    if (name.rfind("blk.", 0) == 0) {
        const size_t dot = name.find('.', 4);
        if (dot == std::string::npos) return nullptr;
        const int il = std::atoi(name.substr(4, dot - 4).c_str());
        if (il < 0 || il >= n_layer_) return nullptr;
        const std::string rest = name.substr(dot + 1);
        const LayerWeights& L = layers_[il];
        if (rest == "attn_q.weight") return &L.wq;
        if (rest == "attn_k.weight") return &L.wk;
        if (rest == "attn_v.weight") return &L.wv;
        if (rest == "attn_output.weight") return &L.wo;
        if (rest == "ffn_gate.weight") return &L.wgate;
        if (rest == "ffn_up.weight") return &L.wup;
        if (rest == "ffn_down.weight") return &L.wdown;
    }
    return nullptr;
}

// -------------------------------------------------------------------------------------------------
// KV pages
// -------------------------------------------------------------------------------------------------
Status Engine::kv_reset() {
    for (int p : seq_pages_) free_pages_.push_back(p);
    seq_pages_.clear();
    cached_ids_.clear();
    host_pos_ = 0;
    return set_state(0, 0, 0, 0, nullptr);
}

Status Engine::ensure_pages(int n_tokens) {
    if (n_tokens > n_ctx_) return fail(GL_ERR_CONTEXT, "sequence of " + std::to_string(n_tokens) + " tokens exceeds the engine context " + std::to_string(n_ctx_));
    const int need = (n_tokens + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    bool grew = false;
    while ((int)seq_pages_.size() < need) {
        if (free_pages_.empty()) return fail(GL_ERR_NOMEM, "KV page pool exhausted");
        seq_pages_.push_back(free_pages_.back());
        free_pages_.pop_back();
        grew = true;
    }
    if (grew) CU(cudaMemcpyAsync(page_table_, seq_pages_.data(), seq_pages_.size() * 4, cudaMemcpyHostToDevice, stream_));
    return {};
}

// repetition penalties (penalty.cu): repeat_penalty is active when > 0 and != 1; a window of 0, or nothing active, is no penalty
// at all, and such a request replays exactly the graphs of a request without the fields
static bool repeat_penalty_on(const gl_sample_opts& so) { return so.repeat_penalty > 0.f && so.repeat_penalty != 1.f; }
static bool penalties_on(const gl_sample_opts& so) {
    return so.repeat_last_n != 0 && (repeat_penalty_on(so) || so.presence_penalty != 0.f || so.frequency_penalty != 0.f);
}

StepState Engine::make_state(int pos, int token, int n_prompt, int out_idx, const gl_sample_opts* so) const {
    StepState h{};
    h.pos = pos; h.token = token; h.n_prompt = n_prompt; h.out_idx = out_idx; h.done = 0;
    h.ignore_eos = so ? so->ignore_eos : 1;
    h.n_stop = 0;
    if (so && !so->ignore_eos) {
        if (tok_.eos >= 0) h.stop_ids[h.n_stop++] = tok_.eos;
        if (tok_.eot >= 0 && tok_.eot != tok_.eos) h.stop_ids[h.n_stop++] = tok_.eot;
        for (int i = 0; i < so->n_stop_ids && h.n_stop < 8; ++i) h.stop_ids[h.n_stop++] = so->stop_ids[i];
    }
    h.bar_base = 0;
    h.temperature = so ? so->temperature : 0.f;
    h.top_k = so ? so->top_k : 0;
    h.top_p = (so && so->top_p > 0.f) ? so->top_p : 1.f;
    h.seed_lo = so ? (unsigned)(so->seed & 0xffffffffull) : 0u;
    h.seed_hi = so ? (unsigned)(so->seed >> 32) : 0u;
    h.min_p = (so && so->min_p > 0.f) ? so->min_p : 0.f;
    const bool pen = so && penalties_on(*so);
    h.pen_last_n = pen ? so->repeat_last_n : 0;
    h.repeat_penalty = so && repeat_penalty_on(*so) ? so->repeat_penalty : 1.f;
    h.presence_penalty = pen ? so->presence_penalty : 0.f;
    h.frequency_penalty = pen ? so->frequency_penalty : 0.f;
    h.json = so && so->format ? 1 : 0;          // the grammar mask's state lives in the sequence's SchemaSlot
    return h;
}

Status Engine::plan_draw(const gl_sample_opts& so, bool single_path, DrawPlan* plan) {
    if (!(so.temperature >= 0.f) || !std::isfinite(so.temperature)) return fail(GL_ERR_INVALID, "temperature must be a finite number >= 0");
    DrawPlan d;
    // 0 greedy; 1 two-stage top-k sampler (top_k <= 64); 2 single-CTA radix select (sampler.cu)
    d.sampler = so.temperature > 0.f ? (sample_topk_fast_applies(so.top_k, n_vocab_) ? 1 : 2) : 0;
    d.penalised = penalties_on(so);
    d.masked = so.format != 0;
    d.format = so.format;
    const bool mega = single_path && use_mega_;
    if (mega && d.sampler) return fail(GL_ERR_UNSUPPORTED, "the persistent decode kernel (GL_MEGA=1) samples greedily only");
    if (mega && d.penalised) return fail(GL_ERR_UNSUPPORTED, "the persistent decode kernel (GL_MEGA=1) has no repetition penalties");
    if (d.masked) {
        // the value range of format and its clash with ignore_eos are checked at the C boundary (c_api.cpp check_format)
        const bool schema = so.format >= GL_FORMAT_SCHEMA_BASE;
        if (schema && !schemas_.count(so.format)) return fail(GL_ERR_INVALID, "format: unknown or evicted schema code " + std::to_string(so.format));
        if (mega) return fail(GL_ERR_UNSUPPORTED, "the persistent decode kernel (GL_MEGA=1) has no JSON grammar mask");
        ST(ensure_json());
        ST(ensure_schema_state());
        if (schema) schemas_[so.format].used = ++schema_clock_;
        // a stop id that is an ordinary token would be masked wherever it is needed, and the vocabulary guarantee would not hold
        for (int i = 0; i < so.n_stop_ids; ++i) {
            const int32_t id = so.stop_ids ? so.stop_ids[i] : -1;
            if (id >= 0 && id < n_vocab_ && json_hoff_[id + 1] != json_hoff_[id])
                return fail(GL_ERR_INVALID, "format json: stop_ids must be control tokens (empty piece); use stop strings for text");
        }
    }
    *plan = d;
    return {};
}

Status Engine::set_state(int pos, int token, int n_prompt, int out_idx, const gl_sample_opts* so, const DrawPlan& plan) {
    const StepState h = make_state(pos, token, n_prompt, out_idx, so);
    plan_ = plan;
    if (plan.masked) ST(schema_bind(schema_entry(), plan.format));
    if (bar_counter_) CU(cudaMemsetAsync(bar_counter_, 0, 4, stream_));
    CU(cudaMemcpyAsync(st_, &h, sizeof(h), cudaMemcpyHostToDevice, stream_));
    CU(cudaStreamSynchronize(stream_));     // h is on the stack
    return {};
}

// -------------------------------------------------------------------------------------------------
// decode step
// -------------------------------------------------------------------------------------------------
Status Engine::enqueue_gemv(cudaStream_t s, GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, int* n_launch) {
    // slot size: what the widest item of this kernel needs (Q4_K: 4 row segments, Q6_K / Q8_0: 2), ring depth: whatever
    // shared memory is left, capped so that the bytes in flight stay near what the HBM pipe needs
    int need = 0;
    {
        const KSplit ks = ksplit(cols);
        if (!ks.nks) return fail(GL_ERR_UNSUPPORTED, "GEMV shape outside the kernel envelope (cols=" + std::to_string(cols) + ")");
        for (int i = 0; i < nmat; ++i) need = std::max(need, item_rows(mats[i].type) * kseg_bytes(mats[i].type, ks.seg_nb));
    }
    p.slot_bytes = (need + 127) & ~127;
    if (!gemv_plan(p, mats, nmat, pair, cols, p.slot_bytes)) return fail(GL_ERR_UNSUPPORTED, "GEMV shape outside the kernel envelope (cols=" + std::to_string(cols) + ")");
    // prologue variant (= which kernel, gemv.cu): by default the 256-bit-load half-block prologue for every width, so that all
    // GEMV launches of a step are one kernel; GL_XRAW=1 stages narrow rows raw by one bulk copy instead (16 KB of ring)
    p.xraw_bytes = 0;
    p.xraw_nseg = 1;
    const bool variants = gemv_prologue_variants(nw_);
    p.hb256 = (variants && hb256_ && (cols > GEMV_XRAW_MAX_COLS || !xraw_) && cols <= 16 * nw_ * 32 * (nw_ >= 12 ? 3 : 4)) ? 1 : 0;
    if (variants && xraw_ && !p.hb256) {
        const KSplit ks = ksplit(cols);
        if (cols <= GEMV_XRAW_MAX_COLS && cols / 16 <= nw_ * 32) {
            p.xraw_bytes = cols * 4;
        } else if (xraw_wide_ && ks.nks > 1 && cols / ks.nks / 16 <= nw_ * 32) {     // wide rows: K-segment pieces, two buffers
            p.xraw_nseg = ks.nks;
            p.xraw_bytes = 2 * (cols / ks.nks) * 4;
        }
    }
    const size_t fixed = gemv_smem_bytes(cols, 0, 0) + (size_t)p.xraw_bytes;
    const int ns = std::min(RING_MAX_SLOTS, (int)(((size_t)smem_kb_ * 1024 - fixed) / p.slot_bytes));
    // as many consumer warps as there are, each with >= 2 slots; spare slots deepen the tracks (small slots: more bytes in flight)
    // tracks x depth: as many bytes in flight as the ring can hold, giving up at most two consumer warps for depth
    // (small slots -- Q6_K pairs -- would otherwise leave a third of the shared memory unused: lm_head 0.94 -> 0.86 of peak)
    p.n_tracks = std::min(nw_, ns / 2);
    p.depth = p.n_tracks > 0 ? std::min(ring_depth_max_, ns / p.n_tracks) : 0;
    for (int t = std::max(1, nw_ - 2); p.pd.nks > 1 && t < std::min(nw_, ns / 2); ++t) {      // (narrow rows keep every warp: lm_head is issue-bound at 10)
        const int dd = std::min(ring_depth_max_, ns / t);
        if (dd >= 2 && t * dd > p.n_tracks * p.depth) { p.n_tracks = t; p.depth = dd; }
    }
    // a phase in which no warp gets a second slot (one round of items, one K-segment) needs one slot per warp: the smaller
    // footprint (121 KB instead of 232 KB) lets the next kernel's CTAs become resident -- and start their own prefetch --
    // while this one is still running (programmatic dependent launch)
    if (lean_rings_ && p.n_tracks > 0 && p.pd.nks == 1) {
        int items = 0;
        for (int i = 0; i < (pair ? 1 : nmat); ++i) items += p.pd.seg[i].n_items;
        if ((items + sm_count_ - 1) / sm_count_ <= p.n_tracks) p.depth = 1;
    }
    if (p.n_tracks < 1) return fail(GL_ERR_UNSUPPORTED, "GEMV staging does not fit shared memory");
    p.trace = perop_trace_ ? perop_trace_ + 16 * (size_t)std::min(*n_launch, PEROP_TRACE_LAUNCHES - 1) : nullptr;
    CU(gemv_launch(p, abits_, nw_, sm_count_, use_pdl_, s));
    ++*n_launch;
    return {};
}

Status Engine::plain_gemv(cudaStream_t s, const DevMatrix& m, const float* x, float* y, int* n_launch) {
    if (m.quantized()) {
        GemvParams p{};
        p.x = x; p.epi = EPI_STORE; p.out = y; p.st = st_;
        const GemvMat mm[1] = {{m.w, m.type, m.rows, m.tile_rows}};
        return enqueue_gemv(s, p, mm, 1, false, m.cols, n_launch);
    }
    CU(gemv_fp_launch(m.w, m.type, m.rows, m.cols, x, y, s));
    ++*n_launch;
    return {};
}

Status Engine::enqueue_step(cudaStream_t s, bool with_head, bool keep_logits, int* n_launch) {
    const bool pdl = use_pdl_;
    {
        EmbedParams ep{tok_embd_.w, tok_embd_.type, n_embd_, tok_embd_.row_stride, st_, prompt_ids_, x_};
        CU(embed_launch(ep, pdl, s));
        ++*n_launch;
    }
    const float scale = 1.0f / std::sqrt((float)hd_);
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = kcache_ + (size_t)il * kv_layer_elems_;
        __half* vc = vcache_ + (size_t)il * kv_layer_elems_;
        if (fused_) {
            GemvParams p{};
            const GemvMat qkv[3] = {{L.wq.w, L.wq.type, L.wq.rows, L.wq.tile_rows}, {L.wk.w, L.wk.type, L.wk.rows, L.wk.tile_rows}, {L.wv.w, L.wv.type, L.wv.rows, L.wv.tile_rows}};
            p.x = x_; p.norm_w = L.attn_norm; p.eps = eps_; p.epi = EPI_QKV; p.out = q_;
            p.rope_cos = rope_cos_; p.rope_sin = rope_sin_; p.head_dim = hd_; p.n_kv_heads = n_kv_;
            p.k_cache = kc; p.v_cache = vc; p.page_table = page_table_; p.st = st_;
            ST(enqueue_gemv(s, p, qkv, 3, false, n_embd_, n_launch));
        } else {
            CU(rmsnorm_launch(x_, L.attn_norm, n_embd_, eps_, xn_, s)); ++*n_launch;
            ST(plain_gemv(s, L.wq, xn_, q_, n_launch));
            ST(plain_gemv(s, L.wk, xn_, ktmp_, n_launch));
            ST(plain_gemv(s, L.wv, xn_, vtmp_, n_launch));
            CU(rope_kv_launch(q_, ktmp_, vtmp_, n_head_, n_kv_, hd_, rope_cos_, rope_sin_, st_, kc, vc, page_table_, s)); ++*n_launch;
        }
        {
            AttnParams a{};
            a.q = q_; a.k_cache = kc; a.v_cache = vc; a.page_table = page_table_; a.n_table = n_pages_; a.st = st_; a.out = attn_;
            a.n_head = n_head_; a.n_kv_heads = n_kv_; a.head_dim = hd_; a.n_splits = attn_splits_; a.scale = scale;
            a.trace = perop_trace_ ? perop_trace_ + 16 * (size_t)std::min(*n_launch, PEROP_TRACE_LAUNCHES - 1) : nullptr;
            CU(attn_decode_launch(a, pdl && fused_, s));
            ++*n_launch;
        }
        if (fused_) {
            GemvParams p{};
            const GemvMat mo[1] = {{L.wo.w, L.wo.type, L.wo.rows, L.wo.tile_rows}};
            p.x = attn_; p.epi = EPI_ADD; p.out = x_; p.resid = x_; p.st = st_;
            p.polite_tracks = polite_tracks_;      // resident beside the attention CTAs: prefetch politely (gemv.cu)
            ST(enqueue_gemv(s, p, mo, 1, false, n_head_ * hd_, n_launch));
            GemvParams g{};
            const GemvMat mgu[2] = {{L.wgate.w, L.wgate.type, L.wgate.rows, L.wgate.tile_rows}, {L.wup.w, L.wup.type, L.wup.rows, L.wup.tile_rows}};
            g.x = x_; g.norm_w = L.ffn_norm; g.eps = eps_; g.epi = EPI_SILU; g.out = h_; g.st = st_;
            if (L.wgate.type != L.wup.type) return fail(GL_ERR_UNSUPPORTED, "ffn_gate / ffn_up with different types");
            ST(enqueue_gemv(s, g, mgu, 2, true, n_embd_, n_launch));
            GemvParams d{};
            const GemvMat md[1] = {{L.wdown.w, L.wdown.type, L.wdown.rows, L.wdown.tile_rows}};
            d.x = h_; d.epi = EPI_ADD; d.out = x_; d.resid = x_; d.st = st_;
            ST(enqueue_gemv(s, d, md, 1, false, n_ff_, n_launch));
        } else {
            ST(plain_gemv(s, L.wo, attn_, ytmp_, n_launch));
            CU(add_launch(x_, ytmp_, n_embd_, x_, s)); ++*n_launch;
            CU(rmsnorm_launch(x_, L.ffn_norm, n_embd_, eps_, xn_, s)); ++*n_launch;
            ST(plain_gemv(s, L.wgate, xn_, gate_, n_launch));
            ST(plain_gemv(s, L.wup, xn_, up_, n_launch));
            CU(silu_mul_launch(gate_, up_, n_ff_, h_, s)); ++*n_launch;
            ST(plain_gemv(s, L.wdown, h_, ytmp_, n_launch));
            CU(add_launch(x_, ytmp_, n_embd_, x_, s)); ++*n_launch;
        }
    }
    if (with_head) {
        ST(enqueue_head(s, keep_logits, n_launch));
    } else {
        CU(advance_launch(st_, pdl && fused_, s));
        ++*n_launch;
    }
    return {};
}

Status Engine::enqueue_head(cudaStream_t s, bool keep_logits, int* n_launch) {
    const bool pdl = use_pdl_;
    if (fused_) {
        GemvParams p{};
        const GemvMat mh[1] = {{output_.w, output_.type, output_.rows, output_.tile_rows}};
        p.x = x_; p.norm_w = output_norm_; p.eps = eps_; p.epi = EPI_STORE; p.out = logits_; p.st = st_;
        ST(enqueue_gemv(s, p, mh, 1, false, n_embd_, n_launch));
    } else {
        CU(rmsnorm_launch(x_, output_norm_, n_embd_, eps_, xn_, s)); ++*n_launch;
        ST(plain_gemv(s, output_, xn_, logits_, n_launch));
    }
    CU(enqueue_pre_draw(s, 0, plan_.penalised, plan_.masked, prompt_ids_, n_launch));
    SampleParams sp{logits_, n_vocab_, st_, out_ids_, out_lp_, keep_logits ? logits_keep_ : nullptr, keep_logits ? keep_cap_ : max_out_, sample_scratch_, topk_scratch_};
    if (plan_.sampler != 0) CU(sample_topk_launch(sp, plan_.sampler == 1, pdl && fused_ && sampler_pdl_, s));      // temperature > 0: seeded top-k / top-p draw (sampler.cu)
    else CU(sample_greedy_launch(sp, pdl && fused_ && greedy_pdl_, s));
    ++*n_launch;
    return {};
}

// The penalty and mask kernels launch without programmatic dependent launch: plain stream order after the lm_head.
cudaError_t Engine::enqueue_pre_draw(cudaStream_t s, int bucket, bool penalised, bool masked, const int* prompt, int* n_launch) {
    const bool one = bucket == 0;
    float* logits = one ? logits_ : blogits_;
    StepState* st = one ? st_ : bst_;
    const BatchCtl* ctl = one ? nullptr : bctl_;
    const int rows = one ? 1 : bucket;
    if (penalised) {
        const PenaltyParams pp = one ? PenaltyParams{logits, n_vocab_, st, ctl, prompt, 0, out_ids_, 0, pen_counts_}
                                     : PenaltyParams{logits, n_vocab_, st, ctl, bprompt_, n_ctx_, bout_ids_, max_out_, bpen_counts_};
        const cudaError_t e = penalty_launch(pp, rows, false, s);
        if (e != cudaSuccess) return e;
        if (n_launch) ++*n_launch;
    }
    if (masked) {
        const SchemaMaskParams mp{logits, n_vocab_, st, ctl, one ? schema_entry() : sch_ + 1, json_off_, json_bytes_, json_cls_};
        const cudaError_t e = schema_mask_launch(mp, rows, false, s);
        if (e != cudaSuccess) return e;
        if (n_launch) ++*n_launch;
    }
    return cudaSuccess;
}

Status Engine::build_graphs() {
    for (int which = 0; which < 2; ++which) {
        cudaGraph_t g = nullptr;
        int n = 0;
        CU(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
        Status s = enqueue_step(stream_, which == 1, false, &n);
        cudaError_t e = cudaStreamEndCapture(stream_, &g);
        if (!s.ok()) { if (g) cudaGraphDestroy(g); return s; }
        if (e != cudaSuccess) return fail(GL_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
        cudaGraphExec_t ge = nullptr;
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(GL_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
        if (which == 0) { g_nohead_ = ge; launches_nohead_ = n; } else { g_head_var_[0][0][0][0] = ge; launches_head_ = n; }
    }
    return {};
}

Status Engine::run_steps(int n_nohead, int n_head, bool keep_logits) {
    int dummy = 0;
    if (use_mega_) {
        if (n_nohead > 0) ST(launch_mega(n_nohead, false, false));
        if (n_head > 0) ST(launch_mega(n_head, true, keep_logits));
        return {};
    }
    // the step with a head exists in 24 captured variants (sampler x plain / logits kept x without / with the penalty kernel x
    // without / with the mask kernel); all but the first lazily
    cudaGraphExec_t* head = &g_head_var_[plan_.sampler][keep_logits ? 1 : 0][plan_.penalised ? 1 : 0][plan_.masked ? 1 : 0];
    if (use_graph_ && n_head > 0 && !*head) {
        cudaGraph_t g = nullptr;
        CU(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
        Status s = enqueue_step(stream_, true, keep_logits, &dummy);
        cudaError_t e = cudaStreamEndCapture(stream_, &g);
        if (!s.ok()) { if (g) cudaGraphDestroy(g); return s; }
        if (e != cudaSuccess) return fail(GL_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
        e = cudaGraphInstantiate(head, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(GL_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
    }
    for (int i = 0; i < n_nohead; ++i) {
        if (use_graph_) CU(cudaGraphLaunch(g_nohead_, stream_));
        else ST(enqueue_step(stream_, false, false, &dummy));
    }
    for (int i = 0; i < n_head; ++i) {
        if (use_graph_) CU(cudaGraphLaunch(*head, stream_));
        else ST(enqueue_step(stream_, true, keep_logits, &dummy));
    }
    return {};
}

Status Engine::build_mega() {
    CU(mega_configure());
    mega_max_cols_ = std::max(n_embd_, std::max(n_ff_, n_head_ * hd_));
    if (mega_max_cols_ % 256 || mega_max_cols_ > 32768) return {};      // outside the kernel envelope: per-op path
    mega_slot_bytes_ = (env_int("GL_MEGA_SLOT_BYTES", GEMV_MIN_SLOT_BYTES) + 127) & ~127;
    const size_t fixed = mega_smem_bytes(mega_max_cols_, 0, 0);
    const size_t budget = (size_t)env_int("GL_MEGA_SMEM_KB", 227) * 1024;
    if (fixed + 2 * (size_t)mega_slot_bytes_ > budget) return {};
    mega_depth_ = ring_depth_;
    mega_tracks_ = std::min(nw_, (int)std::min<size_t>(RING_MAX_SLOTS, (budget - fixed) / mega_slot_bytes_) / mega_depth_);
    mega_tracks_ = std::min(mega_tracks_, env_int("GL_MEGA_TRACKS", nw_));
    if (mega_tracks_ < 1) return {};
    std::vector<MegaPhase> ph;
    mega_prod_.clear();
    mega_splits_ = std::max(1, std::min(32, sm_count_ / n_kv_));
    auto add_gemv = [&](GemvParams g, const GemvMat* mats, int nmat, bool pair, int cols, int flags) -> bool {
        g.n_tracks = mega_tracks_;
        g.depth = mega_depth_;
        g.slot_bytes = mega_slot_bytes_;
        if (!gemv_plan(g, mats, nmat, pair, cols, mega_slot_bytes_)) return false;
        MegaPhase m{};
        m.kind = PH_GEMV; m.flags = flags; m.g = g;
        ph.push_back(m);
        mega_prod_.push_back(g.pd);
        return true;
    };
    for (int il = 0; il < n_layer_; ++il) {
        const LayerWeights& L = layers_[il];
        __half* kc = kcache_ + (size_t)il * kv_layer_elems_;
        __half* vc = vcache_ + (size_t)il * kv_layer_elems_;
        GemvParams p{};
        const GemvMat qkv[3] = {{L.wq.w, L.wq.type, L.wq.rows, L.wq.tile_rows}, {L.wk.w, L.wk.type, L.wk.rows, L.wk.tile_rows}, {L.wv.w, L.wv.type, L.wv.rows, L.wv.tile_rows}};
        p.x = x_; p.norm_w = L.attn_norm; p.eps = eps_; p.epi = EPI_QKV; p.out = q_;
        p.rope_cos = rope_cos_; p.rope_sin = rope_sin_; p.head_dim = hd_; p.n_kv_heads = n_kv_;
        p.k_cache = kc; p.v_cache = vc; p.page_table = page_table_; p.st = st_;
        if (!add_gemv(p, qkv, 3, false, n_embd_, 0)) return {};
        MegaPhase a{};
        a.kind = PH_ATTN; a.g.k_cache = kc; a.g.v_cache = vc;
        ph.push_back(a);
        GemvParams o{};
        const GemvMat mo[1] = {{L.wo.w, L.wo.type, L.wo.rows, L.wo.tile_rows}};
        o.x = attn_; o.epi = EPI_ADD; o.out = x_; o.resid = x_; o.st = st_;
        if (!add_gemv(o, mo, 1, false, n_head_ * hd_, 0)) return {};
        if (L.wgate.type != L.wup.type) return {};
        GemvParams g{};
        const GemvMat mgu[2] = {{L.wgate.w, L.wgate.type, L.wgate.rows, L.wgate.tile_rows}, {L.wup.w, L.wup.type, L.wup.rows, L.wup.tile_rows}};
        g.x = x_; g.norm_w = L.ffn_norm; g.eps = eps_; g.epi = EPI_SILU; g.out = h_; g.st = st_;
        if (!add_gemv(g, mgu, 2, true, n_embd_, 0)) return {};
        GemvParams d{};
        const GemvMat md[1] = {{L.wdown.w, L.wdown.type, L.wdown.rows, L.wdown.tile_rows}};
        d.x = h_; d.epi = EPI_ADD; d.out = x_; d.resid = x_; d.st = st_;
        if (!add_gemv(d, md, 1, false, n_ff_, 0)) return {};
    }
    mega_n_nohead_ = (int)ph.size();
    {
        GemvParams p{};
        const GemvMat mh[1] = {{output_.w, output_.type, output_.rows, output_.tile_rows}};
        p.x = x_; p.norm_w = output_norm_; p.eps = eps_; p.epi = EPI_STORE; p.out = logits_; p.st = st_;
        if (!add_gemv(p, mh, 1, false, n_embd_, PHF_HEAD)) return {};
    }
    mega_n_head_ = (int)ph.size();
    if ((int)mega_prod_.size() > MEGA_MAX_GEMV_PHASES) return {};          // too many layers for the parameter bank: per-op path
    CU(cudaMalloc((void**)&mega_head_, ph.size() * sizeof(MegaPhase)));
    allocs_.push_back(mega_head_);
    CU(cudaMemcpy(mega_head_, ph.data(), ph.size() * sizeof(MegaPhase), cudaMemcpyHostToDevice));
    mega_nohead_ = mega_head_;          // same table, shorter count
    CU(cudaMalloc((void**)&bar_counter_, 64));
    allocs_.push_back(bar_counter_);
    CU(cudaMemset(bar_counter_, 0, 64));
    CU(cudaMalloc((void**)&head_part_, (size_t)sm_count_ * 16));
    allocs_.push_back(head_part_);
    CU(cudaMemset(head_part_, 0, (size_t)sm_count_ * 16));
    if (env_int("GL_MEGA_TRACE", 0)) {
        const size_t n = (size_t)sm_count_ * (mega_n_head_ + 1) * 4;
        CU(cudaMalloc((void**)&mega_trace_, n * 8));
        allocs_.push_back(mega_trace_);
        CU(cudaMemset(mega_trace_, 0, n * 8));
    }
    use_mega_ = true;
    launches_head_ = 1;
    launches_nohead_ = 1;
    return {};
}

Status Engine::launch_mega(int n_steps, bool with_head, bool keep_logits) {
    MegaParams mp{};
    mp.phases = mega_head_;
    mp.n_phases = with_head ? mega_n_head_ : mega_n_nohead_;
    mp.n_steps = n_steps;
    mp.with_head = with_head ? 1 : 0;
    mp.st = st_; mp.bar_counter = bar_counter_; mp.prompt_ids = prompt_ids_;
    mp.embd_w = tok_embd_.w; mp.embd_type = tok_embd_.type; mp.embd_row_bytes = tok_embd_.row_stride; mp.n_embd = n_embd_;
    mp.x = x_; mp.q = q_; mp.attn_out = attn_; mp.part_o = part_o_; mp.part_ml = part_ml_; mp.attn_counters = counters_;
    mp.page_table = page_table_;
    mp.n_head = n_head_; mp.n_kv = n_kv_; mp.head_dim = hd_;
    mp.attn_splits = mega_splits_;
    mp.attn_scale = 1.0f / std::sqrt((float)hd_);
    mp.logits = logits_; mp.head_part = head_part_; mp.out_ids = out_ids_; mp.out_logprobs = out_lp_;
    mp.logits_keep = keep_logits ? logits_keep_ : nullptr;
    mp.max_out = keep_logits ? keep_cap_ : max_out_;
    mp.n_tracks = mega_tracks_; mp.depth = mega_depth_; mp.slot_bytes = mega_slot_bytes_; mp.max_cols = mega_max_cols_;
    mp.trace = with_head ? mega_trace_ : nullptr;
    // producer descriptors: all GEMV phases of the token; the head phase is the last entry
    mp.n_prod = with_head ? (int)mega_prod_.size() : (int)mega_prod_.size() - 1;
    std::memcpy(mp.prod, mega_prod_.data(), mega_prod_.size() * sizeof(ProdDesc));
    CU(mega_launch(mp, abits_, nw_, sm_count_, stream_));
    ++mega_launches_;
    return {};
}

// -------------------------------------------------------------------------------------------------
// drivers
// -------------------------------------------------------------------------------------------------
Status Engine::generate(const int32_t* prompt, int n_prompt, const gl_sample_opts& so, gl_token_cb cb, void* user,
                        int32_t* out_ids, float* out_lp, gl_gen_stats* stats) {
    CU(cudaSetDevice(device_));
    const int64_t t0 = now_ns();
    if (n_prompt <= 0 || !prompt) return fail(GL_ERR_INVALID, "empty prompt");
    const int n_pred = so.num_predict > 0 ? so.num_predict : 128;     // OllamaService.ts:105
    DrawPlan plan;
    ST(plan_draw(so, true, &plan));
    for (int i = 0; i < n_prompt; ++i)
        if (prompt[i] < 0 || prompt[i] >= n_vocab_) return fail(GL_ERR_INVALID, "prompt token id out of range");
    // prefix reuse: keep the pages of the positions the previous request left final and that this prompt repeats
    const int reuse = (prefix_cache_ && !use_mega_) ? prefix_reuse(prompt, n_prompt, cached_ids_.data(), (int)cached_ids_.size(), prefill_min_) : 0;
    if (reuse > 0) {
        cached_ids_.clear();                         // rebuilt below once this request's K / V are final
        host_pos_ = reuse;
    } else {
        ST(kv_reset());
    }
    ST(ensure_pages(n_prompt + n_pred));
    if (so.want_logits) {
        if (keep_cap_ < n_pred) {
            float* p = nullptr;
            CU(cudaMalloc((void**)&p, (size_t)n_pred * n_vocab_ * 4));
            allocs_.push_back(p);
            logits_keep_ = p;
            keep_cap_ = n_pred;
            for (auto& v : g_head_var_)
                for (auto& k : v[1])
                    for (auto& g : k)
                        if (g) { cudaGraphExecDestroy(g); g = nullptr; }      // captured with the old logits buffer
        }
    }
    // the whole prompt is the penalty history, whatever part of it is reused
    CU(cudaMemcpyAsync(prompt_ids_, prompt, (size_t)n_prompt * 4, cudaMemcpyHostToDevice, stream_));
    const bool batched = can_batch_prefill(reuse, n_prompt - reuse);
    int prefill_launches = 0;
    const int mega0 = mega_launches_;
    if (batched) {
        // prompt positions [reuse, n_prompt) through the tensor-core path; the sampler then moves pos from T-1 to T
        ST(set_state(n_prompt - 1, prompt[n_prompt - 1], n_prompt, 0, &so, plan));
        CU(cudaEventRecord(ev_[0], stream_));
        ST(prefill_batched(reuse, n_prompt - reuse, &prefill_launches));
        CU(cudaEventRecord(ev_[1], stream_));
    } else {
        // sequential prefill: positions reuse .. n_prompt-2 without a head, then the last prompt token produces token 0
        ST(set_state(reuse, prompt[reuse], n_prompt, 0, &so, plan));
        CU(cudaEventRecord(ev_[0], stream_));
        ST(run_steps(n_prompt - 1 - reuse, 0, false));
        CU(cudaEventRecord(ev_[1], stream_));
        prefill_launches = use_mega_ ? 0 : (n_prompt - 1 - reuse) * launches_nohead_;
    }
    bool first_head_only = batched;

    std::vector<int32_t> ids(n_pred);
    std::vector<float> lps(n_pred);
    int produced = 0, done_reason = 1;
    bool cancelled = false;
    const int chunk = cb ? 8 : 32;
    StepState hs{};
    while (produced < n_pred && !cancelled) {
        const int n = std::min(chunk, n_pred - produced);
        int full = n;
        if (first_head_only) {
            int dummy = 0;
            ST(enqueue_head(stream_, so.want_logits != 0, &dummy));
            full = n - 1;
            first_head_only = false;
        }
        ST(run_steps(0, full, so.want_logits != 0));
        CU(cudaMemcpyAsync(ids.data() + produced, out_ids_ + produced, (size_t)n * 4, cudaMemcpyDeviceToHost, stream_));
        CU(cudaMemcpyAsync(lps.data() + produced, out_lp_ + produced, (size_t)n * 4, cudaMemcpyDeviceToHost, stream_));
        CU(cudaMemcpyAsync(&hs, st_, sizeof(hs), cudaMemcpyDeviceToHost, stream_));
        CU(cudaStreamSynchronize(stream_));
        const int upto = std::min(hs.out_idx, produced + n);
        for (int i = produced; i < upto && !cancelled; ++i) {
            const bool is_stop = hs.done && i == hs.out_idx - 1;
            if (is_stop) break;                  // the stop token itself is not part of the response
            if (cb) {
                const std::string pc = tok_.ok() ? tok_.piece(ids[i]) : std::string();
                if (cb(user, ids[i], lps[i], tok_.ok() ? pc.c_str() : nullptr, (int32_t)pc.size()) != 0) cancelled = true;
            }
            if (out_ids) out_ids[i] = ids[i];
            if (out_lp) out_lp[i] = lps[i];
            ++produced;
        }
        if (hs.done) { done_reason = 0; break; }
    }
    CU(cudaEventRecord(ev_[2], stream_));
    CU(cudaEventSynchronize(ev_[2]));
    if (cancelled) done_reason = 2;
    host_pos_ = n_prompt + produced;
    if (prefix_cache_ && !use_mega_) {
        // K / V are final for the prompt and for every generated id the device has FED: a step feeds output i - 1 while it draws
        // output i, so hs.out_idx draws fed hs.out_idx - 1 of them.  The last draw (and a stop token) was never fed; steps the
        // device ran past what the host reported (a cancel mid-chunk, a stop) fed ids the host did not record and stay out.
        const int fed = std::max(0, std::min(produced, hs.out_idx - 1));
        cached_ids_.assign(prompt, prompt + n_prompt);
        cached_ids_.insert(cached_ids_.end(), ids.begin(), ids.begin() + fed);
    }
    if (stats) {
        float ms_p = 0.f, ms_d = 0.f;
        cudaEventElapsedTime(&ms_p, ev_[0], ev_[1]);
        cudaEventElapsedTime(&ms_d, ev_[1], ev_[2]);
        stats->prompt_eval_count = n_prompt - reuse;
        stats->eval_count = produced;
        stats->prompt_eval_duration_ns = (int64_t)(ms_p * 1e6);
        stats->eval_duration_ns = (int64_t)(ms_d * 1e6);
        stats->total_duration_ns = now_ns() - t0;
        stats->load_duration_ns = load_ns_;
        stats->done_reason = done_reason;
        stats->kernel_launches = use_mega_ ? prefill_launches + (mega_launches_ - mega0) + (batched ? 2 : 0)
                                           : prefill_launches + std::max(produced, 1) * head_launches();
    }
    return cancelled ? fail(GL_ERR_CANCELLED, "cancelled by token callback") : Status{};
}

Status Engine::last_logits(int step, float* out, int n_vocab) {
    if (!logits_keep_ || step < 0 || step >= keep_cap_ || n_vocab != n_vocab_) return fail(GL_ERR_INVALID, "no kept logits for that step");
    CU(cudaMemcpy(out, logits_keep_ + (size_t)step * n_vocab_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost));
    return {};
}

// The sampler alone on caller-supplied logits (parity tests of the draw against oracle/sampler.py).  Rewinds the sequence.
Status Engine::sample_logits(const float* logits, int n_vocab, const gl_sample_opts& so, int out_index, int* id, float* logprob) {
    CU(cudaSetDevice(device_));
    if (!logits || n_vocab != n_vocab_) return fail(GL_ERR_INVALID, "logits must hold n_vocab values");
    if (out_index < 0 || out_index >= max_out_) return fail(GL_ERR_INVALID, "output index out of range");
    gl_sample_opts o = so;
    o.ignore_eos = 1;
    o.format = 0;                                      // the sampler alone: the format is not looked at
    DrawPlan plan;
    ST(plan_draw(o, false, &plan));
    ST(kv_reset());
    ST(set_state(0, 0, 0, out_index, &o, plan));
    CU(cudaMemcpyAsync(logits_, logits, (size_t)n_vocab_ * 4, cudaMemcpyHostToDevice, stream_));
    SampleParams sp{logits_, n_vocab_, st_, out_ids_, out_lp_, nullptr, max_out_, sample_scratch_, topk_scratch_};
    if (plan.sampler != 0) CU(sample_topk_launch(sp, plan.sampler == 1, false, stream_));
    else CU(sample_greedy_launch(sp, false, stream_));
    int tid = 0;
    float lp = 0.f;
    CU(cudaMemcpyAsync(&tid, out_ids_ + out_index, 4, cudaMemcpyDeviceToHost, stream_));
    CU(cudaMemcpyAsync(&lp, out_lp_ + out_index, 4, cudaMemcpyDeviceToHost, stream_));
    CU(cudaStreamSynchronize(stream_));
    ST(kv_reset());
    if (id) *id = tid;
    if (logprob) *logprob = lp;
    return {};
}

// The penalty kernel alone on caller-supplied logits with a caller-supplied history (parity tests against tests/penalty_oracle.py):
// the history is the "prompt" of a sequence that has drawn nothing yet.  Rewinds the sequence.
Status Engine::penalize_logits(float* logits, int n_vocab, const gl_sample_opts& so, const int32_t* history, int n_history) {
    CU(cudaSetDevice(device_));
    if (!logits || n_vocab != n_vocab_) return fail(GL_ERR_INVALID, "logits must hold n_vocab values");
    if (n_history < 0 || (n_history > 0 && !history)) return fail(GL_ERR_INVALID, "bad history");
    for (int i = 0; i < n_history; ++i)
        if (history[i] < 0 || history[i] >= n_vocab_) return fail(GL_ERR_INVALID, "history token id out of range");
    gl_sample_opts o = so;
    o.ignore_eos = 1;
    o.temperature = 0.f;                               // the penalty kernel alone: no draw and no mask
    o.format = 0;
    DrawPlan plan;
    ST(plan_draw(o, false, &plan));
    ST(kv_reset());
    ST(set_state(0, 0, n_history, 0, &o, plan));
    int* hist = nullptr;
    if (n_history > 0) CU(cudaMalloc((void**)&hist, (size_t)n_history * 4));
    Status rs;
    do {
        cudaError_t ce = hist ? cudaMemcpyAsync(hist, history, (size_t)n_history * 4, cudaMemcpyHostToDevice, stream_) : cudaSuccess;
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(logits_, logits, (size_t)n_vocab_ * 4, cudaMemcpyHostToDevice, stream_);
        if (ce == cudaSuccess && hist) ce = enqueue_pre_draw(stream_, 0, plan.penalised, false, hist);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(logits, logits_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost, stream_);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(stream_);
        if (ce != cudaSuccess) rs = fail(GL_ERR_CUDA, std::string("penalize_logits: ") + cudaGetErrorString(ce));
    } while (false);
    if (hist) cudaFree(hist);
    ST(rs);
    return kv_reset();
}

// ---- JSON grammar mask (schema_mask.cu) ------------------------------------------------------------------------------
// The vocabulary table the mask kernel reads, built once at the first JSON request.  The vocabulary must guarantee that every
// state the automaton can reach has an allowed token, so that the mask never leaves a draw with nothing: a single-byte piece for
// each of \t, \n and 0x20-0x7E (all of them ordinary tokens, not stop tokens), one for each of 0x80-0xBF as soon as some piece
// is not whole well-formed UTF-8 (a string can then stop inside a character), and an eos token to end on.
Status Engine::ensure_json() {
    if (json_checked_) return json_refused_.empty() ? Status{} : fail(GL_ERR_UNSUPPORTED, json_refused_);
    json_checked_ = true;
    if (!tok_.ok()) json_refused_ = "format json: the model carries no tokenizer";
    else if (tok_.eos < 0) json_refused_ = "format json: the vocabulary has no eos token to end a document on";
    if (!json_refused_.empty()) return fail(GL_ERR_UNSUPPORTED, json_refused_);
    std::vector<uint32_t> off(n_vocab_ + 1, 0);
    std::vector<uint8_t> bytes, cls(n_vocab_, 0);
    bool single[256] = {};
    bool partial_utf8 = false;
    for (int t = 0; t < n_vocab_; ++t) {
        const std::string pc = tok_.piece(t);
        off[t] = (uint32_t)bytes.size();
        bytes.insert(bytes.end(), pc.begin(), pc.end());
        bool plain = !pc.empty();
        for (unsigned char c : pc) plain = plain && c >= 0x20 && c <= 0x7E && c != '"' && c != '\\';
        cls[t] = plain ? JSON_CLS_PLAIN : 0;
        if (pc.size() == 1 && t != tok_.eos && t != tok_.eot) single[(unsigned char)pc[0]] = true;
        // whole well-formed UTF-8?  (the string-body automaton from its own state accepts it and ends outside a character)
        JsonState u{};
        u.mode = JM_STR;
        bool whole = true;
        for (unsigned char c : pc)      // (quotes, backslashes and control bytes stand in for one plain character here)
            if (!json_step(u, (c == '"' || c == '\\' || c < 0x20) ? (uint8_t)'a' : (uint8_t)c)) { whole = false; break; }
        if (!whole || u.mode != JM_STR) partial_utf8 = true;
    }
    off[n_vocab_] = (uint32_t)bytes.size();
    std::string missing;
    auto need = [&](int b) {
        if (!single[b]) {
            char buf[8];
            snprintf(buf, sizeof buf, "0x%02X", b);
            missing += (missing.empty() ? "" : ", ") + std::string(buf);
        }
    };
    need('\t');
    need('\n');
    for (int b = 0x20; b <= 0x7E; ++b) need(b);
    if (partial_utf8)
        for (int b = 0x80; b <= 0xBF; ++b) need(b);
    if (!missing.empty()) {
        json_refused_ = "format json: the vocabulary has no single-byte token for byte(s) " + missing +
                        ", so a JSON continuation cannot be guaranteed";
        return fail(GL_ERR_UNSUPPORTED, json_refused_);
    }
    uint32_t* d_off = nullptr;
    uint8_t *d_bytes = nullptr, *d_cls = nullptr;
    CU(cudaMalloc((void**)&d_off, off.size() * 4));
    allocs_.push_back(d_off);
    CU(cudaMalloc((void**)&d_bytes, std::max<size_t>(bytes.size(), 1)));
    allocs_.push_back(d_bytes);
    CU(cudaMalloc((void**)&d_cls, cls.size()));
    allocs_.push_back(d_cls);
    CU(cudaMemcpy(d_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    if (!bytes.empty()) CU(cudaMemcpy(d_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_cls, cls.data(), cls.size(), cudaMemcpyHostToDevice));
    json_off_ = d_off; json_bytes_ = d_bytes; json_cls_ = d_cls;
    json_hoff_ = std::move(off);
    json_hbytes_ = std::move(bytes);
    return {};
}

bool Engine::json_stop(const gl_sample_opts& so, int32_t id) const {
    const StepState h = make_state(0, 0, 0, 0, &so);      // the stop ids the device sees
    for (int k = 0; k < h.n_stop; ++k)
        if (h.stop_ids[k] == id) return true;
    return false;
}

// The automaton through a caller-supplied output history, then the mask kernel alone on caller-supplied logits (parity tests
// against tests/json_oracle.py).  Rewinds the sequence.
Status Engine::constrain_logits(float* logits, int n_vocab, const gl_sample_opts& so, const int32_t* generated, int n_generated) {
    CU(cudaSetDevice(device_));
    if (!logits || n_vocab != n_vocab_) return fail(GL_ERR_INVALID, "logits must hold n_vocab values");
    if (n_generated < 0 || (n_generated > 0 && !generated)) return fail(GL_ERR_INVALID, "bad history");
    if (n_generated >= max_out_) return fail(GL_ERR_INVALID, "history longer than an output");
    for (int i = 0; i < n_generated; ++i)
        if (generated[i] < 0 || generated[i] >= n_vocab_) return fail(GL_ERR_INVALID, "history token id out of range");
    gl_sample_opts o = so;
    o.ignore_eos = 0;
    o.temperature = 0.f;                               // the mask alone: no draw
    if (o.format == 0) return {};                      // off: the logits stay as they are
    DrawPlan plan;
    ST(plan_draw(o, false, &plan));
    // the history must be a prefix the mask allows: no stop token (it would have ended the output), no control token, every
    // byte accepted
    SchemaState ss;
    SchemaArrayFrames sf{ss.fr};
    const SchemaView sv = schema_view(o.format == GL_FORMAT_JSON ? json_blob_.data() : schemas_[o.format].blob.data());
    schema_init(ss.js, ss.cur, sv);
    for (int i = 0; i < n_generated; ++i) {
        const int32_t t = generated[i];
        const uint32_t a = json_hoff_[t], b = json_hoff_[t + 1];
        const bool ok = schema_run(sv, ss.js, ss.cur, sf, json_hbytes_.data() + a, (int)(b - a));
        if (json_stop(o, t) || a == b || !ok)
            return fail(GL_ERR_INVALID, "format json: the history is not a prefix the grammar allows (token " + std::to_string(i) + ")");
    }
    ST(kv_reset());
    ST(set_state(0, n_generated > 0 ? generated[n_generated - 1] : 0, 0, n_generated, &o, plan));
    int* hist = nullptr;
    if (n_generated > 0) CU(cudaMalloc((void**)&hist, (size_t)n_generated * 4));
    Status rs;
    do {
        cudaError_t ce = hist ? cudaMemcpyAsync(hist, generated, (size_t)n_generated * 4, cudaMemcpyHostToDevice, stream_) : cudaSuccess;
        if (ce == cudaSuccess && hist) ce = schema_replay_launch(sch_, hist, n_generated, json_off_, json_bytes_, stream_);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(logits_, logits, (size_t)n_vocab_ * 4, cudaMemcpyHostToDevice, stream_);
        if (ce == cudaSuccess) ce = enqueue_pre_draw(stream_, 0, false, true);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(logits, logits_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost, stream_);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(stream_);
        if (ce != cudaSuccess) rs = fail(GL_ERR_CUDA, std::string("constrain_logits: ") + cudaGetErrorString(ce));
    } while (false);
    if (hist) cudaFree(hist);
    ST(rs);
    return kv_reset();
}

// ---- JSON schemas (schema_compile.cpp, schema_mask.cu) ---------------------------------------------------------------------
Status Engine::ensure_schema_state() {
    if (sch_) return {};
    std::vector<uint8_t> blob;
    std::string err;
    static const char kAnyObject[] = "{\"type\":\"object\"}";
    if (schema_compile(kAnyObject, sizeof kAnyObject - 1, blob, err) != GL_OK) return fail(GL_ERR_INVALID, err);
    SchemaSlot* d = nullptr;
    uint8_t* t = nullptr;
    const size_t bytes = sizeof(SchemaSlot) * (1 + MAX_BATCH);
    CU(cudaMalloc((void**)&d, bytes));
    allocs_.push_back(d);
    CU(cudaMalloc((void**)&t, blob.size()));
    allocs_.push_back(t);
    CU(cudaMemset(d, 0, bytes));
    CU(cudaMemcpy(t, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    sch_ = d;
    json_tab_ = t;
    json_blob_ = std::move(blob);
    return {};
}

SchemaSlot* Engine::schema_entry() const {
    return (bst_ && st_ >= bst_ && st_ < bst_ + MAX_BATCH) ? sch_ + 1 + (st_ - bst_) : sch_;
}

Status Engine::schema_bind(SchemaSlot* e, int format) {
    const uint8_t* const* tab = &json_tab_;
    if (format != GL_FORMAT_JSON) {
        auto it = schemas_.find(format);
        if (it == schemas_.end()) return fail(GL_ERR_INVALID, "format: unknown or evicted schema code " + std::to_string(format));
        tab = &it->second.dev;
    }
    CU(cudaMemcpyAsync(&e->tab, tab, sizeof(*tab), cudaMemcpyHostToDevice, stream_));
    CU(cudaStreamSynchronize(stream_));
    return {};
}

// Compile and register a schema: identical text gives the code it got before.  The vocabulary must carry a single-byte token
// for every byte of the keys and enum members (beside what ensure_json asks), so that a literal can always be continued.
Status Engine::format_schema(const char* text, int n, int* code) {
    CU(cudaSetDevice(device_));
    if (!text || n < 0 || !code) return fail(GL_ERR_INVALID, "gl_format_schema: bad argument");
    const std::string key(text, (size_t)n);
    auto hit = schema_codes_.find(key);
    if (hit != schema_codes_.end()) {
        schemas_[hit->second].used = ++schema_clock_;
        *code = hit->second;
        return {};
    }
    SchemaEntry en;
    en.text = key;
    std::string err;
    const int rc = schema_compile(text, (size_t)n, en.blob, err);
    if (rc != GL_OK) return fail(rc, err);
    ST(ensure_json());
    bool single[256] = {};
    for (int t = 0; t < n_vocab_; ++t)
        if (json_hoff_[t + 1] - json_hoff_[t] == 1 && t != tok_.eos && t != tok_.eot) single[json_hbytes_[json_hoff_[t]]] = true;
    const SchemaHeader* h = reinterpret_cast<const SchemaHeader*>(en.blob.data());
    const uint32_t* lo = reinterpret_cast<const uint32_t*>(en.blob.data() + h->off_lit_off);
    for (uint32_t i = h->off_lit; i < h->off_lit + lo[h->n_lits]; ++i)
        if (!single[en.blob[i]]) {
            char buf[8];
            snprintf(buf, sizeof buf, "0x%02X", en.blob[i]);
            return fail(GL_ERR_UNSUPPORTED, std::string("format schema: the vocabulary has no single-byte token for byte ") + buf +
                                                " of a key or enum member, so a continuation cannot be guaranteed");
        }
    if ((int)schemas_.size() >= SCHEMA_CACHE) {                 // evict the least recently used schema no open sequence uses
        int victim = -1;
        uint64_t oldest = UINT64_MAX;
        for (auto& kv : schemas_) {
            bool in_use = false;
            for (auto& S : slots_) in_use = in_use || (S.open && S.plan.format == kv.first);
            if (!in_use && kv.second.used < oldest) { oldest = kv.second.used; victim = kv.first; }
        }
        if (victim < 0) return fail(GL_ERR_NOMEM, "format schema: all 64 registered schemas are in use by open sequences");
        cudaFree(schemas_[victim].dev);
        schema_codes_.erase(schemas_[victim].text);
        schemas_.erase(victim);
    }
    CU(cudaMalloc((void**)&en.dev, en.blob.size()));
    const cudaError_t ce = cudaMemcpy(en.dev, en.blob.data(), en.blob.size(), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { cudaFree(en.dev); CU(ce); }
    en.used = ++schema_clock_;
    const int c = next_schema_++;
    schema_codes_[key] = c;
    schemas_[c] = std::move(en);
    *code = c;
    return {};
}

Status Engine::decode_step(int token, float* logits, int* argmax, float* logprob) {
    CU(cudaSetDevice(device_));
    if (token < 0 || token >= n_vocab_) return fail(GL_ERR_INVALID, "token id out of range");
    cached_ids_.clear();                              // the pages and the step state are now this call's: no prefix reuse
    ST(ensure_pages(host_pos_ + 1));
    gl_sample_opts so{};
    so.ignore_eos = 1;
    ST(set_state(host_pos_, token, 0, 0, &so));
    ST(run_steps(0, 1, false));
    int id = 0;
    float lp = 0.f;
    CU(cudaMemcpyAsync(&id, out_ids_, 4, cudaMemcpyDeviceToHost, stream_));
    CU(cudaMemcpyAsync(&lp, out_lp_, 4, cudaMemcpyDeviceToHost, stream_));
    if (logits) CU(cudaMemcpyAsync(logits, logits_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost, stream_));
    CU(cudaStreamSynchronize(stream_));
    if (argmax) *argmax = id;
    if (logprob) *logprob = lp;
    ++host_pos_;
    return {};
}

Status Engine::prefill(const int32_t* ids, int n, float* last_logits) {
    CU(cudaSetDevice(device_));
    if (n <= 0) return fail(GL_ERR_INVALID, "empty prefill");
    for (int i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= n_vocab_) return fail(GL_ERR_INVALID, "token id out of range");
    cached_ids_.clear();                              // the pages and the step state are now this call's: no prefix reuse
    ST(ensure_pages(host_pos_ + n));
    gl_sample_opts so{};
    so.ignore_eos = 1;
    // both paths read the tokens from prompt_ids_ indexed by absolute position
    CU(cudaMemcpyAsync(prompt_ids_ + host_pos_, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
    if (can_batch_prefill(host_pos_, n)) {
        // positions [host_pos_, host_pos_ + n) on the tensor cores, attending to everything before them through the pages
        int dummy = 0;
        ST(set_state(host_pos_ + n - 1, ids[n - 1], host_pos_ + n, 0, &so));
        ST(prefill_batched(host_pos_, n, &dummy));
        ST(enqueue_head(stream_, false, &dummy));
    } else {
        // sequential prefill
        ST(set_state(host_pos_, ids[0], host_pos_ + n, 0, &so));
        ST(run_steps(n - 1, 1, false));
    }
    if (last_logits) CU(cudaMemcpyAsync(last_logits, logits_, (size_t)n_vocab_ * 4, cudaMemcpyDeviceToHost, stream_));
    CU(cudaStreamSynchronize(stream_));
    host_pos_ += n;
    return {};
}

// generateEmbedding (/root/reference/client/src/services/OllamaService.ts:601-665; the batched form is `input: string[]` of
// /api/embed, server/src/routes/ollama.ts:574-643): prompt pass only -> output_norm -> mean over positions -> L2 normalise.
// The sequences of a call are PACKED: up to EMB_PACK_TOKENS rows share one pass over the layers (engine_prefill.cu
// prefill_packed), each sequence attending only to itself.  No allocation per call (buffers grow on demand and stay), the
// device time in the stats is bracketed by events around device work only.
Status Engine::embed(const int32_t* ids, const int32_t* offs, int n_seq, float* out, gl_gen_stats* stats) {
    CU(cudaSetDevice(device_));
    const int64_t t0 = now_ns();
    int total = 0, launches = 0, max_n = 0;
    for (int sidx = 0; sidx < n_seq; ++sidx) {
        const int n = offs[sidx + 1] - offs[sidx];
        if (n <= 0) return fail(GL_ERR_INVALID, "empty sequence in gl_embed");
        if (n > n_ctx_) return fail(GL_ERR_CONTEXT, "sequence of " + std::to_string(n) + " tokens exceeds the engine context " + std::to_string(n_ctx_));
        for (int i = 0; i < n; ++i)
            if (ids[offs[sidx] + i] < 0 || ids[offs[sidx] + i] >= n_vocab_) return fail(GL_ERR_INVALID, "token id out of range");
        max_n = std::max(max_n, n);
        total += n;
    }
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess) allocs_.push_back(*p);
        return e;
    };
    if (!pk_ids_) {
        CU(dalloc((void**)&pk_ids_, (size_t)EMB_PACK_TOKENS * 4));
        CU(dalloc((void**)&emb_pooled_, (size_t)n_embd_ * 4));
        CU(dalloc((void**)&emb_rstd_, (size_t)std::max(EMB_PACK_TOKENS, n_ctx_) * 4));
    }
    if (n_seq > emb_out_cap_) {                            // grows, never shrinks; the old buffer stays in allocs_ until the engine goes
        CU(cudaStreamSynchronize(stream_));
        CU(dalloc((void**)&emb_out_, (size_t)n_seq * n_embd_ * 4));
        emb_out_cap_ = n_seq;
    }
    const bool packed = have_w16_ && prefill_mode_ != 1;
    float* d_rows = nullptr;                               // sequential path only
    CU(cudaEventRecord(ev_[0], stream_));
    if (packed) {
        // greedy packing in call order; every sequence starts on a 128-row boundary (pad rows hold token 0 and are never read back)
        int sidx = 0;
        std::vector<int32_t> h_ids(EMB_PACK_TOKENS);
        while (sidx < n_seq) {
            std::vector<int> starts, lens, which;
            int rows = 0;
            std::fill(h_ids.begin(), h_ids.end(), 0);
            while (sidx < n_seq) {
                const int n = offs[sidx + 1] - offs[sidx], lp = (n + 127) / 128 * 128;
                if (n > EMB_PACK_TOKENS) break;            // longer than a pack: handled alone below
                if (rows + lp > EMB_PACK_TOKENS) break;
                starts.push_back(rows); lens.push_back(n); which.push_back(sidx);
                std::memcpy(h_ids.data() + rows, ids + offs[sidx], (size_t)n * 4);
                rows += lp;
                ++sidx;
            }
            if (starts.empty()) {                          // one sequence longer than a pack: the single-sequence batched pass
                const int n = offs[sidx + 1] - offs[sidx];
                ST(kv_reset());
                ST(ensure_pages(n));
                CU(cudaMemcpyAsync(prompt_ids_, ids + offs[sidx], (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
                gl_sample_opts so{};
                so.ignore_eos = 1;
                ST(set_state(0, ids[offs[sidx]], n, 0, &so));
                if (!can_batch_prefill(0, n)) return fail(GL_ERR_UNSUPPORTED, "a sequence longer than one prompt pass needs the fused prompt attention");
                if (n <= PF_CHUNK) {
                    ST(prefill_batched(0, n, &launches));
                    CU(pool_embedding_launch(pf_x_, n, n_embd_, output_norm_, eps_, emb_rstd_, emb_pooled_, emb_out_ + (size_t)sidx * n_embd_, stream_));
                    launches += 3;
                } else {
                    // passes of PF_CHUNK rows (each attends to the earlier ones through the pages); the pooling sums the
                    // normalised columns of every pass, then scales and L2-normalises once
                    for (int c0 = 0; c0 < n; c0 += PF_CHUNK) {
                        const int len = std::min(PF_CHUNK, n - c0);
                        ST(prefill_chunk(c0, len, &launches));
                        CU(pool_embedding_sum_launch(pf_x_, len, n_embd_, eps_, emb_rstd_, emb_pooled_, c0 > 0, stream_));
                        launches += 2;
                    }
                    CU(pool_embedding_finish_launch(emb_pooled_, n, n_embd_, output_norm_, emb_out_ + (size_t)sidx * n_embd_, stream_));
                    launches += 2;
                }
                ++sidx;
                continue;
            }
            CU(cudaMemcpyAsync(pk_ids_, h_ids.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, stream_));      // pageable source: staged before return
            ST(prefill_packed(starts, lens, rows, &launches));
            for (size_t i = 0; i < starts.size(); ++i) {
                CU(pool_embedding_launch(pf_x_ + (size_t)starts[i] * n_embd_, lens[i], n_embd_, output_norm_, eps_, emb_rstd_, emb_pooled_,
                                         emb_out_ + (size_t)which[i] * n_embd_, stream_));
                launches += 3;
            }
        }
    } else {
        // no 16-bit copy (prefill_mode 1 / not enough HBM): every sequence steps through the decode kernels, hidden state kept per position
        CU(cudaMalloc((void**)&d_rows, (size_t)max_n * n_embd_ * 4));
        Status st;
        for (int sidx = 0; sidx < n_seq && st.ok(); ++sidx) {
            const int n = offs[sidx + 1] - offs[sidx];
            const int32_t* sid = ids + offs[sidx];
            st = kv_reset();
            if (st.ok()) st = ensure_pages(n);
            if (!st.ok()) break;
            cudaMemcpyAsync(prompt_ids_, sid, (size_t)n * 4, cudaMemcpyHostToDevice, stream_);
            gl_sample_opts so{};
            so.ignore_eos = 1;
            st = set_state(0, sid[0], n, 0, &so);
            for (int i = 0; i < n && st.ok(); ++i) {
                st = run_steps(1, 0, false);
                cudaMemcpyAsync(d_rows + (size_t)i * n_embd_, x_, (size_t)n_embd_ * 4, cudaMemcpyDeviceToDevice, stream_);
            }
            launches += n * launches_nohead_;
            if (st.ok()) {
                cudaError_t ae = pool_embedding_launch(d_rows, n, n_embd_, output_norm_, eps_, emb_rstd_, emb_pooled_, emb_out_ + (size_t)sidx * n_embd_, stream_);
                if (ae != cudaSuccess) st = fail(GL_ERR_CUDA, cudaGetErrorString(ae));
                launches += 3;
            }
        }
        if (!st.ok()) { cudaStreamSynchronize(stream_); cudaFree(d_rows); return st; }
    }
    CU(cudaEventRecord(ev_[1], stream_));
    cudaError_t ae = cudaMemcpyAsync(out, emb_out_, (size_t)n_seq * n_embd_ * 4, cudaMemcpyDeviceToHost, stream_);
    if (ae == cudaSuccess) ae = cudaStreamSynchronize(stream_);
    if (d_rows) cudaFree(d_rows);
    CU(ae);
    if (stats) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev_[0], ev_[1]);
        std::memset(stats, 0, sizeof(*stats));
        stats->prompt_eval_count = total;
        stats->prompt_eval_duration_ns = (int64_t)(ms * 1e6);
        stats->total_duration_ns = now_ns() - t0;
        stats->load_duration_ns = load_ns_;
        stats->kernel_launches = launches;
    }
    return {};
}

Status Engine::rmsnorm(const float* x, const float* w, int n, float eps, float* y) {
    CU(cudaSetDevice(device_));
    float *dx, *dw, *dy;
    CU(cudaMalloc((void**)&dx, (size_t)n * 4));
    CU(cudaMalloc((void**)&dw, (size_t)n * 4));
    CU(cudaMalloc((void**)&dy, (size_t)n * 4));
    cudaMemcpy(dx, x, (size_t)n * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dw, w, (size_t)n * 4, cudaMemcpyHostToDevice);
    cudaError_t e = rmsnorm_launch(dx, dw, n, eps, dy, stream_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream_);
    if (e == cudaSuccess) e = cudaMemcpy(y, dy, (size_t)n * 4, cudaMemcpyDeviceToHost);
    cudaFree(dx); cudaFree(dw); cudaFree(dy);
    CU(e);
    return {};
}

Status Engine::gemv_host(int type, const void* w_host, int rows, int cols, const float* x, float* y, int iters, float* ms) {
    CU(cudaSetDevice(device_));
    if (rows <= 0 || cols <= 0 || !w_host || !x || !y) return fail(GL_ERR_INVALID, "bad gl_gemv arguments");
    GGUFTensor t;
    t.name = "<gl_gemv>";
    t.type = (uint32_t)type;
    t.ne = {cols, rows};
    BlockGeom g = block_geom(t.type);
    if (!g.weights || cols % g.weights) return fail(GL_ERR_UNSUPPORTED, "gl_gemv: unsupported type / cols");
    t.data = static_cast<const uint8_t*>(w_host);
    t.nbytes = row_bytes(t.type, cols) * (size_t)rows;
    DevMatrix m;
    const size_t mark = allocs_.size();
    Status s = upload_matrix(t, m, false);
    float *dx = nullptr, *dy = nullptr;
    auto cleanup = [&]() {
        if (dx) cudaFree(dx);
        if (dy) cudaFree(dy);
        while (allocs_.size() > mark) { cudaFree(allocs_.back()); allocs_.pop_back(); }
    };
    if (!s.ok()) { cleanup(); return s; }
    cudaError_t e = cudaMalloc((void**)&dx, (size_t)cols * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&dy, (size_t)rows * 4);
    if (e == cudaSuccess) e = cudaMemcpy(dx, x, (size_t)cols * 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cleanup(); CU(e); }
    int nl = 0;
    const int warm = iters > 1 ? 2 : 0;
    for (int i = 0; i < warm && s.ok(); ++i) s = plain_gemv(stream_, m, dx, dy, &nl);
    if (s.ok()) {
        cudaEventRecord(ev_[0], stream_);
        for (int i = 0; i < std::max(1, iters) && s.ok(); ++i) s = plain_gemv(stream_, m, dx, dy, &nl);
        cudaEventRecord(ev_[1], stream_);
        e = cudaStreamSynchronize(stream_);
        if (s.ok() && e != cudaSuccess) s = fail(GL_ERR_CUDA, std::string("gl_gemv: ") + cudaGetErrorString(e));
    }
    if (s.ok()) {
        float t_ms = 0.f;
        cudaEventElapsedTime(&t_ms, ev_[0], ev_[1]);
        if (ms) *ms = t_ms / std::max(1, iters);
        e = cudaMemcpy(y, dy, (size_t)rows * 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) s = fail(GL_ERR_CUDA, cudaGetErrorString(e));
    }
    cleanup();
    return s;
}

Status Engine::gemv_tensor(const std::string& name, const float* x, float* y, int iters, int flush, float* ms, uint64_t* wbytes) {
    CU(cudaSetDevice(device_));
    const DevMatrix* m = find_matrix(name);
    if (!m) return fail(GL_ERR_INVALID, "no such matrix: " + name);
    float *dx = nullptr, *dy = nullptr;
    CU(cudaMalloc((void**)&dx, (size_t)m->cols * 4));
    CU(cudaMalloc((void**)&dy, (size_t)m->rows * 4));
    CU(cudaMemcpy(dx, x, (size_t)m->cols * 4, cudaMemcpyHostToDevice));
    if (flush && !flush_buf_) {
        flush_elems_ = (size_t)64 << 20;     // 256 MB > 50 MB L2
        CU(cudaMalloc((void**)&flush_buf_, flush_elems_ * 4));
        allocs_.push_back(flush_buf_);
        CU(cudaMemset(flush_buf_, 0, flush_elems_ * 4));
    }
    int nl = 0;
    Status s;
    for (int i = 0; i < 3 && s.ok(); ++i) s = plain_gemv(stream_, *m, dx, dy, &nl);
    double tot = 0;
    for (int i = 0; i < std::max(1, iters) && s.ok(); ++i) {
        if (flush) l2_flush_launch(flush_buf_, flush_elems_, stream_);
        cudaEventRecord(ev_[0], stream_);
        s = plain_gemv(stream_, *m, dx, dy, &nl);
        cudaEventRecord(ev_[1], stream_);
        cudaError_t e = cudaStreamSynchronize(stream_);
        if (s.ok() && e != cudaSuccess) s = fail(GL_ERR_CUDA, cudaGetErrorString(e));
        float t_ms = 0.f;
        cudaEventElapsedTime(&t_ms, ev_[0], ev_[1]);
        tot += t_ms;
    }
    if (s.ok()) {
        if (ms) *ms = (float)(tot / std::max(1, iters));
        if (wbytes) *wbytes = m->gguf_bytes;
        cudaError_t e = cudaMemcpy(y, dy, (size_t)m->rows * 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) s = fail(GL_ERR_CUDA, cudaGetErrorString(e));
    }
    cudaFree(dx);
    cudaFree(dy);
    return s;
}

Status Engine::perop_trace(unsigned long long* out, int cap, int* n_launches) {
    if (!perop_trace_) return fail(GL_ERR_UNSUPPORTED, "trace not enabled (GL_TRACE=1)");
    if (cap < PEROP_TRACE_LAUNCHES * 16) return fail(GL_ERR_INVALID, "trace buffer too small");
    CU(cudaMemcpy(out, perop_trace_, (size_t)PEROP_TRACE_LAUNCHES * 16 * 8, cudaMemcpyDeviceToHost));
    *n_launches = launches_head_;
    CU(cudaMemset(perop_trace_, 0, (size_t)PEROP_TRACE_LAUNCHES * 16 * 8));      // the atomicMax slots start from zero again
    return {};
}

Status Engine::mega_trace(unsigned long long* out, int cap, int* n_ctas, int* n_phases) {
    if (!mega_trace_) return fail(GL_ERR_UNSUPPORTED, "trace not enabled (GL_MEGA_TRACE=1)");
    const size_t n = (size_t)sm_count_ * (mega_n_head_ + 1) * 4;
    if ((size_t)cap < n) return fail(GL_ERR_INVALID, "trace buffer too small");
    CU(cudaMemcpy(out, mega_trace_, n * 8, cudaMemcpyDeviceToHost));
    *n_ctas = sm_count_;
    *n_phases = mega_n_head_;
    return {};
}

Status Engine::time_decode(int ctx_len, int iters, float* ms, int* launches) {
    CU(cudaSetDevice(device_));
    if (ctx_len < 1 || iters < 1) return fail(GL_ERR_INVALID, "bad arguments");
    ST(kv_reset());
    ST(ensure_pages(ctx_len + iters + 4));
    gl_sample_opts so{};
    so.ignore_eos = 1;
    ST(set_state(ctx_len - 1, 1 % n_vocab_, 0, 0, &so));
    ST(run_steps(0, 3, false));                       // warm-up
    ST(set_state(ctx_len - 1, 1 % n_vocab_, 0, 0, &so));
    CU(cudaEventRecord(ev_[0], stream_));
    ST(run_steps(0, iters, false));
    CU(cudaEventRecord(ev_[1], stream_));
    CU(cudaEventSynchronize(ev_[1]));
    float t_ms = 0.f;
    cudaEventElapsedTime(&t_ms, ev_[0], ev_[1]);
    if (ms) *ms = t_ms / iters;
    if (launches) *launches = launches_head_;
    ST(kv_reset());
    return {};
}

}  // namespace gl
