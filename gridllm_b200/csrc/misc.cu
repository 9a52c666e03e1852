// Small kernels of the decode step: token-embedding row gather (dequantise one row), greedy sampler
// (argmax + log-softmax, advances the device-resident StepState), and the standalone RMSNorm / RoPE+KV
// append / SiLU*mul / add pieces used for fp-weight models and as unfused cross-checks of the fused
// GEMV prologue / epilogues.  Reference call sites: see gemv.cu header.
#include "common.cuh"
#include "kernels.h"
#include "rowdot.h"
#include "gguf_file.h"

namespace gl {

namespace {

__device__ __forceinline__ float dequant_native(const uint8_t* row, int type, int c) {
    switch (type) {
        case T_F32: return reinterpret_cast<const float*>(row)[c];
        case T_F16: return __half2float(reinterpret_cast<const __half*>(row)[c]);
        case T_BF16: return __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(row)[c] << 16);
        case T_Q8_0: {
            const uint8_t* b = row + (size_t)(c >> 5) * 34;
            return half_bits_to_float(*reinterpret_cast<const uint16_t*>(b)) * (float)(int8_t)b[2 + (c & 31)];
        }
        case T_Q4_K: {
            const uint8_t* b = row + (size_t)(c >> 8) * 144;
            const int e = c & 255, sub = e >> 5, l = e & 31;
            const float d = half_bits_to_float(*reinterpret_cast<const uint16_t*>(b));
            const float dmin = half_bits_to_float(*reinterpret_cast<const uint16_t*>(b + 2));
            const uint8_t* sc = b + 4;
            int s, m;
            if (sub < 4) { s = sc[sub] & 63; m = sc[4 + sub] & 63; }
            else { s = (sc[4 + sub] & 0xF) | ((sc[sub - 4] >> 6) << 4); m = (sc[4 + sub] >> 4) | ((sc[sub] >> 6) << 4); }
            const uint8_t qb = b[16 + (sub >> 1) * 32 + l];
            const int q = (sub & 1) ? (qb >> 4) : (qb & 0xF);
            return d * (float)s * (float)q - dmin * (float)m;
        }
        case T_Q6_K: {
            const uint8_t* b = row + (size_t)(c >> 8) * 210;
            const int e = c & 255, h = e >> 7, r = e & 127;
            const int s = r >> 6, i = r & 63;            // ql nibble s of byte h*64+i
            const int t = r >> 5, j = r & 31;            // qh bits 2t of byte h*32+j
            const int qlv = (b[h * 64 + i] >> (4 * s)) & 0xF;
            const int qhv = (b[128 + h * 32 + j] >> (2 * t)) & 3;
            const int q = (qlv | (qhv << 4)) - 32;
            const float d = half_bits_to_float(*reinterpret_cast<const uint16_t*>(b + 208));
            return d * (float)(int8_t)b[192 + (e >> 4)] * (float)q;
        }
        default: return 0.f;
    }
}

__global__ void __launch_bounds__(256) embed_kernel(const __grid_constant__ EmbedParams p) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ int tok_s;
    if (threadIdx.x == 0) {
        const int pos = __ldcg(&p.st->pos);
        const int np = __ldcg(&p.st->n_prompt);
        int tok = __ldcg(&p.st->token);
        // prompt positions step through here only before the first draw: after a context shift a generated token may sit at a
        // position below n_prompt
        if (pos < np && __ldcg(&p.st->out_idx) == 0) tok = __ldcg(p.prompt_ids + pos);
        if (blockIdx.x == 0) p.st->token = tok;       // same value every CTA derives: no ordering needed
        tok_s = tok;
    }
    __syncthreads();
    // one column per thread: the row's bytes arrive in a single round trip
    const uint8_t* row = p.w + (size_t)tok_s * p.row_bytes;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < p.cols; c += gridDim.x * blockDim.x) p.x[c] = dequant_native(row, p.type, c);
}

// Greedy sampling over SAMPLE_CTAS CTAs: each scans a slice of the logits once (online max / argmax / sum of exp, all
// loads of a thread in flight together), the last CTA to finish (atomic ticket) merges the per-CTA triples and
// advances the step state.  Ties go to the lowest index.
constexpr int SAMPLE_THREADS = 256;
constexpr int SAMPLE_ILP = 8;

struct Cand { float m; int i; float s; };     // running max, its index, sum of exp(x - m)
__device__ __forceinline__ Cand cand_merge(const Cand& a, const Cand& b) {
    Cand r;
    const bool ta = a.m > b.m || (a.m == b.m && a.i <= b.i);
    r.m = ta ? a.m : b.m;
    r.i = ta ? a.i : b.i;
    const float ea = (a.m == -INFINITY) ? 0.f : expf(a.m - r.m), eb = (b.m == -INFINITY) ? 0.f : expf(b.m - r.m);
    r.s = a.s * ea + b.s * eb;
    return r;
}
__device__ __forceinline__ Cand cand_warp(Cand c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Cand t;
        t.m = __shfl_xor_sync(0xffffffffu, c.m, o);
        t.i = __shfl_xor_sync(0xffffffffu, c.i, o);
        t.s = __shfl_xor_sync(0xffffffffu, c.s, o);
        c = cand_merge(c, t);
    }
    return c;
}

__global__ void __launch_bounds__(SAMPLE_THREADS) sample_greedy_kernel(const __grid_constant__ SampleParams p) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ Cand sc[SAMPLE_THREADS / 32];
    __shared__ int is_last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    StepState* st = p.st;
    const int done = __ldcg(&st->done);
    const int out_idx = __ldcg(&st->out_idx);
    const bool keep = p.logits_keep != nullptr && !done && out_idx < p.max_out;
    float* dst = keep ? p.logits_keep + (size_t)out_idx * p.n_vocab : nullptr;
    Cand c{-INFINITY, 0x7fffffff, 0.f};
    const int stride = SAMPLE_CTAS * SAMPLE_THREADS;
    for (int i0 = blockIdx.x * SAMPLE_THREADS + tid; i0 < p.n_vocab; i0 += stride * SAMPLE_ILP) {
        float v[SAMPLE_ILP];
#pragma unroll
        for (int k = 0; k < SAMPLE_ILP; ++k) {
            const int i = i0 + k * stride;
            v[k] = i < p.n_vocab ? __ldcg(p.logits + i) : -INFINITY;
        }
        float m = c.m;
#pragma unroll
        for (int k = 0; k < SAMPLE_ILP; ++k)
            if (v[k] > m) { m = v[k]; c.i = i0 + k * stride; }       // ascending indices: strict > keeps the lowest on ties
        float sum = (c.m == -INFINITY) ? 0.f : c.s * expf(c.m - m);
#pragma unroll
        for (int k = 0; k < SAMPLE_ILP; ++k) {
            if (v[k] != -INFINITY) sum += expf(v[k] - m);
            if (keep && i0 + k * stride < p.n_vocab) dst[i0 + k * stride] = v[k];
        }
        c.m = m;
        c.s = sum;
    }
    c = cand_warp(c);
    if (lane == 0) sc[warp] = c;
    __syncthreads();
    float* pm = p.scratch;
    int* pi = reinterpret_cast<int*>(p.scratch + SAMPLE_CTAS);
    float* ps = p.scratch + 2 * SAMPLE_CTAS;
    unsigned* ticket_ctr = reinterpret_cast<unsigned*>(p.scratch + 3 * SAMPLE_CTAS);
    if (tid == 0) {
        Cand t = sc[0];
        for (int w = 1; w < SAMPLE_THREADS / 32; ++w) t = cand_merge(t, sc[w]);
        pm[blockIdx.x] = t.m; pi[blockIdx.x] = t.i; ps[blockIdx.x] = t.s;
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(ticket_ctr) : "memory");
        is_last = (ticket == SAMPLE_CTAS - 1);
        if (is_last) *ticket_ctr = 0;
    }
    __syncthreads();
    if (!is_last || warp != 0) return;
    Cand t{-INFINITY, 0x7fffffff, 0.f};
    for (int k = lane; k < SAMPLE_CTAS; k += 32) {
        Cand u{__ldcg(pm + k), __ldcg(pi + k), __ldcg(ps + k)};
        t = cand_merge(t, u);
    }
    t = cand_warp(t);
    if (lane == 0 && !done) {
        if (out_idx < p.max_out) {
            p.out_ids[out_idx] = t.i;
            p.out_logprobs[out_idx] = -logf(t.s);
        }
        st->token = t.i;
        st->pos = st->pos + 1;
        st->out_idx = out_idx + 1;
        if (!st->ignore_eos) {
            for (int k = 0; k < st->n_stop; ++k)
                if (st->stop_ids[k] == t.i) st->done = 1;
        }
    }
}

__global__ void advance_kernel(StepState* st) {
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) st->pos = st->pos + 1;
}

__global__ void __launch_bounds__(256) rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, int n, float eps,
                                                      float* __restrict__ y) {
    __shared__ float red[8];
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) { const float v = x[i]; ss += v * v; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += red[k];
    const float rstd = 1.0f / sqrtf(tot / (float)n + eps);
    for (int i = threadIdx.x; i < n; i += 256) y[i] = (x[i] * rstd) * w[i];
}

__global__ void rope_kv_kernel(float* q, const float* k, const float* v, int n_head, int n_kv, int hd, const float* cos_t,
                               const float* sin_t, const StepState* st, __half* k_cache, __half* v_cache, const int* page_table) {
    const int pos = st->pos;
    const int page = page_table[pos / KV_PAGE_TOKENS];
    const int tok = pos % KV_PAGE_TOKENS;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;        // pair index
    const int nq = n_head * hd / 2, nk = n_kv * hd / 2;
    if (i < nq) {
        const int d = (2 * i) % hd;
        const float c = cos_t[(size_t)pos * (hd / 2) + d / 2], s = sin_t[(size_t)pos * (hd / 2) + d / 2];
        const float a = q[2 * i], b = q[2 * i + 1];
        q[2 * i] = a * c - b * s;
        q[2 * i + 1] = a * s + b * c;
    } else if (i < nq + nk) {
        const int j = i - nq;
        const int r = 2 * j, kvh = r / hd, d = r % hd;
        const float c = cos_t[(size_t)pos * (hd / 2) + d / 2], s = sin_t[(size_t)pos * (hd / 2) + d / 2];
        const float a = k[r], b = k[r + 1];
        const size_t off = (((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d;
        k_cache[off] = __float2half_rn(a * c - b * s);
        k_cache[off + 1] = __float2half_rn(a * s + b * c);
        v_cache[off] = __float2half_rn(v[r]);
        v_cache[off + 1] = __float2half_rn(v[r + 1]);
    }
}

__global__ void silu_mul_kernel(const float* g, const float* u, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const float a = g[i]; out[i] = (a / (1.0f + expf(-a))) * u[i]; }
}
__global__ void add_kernel(const float* a, const float* b, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] + b[i];
}
__global__ void l2_flush_kernel(float* buf, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) buf[i] = buf[i] * 0.5f + 1.0f;
}

// ---- embedding pooling (generateEmbedding: prefill -> output_norm -> mean over positions -> L2 normalise) -----------
// h [rows x n] fp32 hidden states of one sequence.  Three tiny launches, fixed summation orders (deterministic):
//   rstd[t] = 1/sqrt(mean(h_t^2) + eps);  pooled[d] = w[d]/rows * sum_t h[t][d] * rstd[t];  out = pooled / |pooled|
__global__ void __launch_bounds__(256) pool_rstd_kernel(const float* __restrict__ h, int rows, int n, float eps, float* __restrict__ rstd) {
    const int t = blockIdx.x;
    __shared__ float red[8];
    const float* hr = h + (size_t)t * n;
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) { const float v = hr[i]; ss += v * v; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int k = 0; k < 8; ++k) tot += red[k];
        rstd[t] = 1.0f / sqrtf(tot / (float)n + eps);
    }
}
__global__ void __launch_bounds__(256) pool_cols_kernel(const float* __restrict__ h, const float* __restrict__ rstd, const float* __restrict__ w,
                                                        int rows, int n, float* __restrict__ pooled) {
    const int d = blockIdx.x * 256 + threadIdx.x;
    if (d >= n) return;
    float acc = 0.f;
    for (int t = 0; t < rows; ++t) acc += h[(size_t)t * n + d] * rstd[t];
    pooled[d] = acc * w[d] / (float)rows;
}
__global__ void __launch_bounds__(256) pool_sum_kernel(const float* __restrict__ h, const float* __restrict__ rstd, int rows, int n,
                                                       int accumulate, float* __restrict__ sum) {
    const int d = blockIdx.x * 256 + threadIdx.x;
    if (d >= n) return;
    float acc = 0.f;
    for (int t = 0; t < rows; ++t) acc += h[(size_t)t * n + d] * rstd[t];
    sum[d] = accumulate ? sum[d] + acc : acc;
}
__global__ void __launch_bounds__(256) pool_scale_kernel(float* __restrict__ sum, const float* __restrict__ w, int rows, int n) {
    const int d = blockIdx.x * 256 + threadIdx.x;
    if (d < n) sum[d] = sum[d] * w[d] / (float)rows;
}
__global__ void __launch_bounds__(1024) pool_normalize_kernel(const float* __restrict__ pooled, int n, float* __restrict__ out) {
    __shared__ float red[32];
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 1024) ss += pooled[i] * pooled[i];
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 32; ++k) tot += red[k];
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
    for (int i = threadIdx.x; i < n; i += 1024) out[i] = pooled[i] * inv;
}

template <typename... Args>
cudaError_t launch_pdl(void (*kern)(Args...), dim3 grid, dim3 block, bool pdl, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

}  // namespace

cudaError_t embed_launch(const EmbedParams& p, bool pdl, cudaStream_t s) {
    return launch_pdl(embed_kernel, dim3((unsigned)((p.cols + 255) / 256)), dim3(256), pdl, s, p);
}
cudaError_t sample_greedy_launch(const SampleParams& p, bool pdl, cudaStream_t s) {
    return launch_pdl(sample_greedy_kernel, dim3(SAMPLE_CTAS), dim3(SAMPLE_THREADS), pdl, s, p);
}
cudaError_t advance_launch(StepState* st, bool pdl, cudaStream_t s) {
    return launch_pdl(advance_kernel, dim3(1), dim3(32), pdl, s, st);
}
cudaError_t rmsnorm_launch(const float* x, const float* w, int n, float eps, float* y, cudaStream_t s) {
    rmsnorm_kernel<<<1, 256, 0, s>>>(x, w, n, eps, y);
    return cudaGetLastError();
}
cudaError_t rope_kv_launch(float* q, const float* k, const float* v, int n_head, int n_kv, int head_dim, const float* cos_t,
                           const float* sin_t, const StepState* st, __half* k_cache, __half* v_cache, const int* page_table,
                           cudaStream_t s) {
    const int n = (n_head + n_kv) * head_dim / 2;
    rope_kv_kernel<<<(n + 255) / 256, 256, 0, s>>>(q, k, v, n_head, n_kv, head_dim, cos_t, sin_t, st, k_cache, v_cache, page_table);
    return cudaGetLastError();
}
cudaError_t silu_mul_launch(const float* g, const float* u, int n, float* out, cudaStream_t s) {
    silu_mul_kernel<<<(n + 255) / 256, 256, 0, s>>>(g, u, n, out);
    return cudaGetLastError();
}
cudaError_t add_launch(const float* a, const float* b, int n, float* out, cudaStream_t s) {
    add_kernel<<<(n + 255) / 256, 256, 0, s>>>(a, b, n, out);
    return cudaGetLastError();
}
cudaError_t pool_embedding_launch(const float* h, int rows, int n, const float* norm_w, float eps, float* rstd_scratch, float* pooled_scratch,
                                  float* out, cudaStream_t s) {
    pool_rstd_kernel<<<rows, 256, 0, s>>>(h, rows, n, eps, rstd_scratch);
    pool_cols_kernel<<<(n + 255) / 256, 256, 0, s>>>(h, rstd_scratch, norm_w, rows, n, pooled_scratch);
    pool_normalize_kernel<<<1, 1024, 0, s>>>(pooled_scratch, n, out);
    return cudaGetLastError();
}
cudaError_t pool_embedding_sum_launch(const float* h, int rows, int n, float eps, float* rstd_scratch, float* sum, bool accumulate, cudaStream_t s) {
    pool_rstd_kernel<<<rows, 256, 0, s>>>(h, rows, n, eps, rstd_scratch);
    pool_sum_kernel<<<(n + 255) / 256, 256, 0, s>>>(h, rstd_scratch, rows, n, accumulate ? 1 : 0, sum);
    return cudaGetLastError();
}
cudaError_t pool_embedding_finish_launch(float* sum, int total_rows, int n, const float* norm_w, float* out, cudaStream_t s) {
    pool_scale_kernel<<<(n + 255) / 256, 256, 0, s>>>(sum, norm_w, total_rows, n);
    pool_normalize_kernel<<<1, 1024, 0, s>>>(sum, n, out);
    return cudaGetLastError();
}

cudaError_t l2_flush_launch(float* buf, size_t n, cudaStream_t s) {
    l2_flush_kernel<<<132 * 4, 256, 0, s>>>(buf, n);
    return cudaGetLastError();
}

}  // namespace gl
