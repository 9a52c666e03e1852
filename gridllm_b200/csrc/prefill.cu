// Batched prefill: the whole prompt goes through every layer as a [T x n_embd] activation matrix, so
// each weight matrix is read once per prompt instead of once per token, and the contraction runs on
// the tensor cores (north_star: "tensor cores only for the batched-prefill GEMM where it is a true
// dense contraction").  Reference call site: the prompt-evaluation phase inside Ollama behind
// OllamaService.generate*Response / generateEmbedding
// (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237, 633-636).
//
// The general GEMM: a TN GEMM  C[M x N] = A[M x K] * B[N x K]^T  on 16-bit inputs with fp32 accumulation
// (mma.sync m16n8k16; the plain linear layers run on the TMA + wgmma kernel of prefill_tc5.cu), cp.async
// 3-stage pipeline, XOR-swizzled shared memory, ldmatrix fragments, fused epilogues (residual add,
// SiLU*mul).  Weights are dequantised once at load into a resident 16-bit copy (HBM is 80 GB; 16 GB for
// Llama-3-8B).  Attention over the prompt is two batched GEMMs
// (Q K^T, P V) around a causal softmax.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "gguf_file.h"
#include "kernels.h"
#include "prefill.h"
#include "rowdot.h"

namespace gl {

namespace {

// ---------------------------------------------------------------------------------------------
// element access into ENGINE row layouts (rowdot.h) -- used once at load to build the 16-bit copy
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float dequant_engine(const uint8_t* mat, int type, int cols, int row_stride, int tile_rows, int r, int c) {
    const uint8_t* row = mat + (size_t)r * row_stride;      // fp types: plain row-major
    switch (type) {
        case T_F32: return reinterpret_cast<const float*>(row)[c];
        case T_F16: return __half2float(reinterpret_cast<const __half*>(row)[c]);
        case T_BF16: return __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(row)[c] << 16);
        case T_Q4_K:
        case T_Q6_K:
        case T_Q8_0: return dequant_engine_quant(mat, type, cols, tile_rows, r, c);
        default: return 0.f;
    }
}

template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(256) dequant_rows_kernel(const uint8_t* __restrict__ src, int type, int rows, int cols, int row_stride, int tile_rows,
                                                           T* __restrict__ dst, int dst_ld, int dst_row0, int interleave) {
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
        int dr = r;
        if (interleave == 1) dr = (r >> 3) * 16 + (r & 7);            // gate rows
        else if (interleave == 2) dr = (r >> 3) * 16 + 8 + (r & 7);   // up rows
        T* out = dst + (size_t)(dst_row0 + dr) * dst_ld;
        for (int c = threadIdx.x; c < cols; c += blockDim.x) out[c] = from_float<T>(dequant_engine(src, type, cols, row_stride, tile_rows, r, c));
    }
}

// ---------------------------------------------------------------------------------------------
// TN GEMM on mma.sync
// ---------------------------------------------------------------------------------------------
constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3, GEMM_THREADS = 256;
constexpr int STAGE_BYTES = (BM + BN) * BK * 2;   // 32 KB

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool pred) {
    const int sz = pred ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
template <typename T> __device__ __forceinline__ void mma16816(float* c, const uint32_t* a, const uint32_t* b);
template <> __device__ __forceinline__ void mma16816<__half>(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
template <> __device__ __forceinline__ void mma16816<__nv_bfloat16>(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// smem tile: rows of BK 16-bit elements = 128 B = 8 chunks of 16 B; chunk c of row r lives at chunk c ^ (r & 7)
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

template <typename T, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS) gemm_tn_kernel(const __grid_constant__ GemmParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bz = blockIdx.z;
    const T* A = reinterpret_cast<const T*>(p.a) + (size_t)bz * p.a_batch_stride;
    const T* B = reinterpret_cast<const T*>(p.b) + (size_t)(bz / p.b_batch_div) * p.b_batch_stride;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    if (p.causal_skip && n0 > m0 + BM - 1) return;          // S tile entirely above the diagonal
    const int k_end = p.causal_k ? min(p.k, m0 + BM) : p.k; // P V: keys beyond the last query of the tile are zero
    const int nk = (k_end + BK - 1) / BK;
    const uint32_t sbase = smem_u32(smem);

    auto load_stage = [&](int stage, int kt) {
        const int k0 = kt * BK;
        const uint32_t sa = sbase + stage * STAGE_BYTES, sb = sa + BM * BK * 2;
#pragma unroll
        for (int i = 0; i < (BM * 8) / GEMM_THREADS; ++i) {
            const int idx = tid + i * GEMM_THREADS, r = idx >> 3, c = idx & 7;
            const bool ok = (m0 + r) < p.m && (k0 + c * 8) < p.k;
            cp_async16(sa + swz(r, c), A + (size_t)(ok ? m0 + r : 0) * p.lda + (ok ? k0 + c * 8 : 0), ok);
        }
#pragma unroll
        for (int i = 0; i < (BN * 8) / GEMM_THREADS; ++i) {
            const int idx = tid + i * GEMM_THREADS, r = idx >> 3, c = idx & 7;
            const bool ok = (n0 + r) < p.n && (k0 + c * 8) < p.k;
            cp_async16(sb + swz(r, c), B + (size_t)(ok ? n0 + r : 0) * p.ldb + (ok ? k0 + c * 8 : 0), ok);
        }
    };

    const int wm = warp >> 2, wn = warp & 3;     // 2 x 4 warps, warp tile 64 x 32
    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nxt = kt + STAGES - 1;
            if (nxt < nk) load_stage(nxt % STAGES, nxt);
            cp_async_commit();
        }
        const int stage = kt % STAGES;
        const uint32_t sa = sbase + stage * STAGE_BYTES, sb = sa + BM * BK * 2;
#pragma unroll
        for (int ks = 0; ks < BK / 16; ++ks) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) {
                const int r = wm * 64 + mi * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
                const int c = ks * 2 + (lane >> 4);
                ldmatrix_x4(sa + swz(r, c), af[mi][0], af[mi][1], af[mi][2], af[mi][3]);
            }
#pragma unroll
            for (int nj = 0; nj < 2; ++nj) {
                const int r = wn * 32 + nj * 16 + (lane & 7) + 8 * (lane >> 4);
                const int c = ks * 2 + ((lane >> 3) & 1);
                uint32_t r0, r1, r2, r3;
                ldmatrix_x4(sb + swz(r, c), r0, r1, r2, r3);
                bf[nj * 2][0] = r0; bf[nj * 2][1] = r1; bf[nj * 2 + 1][0] = r2; bf[nj * 2 + 1][1] = r3;
            }
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) mma16816<T>(acc[mi][ni], af[mi], bf[ni]);
        }
    }
    cp_async_wait<0>();

    // ---- epilogue ---------------------------------------------------------------------------------
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int mi = 0; mi < 4; ++mi) {
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int m = m0 + wm * 64 + mi * 16 + g + 8 * hrow;
            if (m >= p.m) continue;
            if (EPI == GEMM_EPI_SILU) {
                // n8 tiles alternate gate / up (B rows interleaved in groups of 8 at load time)
#pragma unroll
                for (int pj = 0; pj < 2; ++pj) {
                    const int ncol = n0 + wn * 32 + pj * 16;            // gate tile start (global interleaved row)
                    const int hcol = (ncol >> 4) * 8 + 2 * t4;           // hidden column
                    if (ncol >= p.n) continue;
                    const float g0 = acc[mi][2 * pj][2 * hrow], g1 = acc[mi][2 * pj][2 * hrow + 1];
                    const float u0 = acc[mi][2 * pj + 1][2 * hrow], u1 = acc[mi][2 * pj + 1][2 * hrow + 1];
                    T* out = reinterpret_cast<T*>(p.c) + (size_t)bz * p.c_batch_stride + (size_t)m * p.ldc + hcol;
                    out[0] = from_float<T>((g0 / (1.0f + expf(-g0))) * u0);
                    out[1] = from_float<T>((g1 / (1.0f + expf(-g1))) * u1);
                }
            } else {
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int n = n0 + wn * 32 + ni * 8 + 2 * t4;
                    if (n >= p.n) continue;
                    const float v0 = acc[mi][ni][2 * hrow], v1 = acc[mi][ni][2 * hrow + 1];
                    if (EPI == GEMM_EPI_F32) {
                        float* out = reinterpret_cast<float*>(p.c) + (size_t)bz * p.c_batch_stride + (size_t)m * p.ldc + n;
                        out[0] = v0;
                        if (n + 1 < p.n) out[1] = v1;
                    } else if (EPI == GEMM_EPI_ADD_F32) {
                        float* out = reinterpret_cast<float*>(p.c) + (size_t)bz * p.c_batch_stride + (size_t)m * p.ldc + n;
                        out[0] += v0;
                        if (n + 1 < p.n) out[1] += v1;
                    } else {   // GEMM_EPI_T16
                        T* out = reinterpret_cast<T*>(p.c) + (size_t)bz * p.c_batch_stride + (size_t)m * p.ldc + n;
                        out[0] = from_float<T>(v0);
                        if (n + 1 < p.n) out[1] = from_float<T>(v1);
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// row-wise helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float dequant_native_row(const uint8_t* row, int type, int c);

template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_rows_kernel(const float* __restrict__ x, const float* __restrict__ w, int rows, int rows_pad, int n,
                                                           float eps, T* __restrict__ y) {
    const int r = blockIdx.x;
    T* yr = y + (size_t)r * n;
    if (r >= rows) {
        for (int i = threadIdx.x; i < n; i += 256) yr[i] = from_float<T>(0.f);
        return;
    }
    __shared__ float red[8];
    const float* xr = x + (size_t)r * n;
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) { const float v = xr[i]; ss += v * v; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += red[k];
    const float rstd = 1.0f / sqrtf(tot / (float)n + eps);
    for (int i = threadIdx.x; i < n; i += 256) yr[i] = from_float<T>((xr[i] * rstd) * w[i]);
}

// QKV fp32 [T x (qd + 2 kvd)] -> RoPE -> Q (16-bit) [T_pad x qd], K (16-bit) [T_pad x kvd], V^T [kvd][T_pad], + fp16 cache pages
template <typename T>
__global__ void __launch_bounds__(256) rope_split_kernel(const float* __restrict__ qkv, int t_rows, int t_pad, int pos0, int n_head, int n_kv, int hd,
                                                         const float* __restrict__ cos_t, const float* __restrict__ sin_t, T* __restrict__ qo,
                                                         T* __restrict__ ko, T* __restrict__ vt, __half* __restrict__ k_cache,
                                                         __half* __restrict__ v_cache, const int* __restrict__ page_table, int vt_ld) {
    const int t = blockIdx.x;
    const int qd = n_head * hd, kvd = n_kv * hd, ld = qd + 2 * kvd;
    if (t >= t_rows) {   // padding rows: zeros (finite inputs for the padded GEMM tiles)
        for (int i = threadIdx.x; i < qd; i += 256) qo[(size_t)t * qd + i] = from_float<T>(0.f);
        for (int i = threadIdx.x; i < kvd; i += 256) { ko[(size_t)t * kvd + i] = from_float<T>(0.f); vt[(size_t)i * vt_ld + t] = from_float<T>(0.f); }
        return;
    }
    const int pos = pos0 + t;
    const float* row = qkv + (size_t)t * ld;
    // k_cache == nullptr: embeddings -- the prompt pass is all there is, nothing is cached
    const bool cache = k_cache != nullptr;
    const int page = cache ? page_table[pos / KV_PAGE_TOKENS] : 0, tok = pos % KV_PAGE_TOKENS;
    for (int i = threadIdx.x; i < (qd + kvd) / 2; i += 256) {
        const int r = 2 * i;                       // even element index into [q | k]
        const int d = r % hd;
        const float c = cos_t[(size_t)pos * (hd / 2) + d / 2], s = sin_t[(size_t)pos * (hd / 2) + d / 2];
        const float a = row[r], b = row[r + 1];
        const float o0 = a * c - b * s, o1 = a * s + b * c;
        if (r < qd) {
            qo[(size_t)t * qd + r] = from_float<T>(o0);
            qo[(size_t)t * qd + r + 1] = from_float<T>(o1);
        } else {
            const int rk = r - qd, kvh = rk / hd;
            // K is cached in fp16; the attention GEMM must see exactly the cached value
            const __half h0 = __float2half_rn(o0), h1 = __float2half_rn(o1);
            ko[(size_t)t * kvd + rk] = from_float<T>(__half2float(h0));
            ko[(size_t)t * kvd + rk + 1] = from_float<T>(__half2float(h1));
            if (cache) {
                const size_t off = (((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d;
                k_cache[off] = h0;
                k_cache[off + 1] = h1;
            }
        }
    }
    for (int i = threadIdx.x; i < kvd; i += 256) {
        const __half hv = __float2half_rn(row[qd + kvd + i]);
        vt[(size_t)i * vt_ld + t] = from_float<T>(__half2float(hv));
        const int kvh = i / hd, d = i % hd;
        if (cache) v_cache[(((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d] = hv;
    }
}

// S fp32 [H][T_pad][T_pad] -> P (16-bit), causal, scaled
template <typename T>
__global__ void __launch_bounds__(256) softmax_causal_kernel(const float* __restrict__ s, int t_rows, int t_pad, float scale, T* __restrict__ p) {
    const int i = blockIdx.x, h = blockIdx.y;
    const float* sr = s + ((size_t)h * t_pad + i) * t_pad;
    T* pr = p + ((size_t)h * t_pad + i) * t_pad;
    if (i >= t_rows) {
        for (int j = threadIdx.x; j < t_pad; j += 256) pr[j] = from_float<T>(0.f);
        return;
    }
    __shared__ float red[8];
    float mx = -INFINITY;
    for (int j = threadIdx.x; j <= i; j += 256) mx = fmaxf(mx, sr[j] * scale);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
    __syncthreads();
    float sum = 0.f;
    for (int j = threadIdx.x; j <= i; j += 256) sum += expf(sr[j] * scale - mx);
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += red[k];
    const float inv = 1.0f / tot;
    for (int j = threadIdx.x; j < t_pad; j += 256) pr[j] = from_float<T>(j <= i ? expf(sr[j] * scale - mx) * inv : 0.f);
}

__device__ __forceinline__ float dequant_native_row(const uint8_t* row, int type, int c) {
    // native GGUF layouts (token_embd is kept native for row gathers)
    if (type == T_Q6_K) {
        const uint8_t* b = row + (size_t)(c >> 8) * 210;
        const int e = c & 255, h = e >> 7, r = e & 127;
        const int qlv = (b[h * 64 + (r & 63)] >> (4 * (r >> 6))) & 0xF;
        const int qhv = (b[128 + h * 32 + (r & 31)] >> (2 * (r >> 5))) & 3;
        const float d = half_bits_to_float(*reinterpret_cast<const uint16_t*>(b + 208));
        return d * (float)(int8_t)b[192 + (e >> 4)] * (float)((qlv | (qhv << 4)) - 32);
    }
    if (type == T_Q8_0) {
        const uint8_t* b = row + (size_t)(c >> 5) * 34;
        return half_bits_to_float(*reinterpret_cast<const uint16_t*>(b)) * (float)(int8_t)b[2 + (c & 31)];
    }
    if (type == T_Q4_K) return dequant_native_q4k(row, c);
    return dequant_engine(row, type, 0, 0, 1, 0, c);     // F32 / F16 / BF16: plain rows
}

__global__ void __launch_bounds__(256) embed_rows_kernel(const uint8_t* __restrict__ w, int type, int cols, int row_bytes, const int* __restrict__ ids,
                                                         int t_rows, float* __restrict__ x) {
    const int t = blockIdx.x;
    if (t >= t_rows) return;
    const uint8_t* row = w + (size_t)ids[t] * row_bytes;
    for (int c = threadIdx.x; c < cols; c += 256) x[(size_t)t * cols + c] = dequant_native_row(row, type, c);
}

template <typename T, int EPI>
cudaError_t gemm_launch_t(const GemmParams& p, cudaStream_t s) {
    dim3 grid((p.n + BN - 1) / BN, (p.m + BM - 1) / BM, p.batch);
    gemm_tn_kernel<T, EPI><<<grid, GEMM_THREADS, STAGES * STAGE_BYTES, s>>>(p);
    return cudaGetLastError();
}

template <typename T>
cudaError_t gemm_configure_t() {
    cudaError_t e = cudaFuncSetAttribute(gemm_tn_kernel<T, GEMM_EPI_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * STAGE_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tn_kernel<T, GEMM_EPI_ADD_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * STAGE_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tn_kernel<T, GEMM_EPI_T16>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * STAGE_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tn_kernel<T, GEMM_EPI_SILU>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * STAGE_BYTES);
    return e;
}

template <typename T>
cudaError_t gemm_launch_d(const GemmParams& p, cudaStream_t s) {
    switch (p.epi) {
        case GEMM_EPI_F32: return gemm_launch_t<T, GEMM_EPI_F32>(p, s);
        case GEMM_EPI_ADD_F32: return gemm_launch_t<T, GEMM_EPI_ADD_F32>(p, s);
        case GEMM_EPI_T16: return gemm_launch_t<T, GEMM_EPI_T16>(p, s);
        case GEMM_EPI_SILU: return gemm_launch_t<T, GEMM_EPI_SILU>(p, s);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace

cudaError_t prefill_configure() {
    cudaError_t e = gemm_configure_t<__half>();
    if (e == cudaSuccess) e = gemm_configure_t<__nv_bfloat16>();
    return e;
}

cudaError_t gemm_tn_launch(const GemmParams& p, bool bf16, cudaStream_t s) {
    if (p.k % 8 || p.lda % 8 || p.ldb % 8 || p.batch < 1 || p.b_batch_div < 1) return cudaErrorInvalidValue;
    return bf16 ? gemm_launch_d<__nv_bfloat16>(p, s) : gemm_launch_d<__half>(p, s);
}

cudaError_t dequant_rows_launch(const uint8_t* src, int type, int rows, int cols, int row_stride, int tile_rows, void* dst, int dst_ld, int dst_row0,
                                int interleave, bool bf16, cudaStream_t s) {
    const int blocks = rows < 132 * 8 ? rows : 132 * 8;
    if (bf16) dequant_rows_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>(src, type, rows, cols, row_stride, tile_rows, (__nv_bfloat16*)dst, dst_ld, dst_row0, interleave);
    else dequant_rows_kernel<__half><<<blocks, 256, 0, s>>>(src, type, rows, cols, row_stride, tile_rows, (__half*)dst, dst_ld, dst_row0, interleave);
    return cudaGetLastError();
}

cudaError_t rmsnorm_rows_launch(const float* x, const float* w, int rows, int rows_pad, int n, float eps, void* y, bool bf16, cudaStream_t s) {
    if (bf16) rmsnorm_rows_kernel<__nv_bfloat16><<<rows_pad, 256, 0, s>>>(x, w, rows, rows_pad, n, eps, (__nv_bfloat16*)y);
    else rmsnorm_rows_kernel<__half><<<rows_pad, 256, 0, s>>>(x, w, rows, rows_pad, n, eps, (__half*)y);
    return cudaGetLastError();
}

cudaError_t rope_split_launch(const float* qkv, int t_rows, int t_pad, int pos0, int n_head, int n_kv, int hd, const float* cos_t,
                              const float* sin_t, __half* qo, __half* ko, __half* vt, __half* k_cache, __half* v_cache,
                              const int* page_table, int vt_ld, cudaStream_t s) {
    rope_split_kernel<__half><<<t_pad, 256, 0, s>>>(qkv, t_rows, t_pad, pos0, n_head, n_kv, hd, cos_t, sin_t, qo, ko, vt, k_cache, v_cache, page_table, vt_ld);
    return cudaGetLastError();
}

cudaError_t softmax_causal_launch(const float* sc, int n_head, int t_rows, int t_pad, float scale, __half* p, cudaStream_t s) {
    softmax_causal_kernel<__half><<<dim3(t_pad, n_head), 256, 0, s>>>(sc, t_rows, t_pad, scale, p);
    return cudaGetLastError();
}

cudaError_t embed_rows_launch(const uint8_t* w, int type, int cols, int row_bytes, const int* ids, int t_rows, float* x, cudaStream_t s) {
    embed_rows_kernel<<<t_rows, 256, 0, s>>>(w, type, cols, row_bytes, ids, t_rows, x);
    return cudaGetLastError();
}

}  // namespace gl
