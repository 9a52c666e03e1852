// Batched-prefill linear layers on the Hopper tensor cores: C[M x N] = A[M x K] * B[N x K]^T, 16-bit inputs, fp32 accumulation
// in registers (wgmma).  This is the one place on the hot path where the work is a true dense contraction: the prompt's
// [T x n_embd] activations against each resident 16-bit weight matrix.
// Reference call site: the prompt-evaluation phase inside Ollama behind OllamaService.generate*Response / generateEmbedding
// (client/src/services/OllamaService.ts:142-145, 235-237, 633-636 of the reference project).
//
// Shape of the kernel (persistent: one CTA per SM walks 128 x 128 output tiles, three warpgroups, hand-written PTX):
//   warpgroup 0, one lane : TMA producer -- cp.async.bulk.tensor.2d of a 128 x 64 A box and a 128 x 64 B box per K-step into a
//                           4-stage mbarrier ring (128-byte swizzle, 32 KB per stage); the ring runs on across tile boundaries;
//   warpgroups 1, 2       : consumers -- warpgroup c owns rows 64c..64c+63 of the tile: per stage four wgmma.m64n128k16
//                           (operands addressed by shared-memory matrix descriptors, accumulator in 64 registers per thread),
//                           the stage goes back to the producer once the MMAs that read it have completed; after the last
//                           K-step the accumulator is staged through shared memory so that each thread owns 32 consecutive
//                           columns of one row, and the fused epilogue (fp32 store, residual add, 16-bit store, SiLU*mul,
//                           RoPE / split) writes global memory.
// SASS to look for: HGMMA (wgmma), UTMALDG (TMA).
#include <cuda.h>
#include <algorithm>
#include <cstdlib>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "kernels.h"
#include "prefill.h"
#include "wgmma.cuh"

namespace gl {

namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int WG_K = 16;
constexpr int TILE_A_BYTES = BM * BK * 2, TILE_B_BYTES = BN * BK * 2;
constexpr int STAGE_BYTES = TILE_A_BYTES + TILE_B_BYTES;
constexpr int STAGES = 4;
constexpr int TC_THREADS = 384;
constexpr int STG_LD = BN + 4;                 // staging row stride in floats: float4 reads of 8 consecutive rows hit 8 distinct bank quads
constexpr size_t STG_BYTES = (size_t)BM * STG_LD * 4;
constexpr size_t TC_SMEM = (size_t)STAGES * STAGE_BYTES + STG_BYTES + 1024 /* alignment slack */ + 256 /* barriers */;

struct Tc5Params {
    CUtensorMap ta;      // A: dims {K, M_alloc}, box {64, 128}, 128-B swizzle
    CUtensorMap tb;      // B: dims {K, N},       box {64, 128}, 128-B swizzle
    void* c;
    int m, n, k, ldc;
    int epi;
    int bf16;
    RopeSplitArgs rope;  // GEMM_EPI_ROPE_SPLIT only
};

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}

template <typename T> __device__ __forceinline__ T cvt16(float v);
template <> __device__ __forceinline__ __half cvt16<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt16<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// 32 consecutive accumulator columns of one output row -> global memory
template <typename T>
__device__ __forceinline__ void epilogue_row(const Tc5Params& p, int row, int col0, const uint32_t* v) {
    if (p.epi == GEMM_EPI_SILU) {
        // B rows are interleaved [8 gate | 8 up] at load time: columns 16g..16g+7 gate, 16g+8..16g+15 up -> hidden column 8g+j
        T* out = reinterpret_cast<T*>(p.c) + (size_t)row * p.ldc + (col0 >> 4) * 8;
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            if (col0 + 16 * g >= p.n) break;
            T o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float gt = __uint_as_float(v[16 * g + j]), up = __uint_as_float(v[16 * g + 8 + j]);
                o[j] = cvt16<T>((gt / (1.0f + expf(-gt))) * up);
            }
            *reinterpret_cast<uint4*>(out + 8 * g) = *reinterpret_cast<const uint4*>(o);
        }
        return;
    }
    const bool full = col0 + 32 <= p.n;
    if (p.epi == GEMM_EPI_T16) {
        T* out = reinterpret_cast<T*>(p.c) + (size_t)row * p.ldc + col0;
        if (full && (p.ldc & 7) == 0) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                T o[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = cvt16<T>(__uint_as_float(v[8 * q + j]));
                *reinterpret_cast<uint4*>(out + 8 * q) = *reinterpret_cast<const uint4*>(o);
            }
        } else {
            for (int j = 0; j < 32 && col0 + j < p.n; ++j) out[j] = cvt16<T>(__uint_as_float(v[j]));
        }
        return;
    }
    float* out = reinterpret_cast<float*>(p.c) + (size_t)row * p.ldc + col0;
    if (full && (p.ldc & 3) == 0) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float4 o = make_float4(__uint_as_float(v[4 * q]), __uint_as_float(v[4 * q + 1]), __uint_as_float(v[4 * q + 2]), __uint_as_float(v[4 * q + 3]));
            float4* dst = reinterpret_cast<float4*>(out) + q;
            if (p.epi == GEMM_EPI_ADD_F32) {
                const float4 r = *dst;
                o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
            }
            *dst = o;
        }
    } else {
        for (int j = 0; j < 32 && col0 + j < p.n; ++j) {
            const float a = __uint_as_float(v[j]);
            out[j] = p.epi == GEMM_EPI_ADD_F32 ? out[j] + a : a;
        }
    }
}

// GEMM_EPI_ROPE_SPLIT: 32 consecutive columns of one row of the QKV projection, straight from the accumulator -- what the
// stand-alone RoPE / split kernel did after a round trip of the fp32 QKV matrix through HBM (50 MB written + 50 MB read per
// layer at 2 048 rows).  pos < 0: a padding row (zeros: finite operands for the padded attention tiles).  The q / k / v
// regions and the heads are multiples of 32 columns wide, so a chunk never straddles two of them.
__device__ __forceinline__ void epilogue_rope_split(const RopeSplitArgs& a, int row, int pos, const int* page_table, int col0, const uint32_t* v) {
    const int qd = a.n_head * a.hd, kvd = a.n_kv * a.hd;
    const bool cache = pos >= 0 && a.k_cache != nullptr && page_table != nullptr;
    size_t cache_off = 0;
    if (cache) {
        const int kvcol = col0 < qd + kvd ? col0 - qd : col0 - qd - kvd;      // (only used for the k / v regions)
        cache_off = (((size_t)__ldg(page_table + pos / KV_PAGE_TOKENS) * a.n_kv + (kvcol >= 0 ? kvcol / a.hd : 0)) * KV_PAGE_TOKENS + pos % KV_PAGE_TOKENS) * a.hd +
                    (kvcol >= 0 ? kvcol % a.hd : 0);
    }
    if (col0 < qd + kvd) {
        __align__(16) __half2 o[16];
        if (pos >= 0) {
            const int d0 = col0 % a.hd;
            const float4* c4 = reinterpret_cast<const float4*>(a.cos_t + (size_t)pos * (a.hd / 2) + d0 / 2);
            const float4* s4 = reinterpret_cast<const float4*>(a.sin_t + (size_t)pos * (a.hd / 2) + d0 / 2);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 c = __ldg(c4 + i), s = __ldg(s4 + i);
                const float cc[4] = {c.x, c.y, c.z, c.w}, ss[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float x0 = __uint_as_float(v[8 * i + 2 * e]), x1 = __uint_as_float(v[8 * i + 2 * e + 1]);
                    o[4 * i + e] = __floats2half2_rn(x0 * cc[e] - x1 * ss[e], x0 * ss[e] + x1 * cc[e]);
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) o[i] = __floats2half2_rn(0.f, 0.f);
        }
        __half* dst = col0 < qd ? a.q + (size_t)row * qd + col0 : a.k + (size_t)row * kvd + (col0 - qd);
#pragma unroll
        for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(o)[i];
        if (cache && col0 >= qd) {
#pragma unroll
            for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(a.k_cache + cache_off)[i] = reinterpret_cast<const uint4*>(o)[i];
        }
    } else {
        // V: the warp's 32 lanes are 32 consecutive rows = 64 contiguous bytes of one V^T row per store instruction
        const int c0 = col0 - qd - kvd;
        __align__(16) __half hv[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            hv[j] = __float2half_rn(pos >= 0 ? __uint_as_float(v[j]) : 0.f);
            a.vt[(size_t)(c0 + j) * a.vt_ld + row] = hv[j];
        }
        if (cache) {
#pragma unroll
            for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(a.v_cache + cache_off)[i] = reinterpret_cast<const uint4*>(hv)[i];
        }
    }
}

template <bool BF16>
__global__ void __launch_bounds__(TC_THREADS, 1) gemm_tc5_kernel(const __grid_constant__ Tc5Params p) {
    extern __shared__ uint8_t smem_raw[];
    // 128-byte-swizzled tiles must sit on 1024-byte boundaries
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float* stg = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE_BYTES);     // [BM][STG_LD] accumulator staging
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)STAGES * STAGE_BYTES + STG_BYTES);
    uint64_t* empty = full + STAGES;

    const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
    const int warp = t >> 5, lane = t & 31;
    // M tiles are the fast grid dimension: the (few) CTAs that share a weight tile run back to back and find it in L2
    const int tiles_m = (p.m + BM - 1) / BM, tiles_n = (p.n + BN - 1) / BN, n_tiles = tiles_m * tiles_n;
    const int nk = (p.k + BK - 1) / BK;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.ta) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tb) : "memory");
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 2);        // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        if (t == 0) {
            // ===== TMA producer =====
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int m0 = (tile % tiles_m) * BM, n0 = (tile / tiles_m) * BN;
                for (int kb = 0; kb < nk; ++kb) {
                    mbar_wait(&empty[st], ph ^ 1u);
                    uint8_t* sa = smem + (size_t)st * STAGE_BYTES;
                    mbar_expect_tx(&full[st], STAGE_BYTES);
                    tma_load_2d(sa, &p.ta, kb * BK, m0, &full[st]);
                    tma_load_2d(sa + TILE_A_BYTES, &p.tb, kb * BK, n0, &full[st]);
                    if (++st == STAGES) { st = 0; ph ^= 1u; }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup c = wg - 1 computes rows 64c..64c+63 of each tile =====
    const int c = wg - 1;
    const uint32_t smem0 = smem_u32(smem);
    float* my_stg = stg + (size_t)(64 * c) * STG_LD;
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = (tile % tiles_m) * BM, n0 = (tile / tiles_m) * BN;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nk; ++kb) {
            mbar_wait(&full[st], ph);
            const uint32_t sa = smem0 + (uint32_t)(st * STAGE_BYTES);
            const uint64_t adesc = wgmma_desc_sw128(sa + (uint32_t)(c * 64 * BK * 2)), bdesc = wgmma_desc_sw128(sa + TILE_A_BYTES);
            wgmma_fence_acc<BN / 2>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / WG_K; ++k) wgmma_m64k16<BN, BF16>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), 1u);
            wgmma_commit();
            // the MMAs of the previous stage have completed once at most this stage's group is outstanding: release that stage
            wgmma_wait<1>();
            wgmma_fence_acc<BN / 2>(acc);
            if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
            prev = st;
            if (++st == STAGES) { st = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc<BN / 2>(acc);
        if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);

        // accumulator fragment -> staging rows (the previous tile's readers of this warpgroup are done: barrier first)
        named_bar_sync(1 + c, 128);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            const int r = 16 * warp + (lane >> 2), col = 8 * i + 2 * (lane & 3);
            *reinterpret_cast<float2*>(my_stg + (size_t)r * STG_LD + col) = make_float2(acc[4 * i], acc[4 * i + 1]);
            *reinterpret_cast<float2*>(my_stg + (size_t)(r + 8) * STG_LD + col) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
        }
        named_bar_sync(1 + c, 128);

        // epilogue: thread = one row (the 32 lanes of a warp are 32 consecutive rows), 32 consecutive columns per chunk
        const int lr = (warp & 1) * 32 + lane, row = m0 + 64 * c + lr;
        int pos = -1;                               // GEMM_EPI_ROPE_SPLIT: the row's absolute position in its sequence (-1: padding)
        const int* page_table = nullptr;
        if (p.epi == GEMM_EPI_ROPE_SPLIT) {
            for (int i = 0; i < p.rope.segs.n; ++i) {
                const int s0 = p.rope.segs.start[i], ln = p.rope.segs.len[i];
                if (row >= s0 && row < s0 + (ln + 127) / 128 * 128) {
                    pos = row - s0 < ln ? p.rope.segs.pos0[i] + row - s0 : -1;
                    page_table = p.rope.segs.table[i];
                }
            }
        }
#pragma unroll 1
        for (int j = 0; j < 2; ++j) {
            const int ch = (warp >> 1) * 2 + j;
            uint32_t v[32];
            const float4* src = reinterpret_cast<const float4*>(my_stg + (size_t)lr * STG_LD + ch * 32);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 f = src[q];
                v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y); v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
            }
            const int col0 = n0 + ch * 32;
            if (row < p.m && col0 < p.n) {
                if (p.epi == GEMM_EPI_ROPE_SPLIT) epilogue_rope_split(p.rope, row, pos, page_table, col0, v);
                else if (BF16) epilogue_row<__nv_bfloat16>(p, row, col0, v);
                else epilogue_row<__half>(p, row, col0, v);
            }
        }
    }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point lookup (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

// rows x k 16-bit elements, row stride ld elements; box = 128 rows x 64 elements, 128-byte swizzle
bool make_map(CUtensorMap* map, const void* base, int rows, int k, int ld, bool bf16) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


}  // namespace

cudaError_t gemm_tc5_configure() {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc5_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tc5_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    return e;
}

bool gemm_tc5_supported(const GemmParams& p) {
    // plain (un-batched, non-causal) TN GEMMs whose rows TMA can address: 16-byte aligned bases and row strides.  The epilogue's
    // 16-byte stores need a 16-byte aligned C; SiLU stores them unconditionally, so its rows must stay aligned too (ldc % 8).
    if ((uintptr_t)p.c % 16) return false;
    if (p.epi == GEMM_EPI_SILU && (p.ldc % 8)) return false;
    if (p.epi == GEMM_EPI_ROPE_SPLIT) {
        const RopeSplitArgs* r = p.rope;
        if (!r || (r->hd % 32) || p.n != (r->n_head + 2 * r->n_kv) * r->hd || (p.m % 128) || (r->vt_ld & 7) || r->segs.n < 1 || r->segs.n > PF_MAX_SEGS) return false;
    }
    return p.batch == 1 && !p.causal_skip && !p.causal_k && (p.lda % 8) == 0 && (p.ldb % 8) == 0 && (p.k % 8) == 0 &&
           ((uintptr_t)p.a % 16) == 0 && ((uintptr_t)p.b % 16) == 0 && (p.epi != GEMM_EPI_SILU || (p.n % 16) == 0);
}

// a_rows_alloc: rows of A that exist in memory (>= m; the scratch is padded to whole tiles and zero-filled)
cudaError_t gemm_tc5_launch(const GemmParams& p, int a_rows_alloc, bool bf16, cudaStream_t s) {
    if (!gemm_tc5_supported(p)) return cudaErrorInvalidValue;
    Tc5Params tp{};
    if (!make_map(&tp.ta, p.a, a_rows_alloc, p.k, p.lda, bf16) || !make_map(&tp.tb, p.b, p.n, p.k, p.ldb, bf16)) return cudaErrorInvalidValue;
    tp.c = p.c; tp.m = p.m; tp.n = p.n; tp.k = p.k; tp.ldc = p.ldc; tp.epi = p.epi; tp.bf16 = bf16 ? 1 : 0;
    if (p.epi == GEMM_EPI_ROPE_SPLIT) tp.rope = *p.rope;
    // persistent grid: one CTA per SM walks the tiles, M tiles fastest (the CTAs that share a weight tile run together)
    static const int n_sm = []() { int dev = 0, n = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n > 0 ? n : 132; }();
    const int tiles = ((p.m + BM - 1) / BM) * ((p.n + BN - 1) / BN);
    const dim3 grid((unsigned)std::min(tiles, n_sm));
    if (bf16) gemm_tc5_kernel<true><<<grid, TC_THREADS, TC_SMEM, s>>>(tp);
    else gemm_tc5_kernel<false><<<grid, TC_THREADS, TC_SMEM, s>>>(tp);
    return cudaGetLastError();
}

}  // namespace gl
