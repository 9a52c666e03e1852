// Prompt attention of the batched prefill as ONE fused kernel: S = Q K^T, causal mask, online softmax and O = P V per
// 128-row query tile, scores never leave the SM.  Replaces the three launches per sequence and layer of the first
// version (Q K^T GEMM -> fp32 scores in HBM -> causal softmax -> P in HBM -> P V GEMM: 1.2 GB of HBM traffic per layer
// at 2 048 tokens) on the path behind OllamaService.generate*Response / generateEmbedding
// (client/src/services/OllamaService.ts of the reference project:142-145, 235-237, 633-636: the prompt-evaluation phase).
//
// Shape of the work: per (query head, 128-row query tile, sequence) one CTA of four warps, 32 query rows per warp,
// KV tiles of 64 rows.  This version keeps the accumulators in registers (mma.sync m16n8k16, fp32 accumulate) and
// spends its effort on what the old path wasted: HBM traffic and launches.  It serves head dims 64 and 128.  K rows [kv][hd] and
// V^T rows [hd][kv] (what rope_split writes) are
// both "n-major with k contiguous", i.e. the B operand of a TN product: plain ldmatrix for both products, no
// transposes.  cp.async double buffering of the K / V^T tiles, XOR-swizzled shared memory, 96 KB per CTA at head dim
// 128: two CTAs per SM.  A pack of sequences (block-diagonal causal attention, section 4.7 of DESIGN.md) is one launch:
// blockIdx.z = sequence, every tile index is relative to the sequence's first row, so a sequence's result does not
// depend on what shares its pack.
#include <cuda_fp16.h>

#include "common.cuh"
#include "kernels.h"
#include "prefill.h"

namespace gl {

namespace {

constexpr int FA_BM = 128, FA_BN = 64, FA_WARPS = 4, FA_THREADS = FA_WARPS * 32;

struct FlashParams {
    const __half* q;     // [rows][qd]
    const __half* k;     // [rows][kvd]
    const __half* vt;    // [kvd][vt_ld]
    __half* out;         // [rows][qd]
    const __half* k_cache;   // PAGED: this layer's pages [page][n_kv][16][hd]
    const __half* v_cache;
    int qd, kvd, vt_ld, grp, n_kv;
    float scale_log2;    // 1/sqrt(hd) * log2(e)
    PrefillSegs segs;
};

__device__ __forceinline__ void fa_cp16(uint32_t dst, const void* src, bool pred) {
    const int sz = pred ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void fa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void fa_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fa_ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void fa_ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void fa_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float fa_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// tile of 64-column rows (128 B): 16-byte chunk c of row r lives at chunk c ^ (r & 7)
__device__ __forceinline__ uint32_t fa_swz(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

// PAGED = false: keys / values of the pass's own rows, from the scratch K rows and V^T columns (a segment that starts at
// position 0).  PAGED = true: query rows at absolute positions pos0 .. pos0 + len - 1 attend to keys 0 .. pos0 + len - 1, read
// from the layer's fp16 pages through the segment's page table (the QKV epilogue of this layer appended the segment's own rows
// one launch earlier).  KV tile kt is absolute positions [64 kt, 64 kt + 64) = four pages; one page of one KV head is a
// contiguous [16][HD] block.  V arrives row-major ([kv][hd]) and is staged like K; its P V operand is loaded with
// ldmatrix.trans, which hands every lane the same values in the same registers as the plain ldmatrix of V^T does, so both
// variants feed the MMAs identical operands and visit the same absolute KV tiles in the same order: a prompt prefilled in
// pieces gives the bits of one pass.
template <int HD, bool PAGED>
__global__ void __launch_bounds__(FA_THREADS, 2) flash_prefill_kernel(const __grid_constant__ FlashParams p) {
    // a [rows][HD] tile is HD / 64 sub-tiles of 64 columns (one 128-byte swizzle row each)
    constexpr int Q_BYTES = FA_BM * HD * 2;
    constexpr int K_BYTES = FA_BN * HD * 2;
    constexpr int V_BYTES = HD * FA_BN * 2;
    constexpr int STAGE_BYTES = K_BYTES + V_BYTES;
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int seq = blockIdx.z, h = blockIdx.x;
    const int len = p.segs.len[seq], r0 = p.segs.start[seq];
    const int pos0 = PAGED ? p.segs.pos0[seq] : 0;    // absolute position of the segment's first row
    const int n_qt = (len + FA_BM - 1) / FA_BM;
    if ((int)blockIdx.y >= n_qt) return;
    const int qt = n_qt - 1 - (int)blockIdx.y;        // the longest tiles of a sequence first
    const int m0 = qt * FA_BM;
    const int kvh = h / p.grp;
    const int kv_len = pos0 + len;                    // keys 0 .. kv_len - 1
    const int n_kt = PAGED ? min((kv_len + FA_BN - 1) / FA_BN, (pos0 + m0 + FA_BM - 1) / FA_BN + 1)
                           : min((len + FA_BN - 1) / FA_BN, (m0 + FA_BM) / FA_BN);
    const uint32_t sq = smem_u32(smem), sk0 = sq + Q_BYTES;

    const __half* qg = p.q + (size_t)(r0 + m0) * p.qd + (size_t)h * HD;
    const __half* kg = p.k + (size_t)r0 * p.kvd + (size_t)kvh * HD;
    const __half* vg = p.vt + (size_t)kvh * HD * p.vt_ld + r0;
    const int* table = PAGED ? p.segs.table[seq] : nullptr;
    const size_t page_elems = (size_t)p.n_kv * KV_PAGE_TOKENS * HD;
    const __half* kcg = PAGED ? p.k_cache + (size_t)kvh * KV_PAGE_TOKENS * HD : nullptr;
    const __half* vcg = PAGED ? p.v_cache + (size_t)kvh * KV_PAGE_TOKENS * HD : nullptr;

    auto load_kv = [&](int stage, int kt) {
        const int kv0 = kt * FA_BN;
        const uint32_t sk = sk0 + stage * STAGE_BYTES, sv = sk + K_BYTES;
        if constexpr (PAGED) {
            // K and V rows alike: [64 kv][HD] tiles; positions past the sequence are zero-filled (their scores are masked, but
            // P V multiplies P = 0 by V, and an unused page slot may hold anything) and their page entries are never read
#pragma unroll
            for (int i = 0; i < (FA_BN * HD / 8) / FA_THREADS; ++i) {
                const int idx = tid + i * FA_THREADS, r = idx / (HD / 8), c = idx % (HD / 8);
                const int pos = kv0 + r;
                const bool ok = pos < kv_len;
                const size_t off = ok ? (size_t)__ldg(table + pos / KV_PAGE_TOKENS) * page_elems + (size_t)(pos % KV_PAGE_TOKENS) * HD + c * 8 : 0;
                const uint32_t so = (c >> 3) * (FA_BN * 128) + fa_swz(r, c & 7);
                fa_cp16(sk + so, kcg + off, ok);
                fa_cp16(sv + so, vcg + off, ok);
            }
        } else {
#pragma unroll
            for (int i = 0; i < (FA_BN * HD / 8) / FA_THREADS; ++i) {
                const int idx = tid + i * FA_THREADS, r = idx / (HD / 8), c = idx % (HD / 8);
                const bool ok = kv0 + r < len;
                fa_cp16(sk + (c >> 3) * (FA_BN * 128) + fa_swz(r, c & 7), kg + (size_t)(ok ? kv0 + r : 0) * p.kvd + c * 8, ok);
            }
#pragma unroll
            for (int i = 0; i < (HD * FA_BN / 8) / FA_THREADS; ++i) {
                const int idx = tid + i * FA_THREADS, r = idx >> 3, c = idx & 7;      // r = head dim, c = chunk of 8 kv columns
                fa_cp16(sv + fa_swz(r, c), vg + (size_t)r * p.vt_ld + kv0 + c * 8, true);
            }
        }
    };

    // Q tile (rows beyond the sequence: zeros) + first K / V^T tile
#pragma unroll
    for (int i = 0; i < (FA_BM * HD / 8) / FA_THREADS; ++i) {
        const int idx = tid + i * FA_THREADS, r = idx / (HD / 8), c = idx % (HD / 8);
        const bool ok = m0 + r < len;
        fa_cp16(sq + (c >> 3) * (FA_BM * 128) + fa_swz(r, c & 7), qg + (size_t)(ok ? r : 0) * p.qd + c * 8, ok);
    }
    load_kv(0, 0);
    fa_commit();

    const int g = lane >> 2, t4 = lane & 3;
    const int wq0 = m0 + warp * 32;                   // first query row of this warp (relative to the segment)
    const int wrow0 = pos0 + wq0;                     // ... its absolute position (what the mask compares with kv columns)
    // lane-dependent part of the ldmatrix addresses (k-step 0).  A operand (Q): row = lane & 15, chunk bit = lane >> 4;
    // B operands (K, V^T): row = (lane & 7) + 8 (lane >> 4), chunk bit = (lane >> 3) & 1;
    // B operand of P V from V rows (PAGED, .trans): kv row = (lane & 7) + 8 ((lane >> 3) & 1), head-dim chunk bit = lane >> 4.
    const uint32_t qoff = fa_swz(warp * 32 + (lane & 15), lane >> 4);
    const uint32_t boff = fa_swz((lane & 7) + 8 * (lane >> 4), (lane >> 3) & 1);
    const uint32_t voff = fa_swz((lane & 7) + 8 * ((lane >> 3) & 1), lane >> 4);
    float o[2][HD / 8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < HD / 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
    float mrow[2][2], lrow[2][2];                      // running maximum (scaled, log2 domain) and partial row sums
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) { mrow[mt][0] = mrow[mt][1] = -INFINITY; lrow[mt][0] = lrow[mt][1] = 0.f; }

    for (int kt = 0; kt < n_kt; ++kt) {
        if (kt + 1 < n_kt) load_kv((kt + 1) & 1, kt + 1);
        fa_commit();
        fa_wait<1>();
        __syncthreads();
        const int kv0 = kt * FA_BN;
        if (kv0 <= wrow0 + 31) {                       // warp-uniform: tiles entirely above this warp's diagonal are skipped
            const uint32_t sk = sk0 + (kt & 1) * STAGE_BYTES, sv = sk + K_BYTES;
            float s[2][FA_BN / 8][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < FA_BN / 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) s[mt][nt][e] = 0.f;
            // ---- S = Q K^T ------------------------------------------------------------------------------
            // ldmatrix addresses: the k-step only flips bits 5-6 of a lane's swizzled offset (chunk = 2 (ks & 3) + lane bit)
#pragma unroll
            for (int ks = 0; ks < HD / 16; ++ks) {
                uint32_t a[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
                    fa_ldsm4(sq + (ks >> 2) * (FA_BM * 128) + mt * (16 * 128) + (qoff ^ ((ks & 3) << 5)), a[mt][0], a[mt][1], a[mt][2], a[mt][3]);
#pragma unroll
                for (int np = 0; np < FA_BN / 16; ++np) {
                    uint32_t b0, b1, b2, b3;
                    fa_ldsm4(sk + (ks >> 2) * (FA_BN * 128) + np * (16 * 128) + (boff ^ ((ks & 3) << 5)), b0, b1, b2, b3);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        fa_mma(s[mt][2 * np], a[mt], b0, b1);
                        fa_mma(s[mt][2 * np + 1], a[mt], b2, b3);
                    }
                }
            }
            // ---- causal mask (only where the tile crosses this warp's diagonal) ------------------------------
            if (kv0 + FA_BN - 1 > wrow0) {
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int nt = 0; nt < FA_BN / 8; ++nt)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int row = wrow0 + mt * 16 + g + 8 * (e >> 1);
                            const int col = kv0 + nt * 8 + 2 * t4 + (e & 1);
                            if (col > row) s[mt][nt][e] = -INFINITY;
                        }
            }
            // ---- online softmax ----------------------------------------------------------------------------
            // Column 0 of the first tile is never masked, so every row's maximum is finite from the first tile on.
            uint32_t pa[2][FA_BN / 16][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int nt = 0; nt < FA_BN / 8; ++nt) mx = fmaxf(mx, fmaxf(s[mt][nt][2 * hh], s[mt][nt][2 * hh + 1]));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    const float m_new = fmaxf(mrow[mt][hh], mx * p.scale_log2);
                    const float corr = fa_exp2(mrow[mt][hh] - m_new);      // first tile: exp2(-inf) = 0
                    mrow[mt][hh] = m_new;
                    float sum = 0.f;
#pragma unroll
                    for (int nt = 0; nt < FA_BN / 8; ++nt) {
                        const float p0 = fa_exp2(fmaf(s[mt][nt][2 * hh], p.scale_log2, -m_new));
                        const float p1 = fa_exp2(fmaf(s[mt][nt][2 * hh + 1], p.scale_log2, -m_new));
                        // the row sum is taken over the ROUNDED probabilities, the values the P V product uses
                        const __half2 ph = __floats2half2_rn(p0, p1);
                        const float2 pf = __half22float2(ph);
                        sum += pf.x + pf.y;
                        pa[mt][nt >> 1][(nt & 1) * 2 + hh] = *reinterpret_cast<const uint32_t*>(&ph);
                    }
                    lrow[mt][hh] = lrow[mt][hh] * corr + sum;
#pragma unroll
                    for (int nt = 0; nt < HD / 8; ++nt) {
                        o[mt][nt][2 * hh] *= corr;
                        o[mt][nt][2 * hh + 1] *= corr;
                    }
                }
            }
            // ---- O += P V  (B = V^T rows: head dim, kv contiguous; PAGED: V rows, transposed by ldmatrix) ----------
#pragma unroll
            for (int ks = 0; ks < FA_BN / 16; ++ks) {
#pragma unroll
                for (int np = 0; np < HD / 16; ++np) {
                    uint32_t b0, b1, b2, b3;
                    if constexpr (PAGED)
                        fa_ldsm4t(sv + (np >> 2) * (FA_BN * 128) + ks * (16 * 128) + (voff ^ ((np & 3) << 5)), b0, b1, b2, b3);
                    else
                        fa_ldsm4(sv + np * (16 * 128) + (boff ^ (ks << 5)), b0, b1, b2, b3);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        fa_mma(o[mt][2 * np], pa[mt][ks], b0, b1);
                        fa_mma(o[mt][2 * np + 1], pa[mt][ks], b2, b3);
                    }
                }
            }
        }
        __syncthreads();                               // stage (kt & 1) is refilled by the next iteration's prefetch
    }
    fa_wait<0>();

    // ---- normalise and store (rows beyond the sequence inside its last tile: zeros) ---------------------------
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float l = lrow[mt][hh];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const int row = wq0 + mt * 16 + g + 8 * hh;
            const float inv = (row < len && l > 0.f) ? 1.0f / l : 0.f;
            __half* orow = p.out + (size_t)(r0 + row) * p.qd + (size_t)h * HD + 2 * t4;
#pragma unroll
            for (int nt = 0; nt < HD / 8; ++nt)
                *reinterpret_cast<__half2*>(orow + nt * 8) = __floats2half2_rn(o[mt][nt][2 * hh] * inv, o[mt][nt][2 * hh + 1] * inv);
        }
    }
}

template <int HD> constexpr int fa_smem_bytes() { return FA_BM * HD * 2 + 2 * (FA_BN * HD * 2 + HD * FA_BN * 2); }

// QKV fp32 rows of a PACK -> RoPE -> Q, K (16-bit rows), V^T columns, + each sequence's own fp16 cache pages.
// One launch for the whole pack: block = EIGHT consecutive rows of the pack (sequences start on 128-row boundaries, so a block
// never straddles two of them); the rows between a sequence's end and its 128-row boundary are written as zeros (finite
// operands for the padded tiles).  Eight rows per block make the V^T store one 16-byte write per (head dim, block) instead of
// eight 2-byte writes a row stride apart (the per-row version moved 16 x the bytes it stored).
constexpr int RS_ROWS = 8;
__global__ void __launch_bounds__(256) rope_split_segs_kernel(const float* __restrict__ qkv, int n_head, int n_kv, int hd,
                                                              const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                              __half* __restrict__ qo, __half* __restrict__ ko, __half* __restrict__ vt,
                                                              __half* __restrict__ k_cache, __half* __restrict__ v_cache, int vt_ld,
                                                              const __grid_constant__ PrefillSegs segs) {
    const int t0 = blockIdx.x * RS_ROWS;
    const int qd = n_head * hd, kvd = n_kv * hd, ld = qd + 2 * kvd;
    int seq = -1;
    for (int i = 0; i < segs.n; ++i) {
        const int lp = (segs.len[i] + 127) / 128 * 128;
        if (t0 >= segs.start[i] && t0 < segs.start[i] + lp) seq = i;
    }
    const int rel0 = seq >= 0 ? t0 - segs.start[seq] : 0;
    const int n_valid = seq >= 0 ? max(0, min(RS_ROWS, segs.len[seq] - rel0)) : 0;      // rows rel0 .. rel0 + n_valid - 1 are tokens
    const int pos0 = seq >= 0 ? segs.pos0[seq] + rel0 : 0;                               // absolute position of the block's first row
    const int* page_table = seq >= 0 ? segs.table[seq] : nullptr;
    const bool cache = k_cache != nullptr && page_table != nullptr;
    for (int j = 0; j < RS_ROWS; ++j) {
        const int t = t0 + j, pos = pos0 + j;
        if (j >= n_valid) {
            for (int i = threadIdx.x; i < qd / 2; i += 256) *reinterpret_cast<__half2*>(qo + (size_t)t * qd + 2 * i) = __floats2half2_rn(0.f, 0.f);
            for (int i = threadIdx.x; i < kvd / 2; i += 256) *reinterpret_cast<__half2*>(ko + (size_t)t * kvd + 2 * i) = __floats2half2_rn(0.f, 0.f);
            continue;
        }
        const float* row = qkv + (size_t)t * ld;
        const int page = cache ? page_table[pos / KV_PAGE_TOKENS] : 0, tok = pos % KV_PAGE_TOKENS;
        for (int i = threadIdx.x; i < (qd + kvd) / 2; i += 256) {
            const int r = 2 * i;
            const int d = r % hd;
            const float c = cos_t[(size_t)pos * (hd / 2) + d / 2], s = sin_t[(size_t)pos * (hd / 2) + d / 2];
            const float2 ab = *reinterpret_cast<const float2*>(row + r);
            const float o0 = ab.x * c - ab.y * s, o1 = ab.x * s + ab.y * c;
            if (r < qd) {
                *reinterpret_cast<__half2*>(qo + (size_t)t * qd + r) = __floats2half2_rn(o0, o1);
            } else {
                const int rk = r - qd, kvh = rk / hd;
                const __half2 hk = __floats2half2_rn(o0, o1);
                *reinterpret_cast<__half2*>(ko + (size_t)t * kvd + rk) = hk;
                if (cache) *reinterpret_cast<__half2*>(k_cache + (((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d) = hk;
            }
        }
    }
    // V: thread = head-dim column, the block's eight tokens side by side in V^T
    for (int i = threadIdx.x; i < kvd; i += 256) {
        __align__(16) __half hv[RS_ROWS];
#pragma unroll
        for (int j = 0; j < RS_ROWS; ++j) hv[j] = __float2half_rn(j < n_valid ? qkv[(size_t)(t0 + j) * ld + qd + kvd + i] : 0.f);
        *reinterpret_cast<uint4*>(vt + (size_t)i * vt_ld + t0) = *reinterpret_cast<const uint4*>(hv);
        if (cache) {
            const int kvh = i / hd, d = i % hd;
            for (int j = 0; j < n_valid; ++j) {
                const int pos = pos0 + j;
                v_cache[(((size_t)page_table[pos / KV_PAGE_TOKENS] * n_kv + kvh) * KV_PAGE_TOKENS + pos % KV_PAGE_TOKENS) * hd + d] = hv[j];
            }
        }
    }
}

}  // namespace

cudaError_t flash_prefill_configure() {
    cudaError_t e = cudaFuncSetAttribute(flash_prefill_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, fa_smem_bytes<128>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(flash_prefill_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, fa_smem_bytes<64>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(flash_prefill_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, fa_smem_bytes<128>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(flash_prefill_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, fa_smem_bytes<64>());
    return e;
}

bool flash_prefill_supported(int hd) { return hd == 64 || hd == 128; }

cudaError_t flash_prefill_launch(const __half* q, const __half* k, const __half* vt, __half* out, const PrefillSegs& segs, int n_head, int n_kv,
                                 int hd, int vt_ld, float scale, const __half* k_cache, const __half* v_cache, cudaStream_t s) {
    if (segs.n < 1 || segs.n > PF_MAX_SEGS || !flash_prefill_supported(hd) || n_kv < 1 || n_head % n_kv || (vt_ld & 7)) return cudaErrorInvalidValue;
    int max_len = 0;
    bool paged = false;
    for (int i = 0; i < segs.n; ++i) {
        if (segs.len[i] < 1 || segs.pos0[i] < 0 || (segs.start[i] & 127)) return cudaErrorInvalidValue;     // 16-byte copies of V^T columns need aligned starts
        max_len = segs.len[i] > max_len ? segs.len[i] : max_len;
        paged = paged || segs.pos0[i] > 0;
    }
    if (paged) {          // every segment then reads its keys from its pages
        if (!k_cache || !v_cache) return cudaErrorInvalidValue;
        for (int i = 0; i < segs.n; ++i)
            if (!segs.table[i]) return cudaErrorInvalidValue;
    }
    FlashParams p{};
    p.q = q; p.k = k; p.vt = vt; p.out = out; p.k_cache = k_cache; p.v_cache = v_cache;
    p.qd = n_head * hd; p.kvd = n_kv * hd; p.vt_ld = vt_ld; p.grp = n_head / n_kv; p.n_kv = n_kv;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.segs = segs;
    const dim3 grid((unsigned)n_head, (unsigned)((max_len + FA_BM - 1) / FA_BM), (unsigned)segs.n);
    if (hd == 128) {
        if (paged) flash_prefill_kernel<128, true><<<grid, FA_THREADS, fa_smem_bytes<128>(), s>>>(p);
        else flash_prefill_kernel<128, false><<<grid, FA_THREADS, fa_smem_bytes<128>(), s>>>(p);
    } else {
        if (paged) flash_prefill_kernel<64, true><<<grid, FA_THREADS, fa_smem_bytes<64>(), s>>>(p);
        else flash_prefill_kernel<64, false><<<grid, FA_THREADS, fa_smem_bytes<64>(), s>>>(p);
    }
    return cudaGetLastError();
}

cudaError_t rope_split_segs_launch(const float* qkv, int rows_pad, int n_head, int n_kv, int hd, const float* cos_t, const float* sin_t, __half* qo,
                                   __half* ko, __half* vt, __half* k_cache, __half* v_cache, int vt_ld, const PrefillSegs& segs, cudaStream_t s) {
    // rows come in whole blocks of eight; the V^T store is 16 bytes wide
    if (segs.n < 1 || segs.n > PF_MAX_SEGS || rows_pad < 1 || (rows_pad % RS_ROWS) || (hd & 1) || (vt_ld & 7) || ((uintptr_t)vt & 15)) return cudaErrorInvalidValue;
    rope_split_segs_kernel<<<rows_pad / RS_ROWS, 256, 0, s>>>(qkv, n_head, n_kv, hd, cos_t, sin_t, qo, ko, vt, k_cache, v_cache, vt_ld, segs);
    return cudaGetLastError();
}

}  // namespace gl
