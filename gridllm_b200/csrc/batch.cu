// Per-sequence kernels of a batched decode step (batch.h): everything of the step that is NOT a weight GEMM.
// Stands in for what Ollama's runner does when it decodes several requests of one model together [external]; on the
// reference side only MAX_CONCURRENT_JOBS_PER_WORKER (server/src/config/index.ts:31) and the worker's busy-drop
// (client/src/services/WorkerClientService.ts:500-505) decide whether a worker ever sees more than one request.
#include "batch.h"

#include <algorithm>
#include <cstdlib>

#include "attn_core.cuh"
#include "common.cuh"

namespace gl {

namespace {

__global__ void __launch_bounds__(MAX_BATCH) batch_gather_tokens_kernel(const BatchCtl* __restrict__ ctl, const StepState* __restrict__ st,
                                                                        int* __restrict__ ids, int bucket) {
    const int r = threadIdx.x;
    if (r >= bucket) return;
    ids[r] = r < ctl->n_rows ? st[ctl->row_slot[r]].token : 0;
}

// Same arithmetic as the EPI_QKV epilogue of the decode GEMV (fp32 rotate of adjacent pairs, fp16 cache), one CTA per row.
__global__ void __launch_bounds__(256) batch_rope_kv_kernel(const float* __restrict__ qkv, const BatchCtl* __restrict__ ctl,
                                                            const StepState* __restrict__ st, const int* __restrict__ tables, int table_stride,
                                                            int n_head, int n_kv, int hd, const float* __restrict__ cos_t,
                                                            const float* __restrict__ sin_t, float* __restrict__ q_out,
                                                            __half* __restrict__ k_cache, __half* __restrict__ v_cache) {
    pdl_launch_dependents();                        // the next kernel of the step may start its own prologue (qgemm: its weight stream)
    pdl_wait();                                     // ... while this one waits here for the QKV rows
    const int r = blockIdx.x;
    if (r >= ctl->n_rows) return;
    const int slot = ctl->row_slot[r];
    const int pos = st[slot].pos;
    const int page = tables[(size_t)slot * table_stride + pos / KV_PAGE_TOKENS], tok = pos % KV_PAGE_TOKENS;
    const int qd = n_head * hd, kvd = n_kv * hd, ld = qd + 2 * kvd;
    const float* row = qkv + (size_t)r * ld;
    // blockIdx.y: the row's work is cut into gridDim.y slices (one CTA per row left 32 CTAs walking ten dependent loads each)
    const int tid = blockIdx.y * 256 + threadIdx.x, nthr = gridDim.y * 256;
    for (int i = tid; i < (qd + kvd) / 2; i += nthr) {
        const int e = 2 * i, d = e % hd;
        const float c = cos_t[(size_t)pos * (hd / 2) + d / 2], s = sin_t[(size_t)pos * (hd / 2) + d / 2];
        const float a = row[e], b = row[e + 1];
        const float o0 = a * c - b * s, o1 = a * s + b * c;
        if (e < qd) {
            *reinterpret_cast<float2*>(q_out + (size_t)r * qd + e) = make_float2(o0, o1);
        } else {
            const int ek = e - qd, kvh = ek / hd;
            const size_t off = (((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d;
            *reinterpret_cast<__half2*>(k_cache + off) = __halves2half2(__float2half_rn(o0), __float2half_rn(o1));
        }
    }
    for (int i = tid; i < kvd / 2; i += nthr) {
        const int e = 2 * i, kvh = e / hd, d = e % hd;
        const size_t off = (((size_t)page * n_kv + kvh) * KV_PAGE_TOKENS + tok) * hd + d;
        *reinterpret_cast<__half2*>(v_cache + off) =
            __halves2half2(__float2half_rn(row[qd + kvd + e]), __float2half_rn(row[qd + kvd + e + 1]));
    }
}

// Paged decode attention for B rows at once: grid (KV head, split, row); a CTA = the GQA group of one KV head of one row
// (one warp per query head, lanes own head dims), split s owns that row's pages s, s + S, ...; pages travel as 1-D TMA bulk
// copies (a page of one KV head is one contiguous 4 KB block), four pages per round trip; partials are merged by the last
// CTA of each (row, KV head) -- atomic ticket -- and the merged row is written as fp16, the operand of the attn_output GEMM.
// The page arithmetic is the single-sequence kernel's (attn_core.cuh): same scores, same online softmax.
constexpr int B_TILE_PAGES = 4;
constexpr int B_MAX_GRP = 8;

template <int DPL>
__global__ void __launch_bounds__(32 * B_MAX_GRP) batch_attn_kernel(const __grid_constant__ BatchAttnParams p) {
    constexpr int HD = DPL * 32;
    constexpr int PAGE_ELEMS = KV_PAGE_TOKENS * HD;
    constexpr uint32_t PAGE_BYTES = PAGE_ELEMS * sizeof(__half);
    __shared__ __align__(128) __half ks[B_TILE_PAGES * PAGE_ELEMS];
    __shared__ __align__(128) __half vs[B_TILE_PAGES * PAGE_ELEMS];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int is_last;

    const int row = blockIdx.z;
    if (row >= p.ctl->n_rows) return;
    const int slot = p.ctl->row_slot[row];
    const int* table = p.tables + (size_t)slot * p.table_stride;
    const int kvh = blockIdx.x, split = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = p.n_head / p.n_kv_heads;
    const int head = kvh * grp + warp;
    const int S = p.n_splits;
    const int L = p.st[slot].pos + 1;                 // this step's K / V row was appended by the launch before this one
    const int n_pages = (L + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    const int active = min(n_pages, S);
    if (split >= active) return;
    const int my_pages = (n_pages - split + S - 1) / S;

    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    __syncthreads();

    float q[DPL], o[DPL];
    {
        const float* qp = p.q + ((size_t)row * p.n_head + head) * HD + lane * DPL;
        if (DPL == 4) {
            const float4 t = *reinterpret_cast<const float4*>(qp);
            q[0] = t.x; q[1] = t.y; q[DPL - 2] = t.z; q[DPL - 1] = t.w;
        } else {
            const float2 t = *reinterpret_cast<const float2*>(qp);
            q[0] = t.x; q[1] = t.y;
        }
#pragma unroll
        for (int d = 0; d < DPL; ++d) { q[d] *= p.scale; o[d] = 0.f; }
    }
    float m_run = -INFINITY, l_run = 0.f;
    uint32_t ph = 0;
    for (int t0 = 0; t0 < my_pages; t0 += B_TILE_PAGES) {
        const int np = min(B_TILE_PAGES, my_pages - t0);
        if (warp == 0) {
            if (lane == 0) mbar_expect_tx(&bar, 2u * np * PAGE_BYTES);
            __syncwarp();
            if (lane < np) {
                const int page = table[split + (t0 + lane) * S];
                const size_t off = ((size_t)page * p.n_kv_heads + kvh) * PAGE_ELEMS;
                tma_load_1d(ks + lane * PAGE_ELEMS, p.k_cache + off, PAGE_BYTES, &bar);
                tma_load_1d(vs + lane * PAGE_ELEMS, p.v_cache + off, PAGE_BYTES, &bar);
            }
        }
        mbar_wait(&bar, ph);
        ph ^= 1;
        for (int i = 0; i < np; ++i) {
            const int pg = split + (t0 + i) * S;
            attn_page_math_smem<DPL>(ks + i * PAGE_ELEMS + lane * DPL, vs + i * PAGE_ELEMS + lane * DPL,
                                     min(KV_PAGE_TOKENS, L - pg * KV_PAGE_TOKENS), q, o, m_run, l_run);
        }
        // every thread has seen this phase complete (and is done with the tile) before the barrier is armed again
        if (t0 + B_TILE_PAGES < my_pages) __syncthreads();
    }

    __half* out = p.out16 + ((size_t)row * p.n_head + head) * HD + lane * DPL;
    if (active == 1) {
        const float inv = 1.0f / l_run;
#pragma unroll
        for (int d = 0; d < DPL; d += 2)
            *reinterpret_cast<__half2*>(out + d) = __halves2half2(__float2half_rn(o[d] * inv), __float2half_rn(o[d + 1] * inv));
        return;
    }
    const size_t pbase = ((size_t)row * p.n_head + head) * S;
    {
        float* po = p.part_o + (pbase + split) * HD + lane * DPL;
#pragma unroll
        for (int d = 0; d < DPL; ++d) po[d] = o[d];
        if (lane == 0) {
            p.part_ml[(pbase + split) * 2] = m_run;
            p.part_ml[(pbase + split) * 2 + 1] = l_run;
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned* ctr = p.counters + (size_t)row * p.n_kv_heads + kvh;
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(ctr) : "memory");
        is_last = (ticket == (unsigned)active - 1);
        if (is_last) *ctr = 0;                         // ready for the next launch
    }
    __syncthreads();
    if (!is_last) return;
    // merge in split order (fixed order: the result does not depend on which CTA came last)
    float M = -INFINITY;
    for (int s2 = 0; s2 < active; ++s2) M = fmaxf(M, __ldcg(p.part_ml + (pbase + s2) * 2));
    float den = 0.f, acc[DPL];
#pragma unroll
    for (int d = 0; d < DPL; ++d) acc[d] = 0.f;
    for (int s2 = 0; s2 < active; ++s2) {
        const float w = expf(__ldcg(p.part_ml + (pbase + s2) * 2) - M);
        den += w * __ldcg(p.part_ml + (pbase + s2) * 2 + 1);
        const float* po = p.part_o + (pbase + s2) * HD + lane * DPL;
#pragma unroll
        for (int d = 0; d < DPL; ++d) acc[d] += w * __ldcg(po + d);
    }
    const float inv = 1.0f / den;
#pragma unroll
    for (int d = 0; d < DPL; d += 2)
        *reinterpret_cast<__half2*>(out + d) = __halves2half2(__float2half_rn(acc[d] * inv), __float2half_rn(acc[d + 1] * inv));
}


// ---- the same attention on the tensor cores (mma.sync m16n8k16) --------------------------------------------------------------
// The kernel above spends ~560 instructions per (page, query head): with B = 32 sequences at 576 tokens that is 20 M warp
// instructions per layer, 39 us of a step in which the KV bytes themselves need 12 us.  Here ONE warp serves
// all the query heads of a KV head at once: the GQA group is the M dimension of the MMA (rows = query heads, padded to 16),
// S = Q K^T and O += P V are 32 tensor-core instructions per 16-token page instead of ~2 000 scalar ones.
//   grid (KV head, split, row), 4 warps; the CTA's pages (split s: pages s, s + S, ...) are dealt round-robin to the warps;
//   each warp streams its pages with cp.async (16-byte chunks, XOR-swizzled by the row so that ldmatrix is conflict-free)
//   through its own double buffer -- no CTA barrier inside the loop; K fragments by ldmatrix, V fragments by ldmatrix.trans;
//   online softmax per query head in the accumulator layout; the four warps' partial (m, l, O) are merged through shared
//   memory, the splits through the same atomic ticket as above.  Bound: HBM (KV pages).
template <int HD> struct BamCfg {
    static constexpr int ROW_BYTES = HD * 2;
    static constexpr int PAGE_BYTES = KV_PAGE_TOKENS * ROW_BYTES;
    static constexpr int CHUNKS_PER_ROW = ROW_BYTES / 16;
    static constexpr int NBUF = 3;                               // pages in flight per warp: two ahead of the one being multiplied
    static constexpr int WARP_BYTES = NBUF * 2 /*K, V*/ * PAGE_BYTES;
    static constexpr size_t SMEM = (size_t)4 * WARP_BYTES;       // 96 KB (head_dim 128): two CTAs per SM; the merge reuses the page buffers
    static_assert(8 * (HD + 2) * 4 <= WARP_BYTES, "a warp's (m, l, O) of 8 heads must fit its own page buffers");
};

__device__ __forceinline__ void bam_cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void bam_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bam_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bam_ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void bam_ldmatrix_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// D (fp32, 16 x 8) += A (fp16, 16 x 16, row) * B (fp16, 16 x 8, col)
__device__ __forceinline__ void bam_mma(float* d, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t bam_pack(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

template <int HD>
__global__ void __launch_bounds__(128, 2) batch_attn_mma_kernel(const __grid_constant__ BatchAttnParams p) {
    using Cfg = BamCfg<HD>;
    constexpr int KSTEPS = HD / 16, NT = HD / 8;
    extern __shared__ __align__(128) uint8_t bam_smem[];
    __shared__ int is_last;

    pdl_launch_dependents();
    pdl_wait();                                     // q and the newest K / V rows come from the kernel before
    const int row = blockIdx.z;
    if (row >= p.ctl->n_rows) return;
    const int slot = p.ctl->row_slot[row];
    const int* table = p.tables + (size_t)slot * p.table_stride;
    const int kvh = blockIdx.x, split = blockIdx.y, S = p.n_splits;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int grp = p.n_head / p.n_kv_heads;
    const int L = p.st[slot].pos + 1;
    const int n_pages = (L + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    const int active = min(n_pages, S);
    if (split >= active) return;
    const int my_pages = (n_pages - split + S - 1) / S;              // pages of this CTA: split, split + S, ...
    const int w_pages = (my_pages - warp + 3) / 4;                   // ... of which this warp takes every fourth

    uint8_t* wbuf = bam_smem + (size_t)warp * Cfg::WARP_BYTES;

    // Q fragments: rows = the group's query heads (g < grp), pre-scaled, fp16.  Rows 8..15 of the MMA tile stay zero.
    // Fused mode: the raw q row is rotated here (a thread's two elements per k-step half are one adjacent RoPE pair).
    const bool fused = p.qkv != nullptr;
    const float* cs = fused ? p.cos_t + (size_t)(L - 1) * (HD / 2) : nullptr;
    const float* sn = fused ? p.sin_t + (size_t)(L - 1) * (HD / 2) : nullptr;
    uint32_t qa[KSTEPS][2];
    {
        const float* q = fused ? p.qkv + (size_t)row * p.ld_qkv + ((size_t)kvh * grp + g) * HD
                               : p.q + ((size_t)row * p.n_head + (size_t)kvh * grp + g) * HD;
#pragma unroll
        for (int ks = 0; ks < KSTEPS; ++ks) {
            float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
            if (g < grp) {
                lo = *reinterpret_cast<const float2*>(q + ks * 16 + 2 * t);
                hi = *reinterpret_cast<const float2*>(q + ks * 16 + 8 + 2 * t);
                if (fused) {
                    const float c0 = cs[ks * 8 + t], s0 = sn[ks * 8 + t], c1 = cs[ks * 8 + 4 + t], s1 = sn[ks * 8 + 4 + t];
                    lo = make_float2(lo.x * c0 - lo.y * s0, lo.x * s0 + lo.y * c0);
                    hi = make_float2(hi.x * c1 - hi.y * s1, hi.x * s1 + hi.y * c1);
                }
            }
            qa[ks][0] = bam_pack(lo.x * p.scale, lo.y * p.scale);
            qa[ks][1] = bam_pack(hi.x * p.scale, hi.y * p.scale);
        }
    }
    // the newest position's K / V rows: who owns its page?
    const int pg_new = (L - 1) / KV_PAGE_TOKENS, tok_new = (L - 1) % KV_PAGE_TOKENS;
    const int j_new = (fused && pg_new % S == split && ((pg_new - split) / S) % 4 == warp) ? ((pg_new - split) / S) / 4 : -1;
    float o[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) { o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f; }
    float m_run = -INFINITY, l_run = 0.f;

    // physical pages of this warp's pages, 32 at a time: lane l holds the entry of page j0 + l.  Looked up inside issue() the
    // entry was a dependent global load in front of every page's copies (a third of the kernel's stall samples, r02 run J).
    int tbl = 0;
    auto load_tbl = [&](int j0) {
        const int j = j0 + lane;
        tbl = j < w_pages ? table[split + (warp + 4 * j) * S] : 0;
    };
    load_tbl(0);
    auto issue = [&](int j) {          // page j of this warp -> buffer j % NBUF (K then V), 16-byte chunks swizzled by the row
        if ((j & 31) == 0 && j > 0) load_tbl(j);
        const int phys = __shfl_sync(0xffffffffu, tbl, j & 31);
        const size_t off = ((size_t)phys * p.n_kv_heads + kvh) * (size_t)(KV_PAGE_TOKENS * HD);
        const uint8_t* ksrc = reinterpret_cast<const uint8_t*>(p.k_cache + off);
        const uint8_t* vsrc = reinterpret_cast<const uint8_t*>(p.v_cache + off);
        const uint32_t kdst = smem_u32(wbuf + (size_t)(j % Cfg::NBUF) * 2 * Cfg::PAGE_BYTES), vdst = kdst + Cfg::PAGE_BYTES;
#pragma unroll
        for (int i = 0; i < Cfg::PAGE_BYTES / 16 / 32; ++i) {
            const int ci = i * 32 + lane, r = ci / Cfg::CHUNKS_PER_ROW, c = ci % Cfg::CHUNKS_PER_ROW;
            const uint32_t d = (uint32_t)(r * Cfg::ROW_BYTES + ((c ^ (r & 7)) << 4));
            bam_cp_async16(kdst + d, ksrc + (size_t)ci * 16);
            bam_cp_async16(vdst + d, vsrc + (size_t)ci * 16);
        }
        bam_commit();
    };
    // a page costs a full HBM round trip (~1 us under load) and ~0.3 us of math: with ONE page ahead a warp is latency-bound
    // (1.2 us per page, r02 run D); two ahead keep the memory pipe of the warp busy.  One commit group per page, empty when the
    // warp has run out of pages, so that wait_group<NBUF - 1> always means "page j has landed".
#pragma unroll
    for (int j = 0; j < Cfg::NBUF - 1; ++j) { if (j < w_pages) issue(j); else bam_commit(); }
    for (int j = 0; j < w_pages; ++j) {
        if (j + Cfg::NBUF - 1 < w_pages) issue(j + Cfg::NBUF - 1); else bam_commit();
        bam_wait<Cfg::NBUF - 1>();
        __syncwarp();
        const uint32_t kb = smem_u32(wbuf + (size_t)(j % Cfg::NBUF) * 2 * Cfg::PAGE_BYTES), vb = kb + Cfg::PAGE_BYTES;
        const int pg = split + (warp + 4 * j) * S;
        const int npos = min(KV_PAGE_TOKENS, L - pg * KV_PAGE_TOKENS);
        if (j == j_new) {
            // this page holds the position of THIS step: its K / V rows are still in the QKV buffer.  Lane l owns elements 4l..4l+3
            // (two RoPE pairs) of both rows: rotate K, round to fp16, patch the copy in shared memory, and write the cache.
            static_assert(HD == 128 || HD == 64, "lane -> 4 elements of the row");
            if (lane * 4 < HD) {
                const float* kr = p.qkv + (size_t)row * p.ld_qkv + (size_t)p.n_head * HD + (size_t)kvh * HD + lane * 4;
                const float* vr = kr + (size_t)p.n_kv_heads * HD;
                const float4 kx = *reinterpret_cast<const float4*>(kr), vx = *reinterpret_cast<const float4*>(vr);
                const float c0 = cs[lane * 2], s0 = sn[lane * 2], c1 = cs[lane * 2 + 1], s1 = sn[lane * 2 + 1];
                uint2 kw, vw;
                kw.x = bam_pack(kx.x * c0 - kx.y * s0, kx.x * s0 + kx.y * c0);
                kw.y = bam_pack(kx.z * c1 - kx.w * s1, kx.z * s1 + kx.w * c1);
                vw.x = bam_pack(vx.x, vx.y);
                vw.y = bam_pack(vx.z, vx.w);
                const int chunk = lane >> 1;
                const uint32_t d = (uint32_t)(tok_new * Cfg::ROW_BYTES + ((chunk ^ (tok_new & 7)) << 4) + (lane & 1) * 8);
                asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(kb + d), "r"(kw.x), "r"(kw.y) : "memory");
                asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(vb + d), "r"(vw.x), "r"(vw.y) : "memory");
                const int phys_new = table[pg];
                const size_t off = (((size_t)phys_new * p.n_kv_heads + kvh) * KV_PAGE_TOKENS + tok_new) * HD + lane * 4;
                *reinterpret_cast<uint2*>(const_cast<__half*>(p.k_cache) + off) = kw;
                *reinterpret_cast<uint2*>(const_cast<__half*>(p.v_cache) + off) = vw;
            }
            __syncwarp();
        }
        // ---- S = Q K^T : two n-tiles (positions 0-7, 8-15) ----
        float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < KSTEPS; ++ks) {
            // matrices: (pos 0-7, dims k0..+7), (pos 0-7, dims k0+8..+15), (pos 8-15, k0..+7), (pos 8-15, k0+8..+15)
            const int m = lane >> 3, pos = (lane & 7) + 8 * (m >> 1), chunk = 2 * ks + (m & 1);
            uint32_t b0, b1, b2, b3;
            bam_ldmatrix_x4(kb + (uint32_t)(pos * Cfg::ROW_BYTES + ((chunk ^ (pos & 7)) << 4)), b0, b1, b2, b3);
            bam_mma(s0, qa[ks][0], 0u, qa[ks][1], 0u, b0, b1);
            bam_mma(s1, qa[ks][0], 0u, qa[ks][1], 0u, b2, b3);
        }
        // ---- online softmax of row g (query head g): this thread holds columns 2t, 2t+1 of both n-tiles ----
        float v0 = (2 * t < npos) ? s0[0] : -INFINITY, v1 = (2 * t + 1 < npos) ? s0[1] : -INFINITY;
        float v2 = (8 + 2 * t < npos) ? s1[0] : -INFINITY, v3 = (9 + 2 * t < npos) ? s1[1] : -INFINITY;
        float mx = fmaxf(fmaxf(v0, v1), fmaxf(v2, v3));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run, mx);                       // npos >= 1: finite
        const float corr = (m_run == -INFINITY) ? 0.f : expf(m_run - m_new);
        const float p0 = expf(v0 - m_new), p1 = expf(v1 - m_new), p2 = expf(v2 - m_new), p3 = expf(v3 - m_new);      // exp(-inf) = 0
        float ps = (p0 + p1) + (p2 + p3);
        ps += __shfl_xor_sync(0xffffffffu, ps, 1);
        ps += __shfl_xor_sync(0xffffffffu, ps, 2);
        l_run = l_run * corr + ps;
        m_run = m_new;
        // P as the A operand of the second MMA (rows 8..15 zero): k = positions
        const uint32_t pa0 = bam_pack(p0, p1), pa2 = bam_pack(p2, p3);
        // ---- O = O * corr + P V ----
#pragma unroll
        for (int n = 0; n < NT; ++n) { o[n][0] *= corr; o[n][1] *= corr; }
#pragma unroll
        for (int n2 = 0; n2 < NT / 2; ++n2) {
            // transposed loads: (pos 0-7, dims n0..+7), (pos 8-15, n0..+7), (pos 0-7, n0+8..+15), (pos 8-15, n0+8..+15)
            const int m = lane >> 3, pos = (lane & 7) + 8 * (m & 1), chunk = 2 * n2 + (m >> 1);
            uint32_t b0, b1, b2, b3;
            bam_ldmatrix_x4_t(vb + (uint32_t)(pos * Cfg::ROW_BYTES + ((chunk ^ (pos & 7)) << 4)), b0, b1, b2, b3);
            bam_mma(o[2 * n2], pa0, 0u, pa2, 0u, b0, b1);
            bam_mma(o[2 * n2 + 1], pa0, 0u, pa2, 0u, b2, b3);
        }
        __syncwarp();                                                 // every lane is done with this buffer before it is refilled
    }

    // ---- merge the four warps (each holds (m, l, O) of heads g < grp over ITS pages), then the splits ----
    // (each warp writes its partial over its OWN page buffers -- it is done with them -- and reads the others' after the barrier)
    if (g < grp) {
        float* mw = reinterpret_cast<float*>(wbuf) + (size_t)g * (HD + 2);
        if (t == 0) { mw[HD] = m_run; mw[HD + 1] = l_run; }
#pragma unroll
        for (int n = 0; n < NT; ++n) { mw[8 * n + 2 * t] = o[n][0]; mw[8 * n + 2 * t + 1] = o[n][1]; }
    }
    __syncthreads();
    const size_t pbase = ((size_t)row * p.n_head + (size_t)kvh * grp) * S;      // partial slots of this KV head's first query head
    for (int e = threadIdx.x; e < grp * HD; e += 128) {
        const int h = e / HD, d = e % HD;
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < 4; ++w) M = fmaxf(M, reinterpret_cast<const float*>(bam_smem + (size_t)w * Cfg::WARP_BYTES)[(size_t)h * (HD + 2) + HD]);
        float den = 0.f, acc = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float* mw = reinterpret_cast<const float*>(bam_smem + (size_t)w * Cfg::WARP_BYTES) + (size_t)h * (HD + 2);
            const float wgt = (mw[HD] == -INFINITY) ? 0.f : expf(mw[HD] - M);
            den += wgt * mw[HD + 1];
            acc += wgt * mw[d];
        }
        if (active == 1) {
            p.out16[((size_t)row * p.n_head + (size_t)kvh * grp + h) * HD + d] = __float2half_rn(acc / den);
        } else {
            p.part_o[(pbase + (size_t)h * S + split) * HD + d] = acc;
            if (d == 0) {
                p.part_ml[(pbase + (size_t)h * S + split) * 2] = M;
                p.part_ml[(pbase + (size_t)h * S + split) * 2 + 1] = den;
            }
        }
    }
    if (active == 1) return;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned* ctr = p.counters + (size_t)row * p.n_kv_heads + kvh;
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(ctr) : "memory");
        is_last = (ticket == (unsigned)active - 1);
        if (is_last) *ctr = 0;
    }
    __syncthreads();
    if (!is_last) return;
    for (int e = threadIdx.x; e < grp * HD; e += 128) {              // splits in order: the result does not depend on who came last
        const int h = e / HD, d = e % HD;
        const size_t pb = pbase + (size_t)h * S;
        float M = -INFINITY;
        for (int s2 = 0; s2 < active; ++s2) M = fmaxf(M, __ldcg(p.part_ml + (pb + s2) * 2));
        float den = 0.f, acc = 0.f;
        for (int s2 = 0; s2 < active; ++s2) {
            const float wgt = expf(__ldcg(p.part_ml + (pb + s2) * 2) - M);
            den += wgt * __ldcg(p.part_ml + (pb + s2) * 2 + 1);
            acc += wgt * __ldcg(p.part_o + (pb + s2) * HD + d);
        }
        p.out16[((size_t)row * p.n_head + (size_t)kvh * grp + h) * HD + d] = __float2half_rn(acc / den);
    }
}

// Greedy rows: one CTA per row scans the row's logits once (max / lowest argmax / sum of exponentials, the single-sequence
// sampler's arithmetic: ties go to the lowest index; logprob = -log(sum exp(l - max))) and advances the row's StepState.
constexpr int BS_THREADS = 512;
constexpr int BS_PARTS = BATCH_SAMPLE_PARTS;
constexpr int BS_ROW_FLOATS = BATCH_SAMPLE_ROW_FLOATS;
struct BCand { float m; int i; float s; };
__device__ __forceinline__ BCand bcand_merge(BCand a, BCand b) {
    if (b.m > a.m || (b.m == a.m && b.i < a.i)) { const BCand t = a; a = b; b = t; }
    // a is the winner; fold b's mass in
    if (b.m != -INFINITY) a.s += b.s * expf(b.m - a.m);
    return a;
}
__global__ void __launch_bounds__(BS_THREADS) batch_sample_greedy_kernel(const float* __restrict__ logits, int n_vocab,
                                                                         const BatchCtl* __restrict__ ctl, StepState* __restrict__ stv,
                                                                         int* __restrict__ out_ids, float* __restrict__ out_lps, int max_out,
                                                                         float* __restrict__ scratch) {
    // grid (row, part): BS_PARTS CTAs scan a row's logits (one CTA per row left 32 CTAs walking 513 KB each: 73 us of a step);
    // the last one of a row (atomic ticket) merges the parts IN PART ORDER and advances the row's state
    const int row = blockIdx.x, part = blockIdx.y;
    if (row >= ctl->n_rows) return;
    const int slot = ctl->row_slot[row];
    StepState* st = stv + slot;
    if (st->temperature > 0.f) return;               // sampled rows: the seeded top-k sampler runs on them after this kernel
    __shared__ BCand sc[BS_THREADS / 32];
    __shared__ int is_last;
    const float* lg = logits + (size_t)row * n_vocab;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (n_vocab + BS_PARTS - 1) / BS_PARTS, i0 = part * per, i1 = min(n_vocab, i0 + per);
    BCand c{-INFINITY, 0x7fffffff, 0.f};
    for (int i = i0 + tid; i < i1; i += BS_THREADS) {
        const float v = lg[i];
        if (v > c.m) {                               // ascending indices per thread: strict > keeps the lowest on ties
            c.s = (c.m == -INFINITY ? 0.f : c.s * expf(c.m - v)) + 1.f;
            c.m = v;
            c.i = i;
        } else if (v != -INFINITY) {
            c.s += expf(v - c.m);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        BCand t{__shfl_xor_sync(0xffffffffu, c.m, o), __shfl_xor_sync(0xffffffffu, c.i, o), __shfl_xor_sync(0xffffffffu, c.s, o)};
        c = bcand_merge(c, t);
    }
    if (lane == 0) sc[warp] = c;
    __syncthreads();
    float* rs = scratch + (size_t)row * BS_ROW_FLOATS;      // [BS_PARTS][m, i, s] + ticket
    if (tid == 0) {
        BCand t = sc[0];
        for (int w = 1; w < BS_THREADS / 32; ++w) t = bcand_merge(t, sc[w]);
        rs[part * 3] = t.m;
        reinterpret_cast<int*>(rs)[part * 3 + 1] = t.i;
        rs[part * 3 + 2] = t.s;
        __threadfence();
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(reinterpret_cast<unsigned*>(rs) + 3 * BS_PARTS) : "memory");
        is_last = ticket == (unsigned)BS_PARTS - 1;
        if (is_last) reinterpret_cast<unsigned*>(rs)[3 * BS_PARTS] = 0;
    }
    __syncthreads();
    if (!is_last || tid != 0) return;
    BCand t{__ldcg(rs), __ldcg(reinterpret_cast<const int*>(rs) + 1), __ldcg(rs + 2)};
    for (int k = 1; k < BS_PARTS; ++k) t = bcand_merge(t, BCand{__ldcg(rs + 3 * k), __ldcg(reinterpret_cast<const int*>(rs) + 3 * k + 1), __ldcg(rs + 3 * k + 2)});
    if (st->done) return;
    const int out_idx = st->out_idx;
    if (out_idx < max_out) {
        out_ids[(size_t)slot * max_out + out_idx] = t.i;
        out_lps[(size_t)slot * max_out + out_idx] = -logf(t.s);
    }
    st->token = t.i;
    st->pos = st->pos + 1;
    st->out_idx = out_idx + 1;
    if (!st->ignore_eos) {
        for (int k = 0; k < st->n_stop; ++k)
            if (st->stop_ids[k] == t.i) st->done = 1;
    }
}

__global__ void __launch_bounds__(MAX_BATCH) batch_collect_kernel(const BatchCtl* __restrict__ ctl, const StepState* __restrict__ st,
                                                                  const float* __restrict__ out_lps, int max_out, BatchOut* __restrict__ out,
                                                                  int bucket) {
    const int r = threadIdx.x;
    if (r >= bucket) return;
    BatchOut o{0, 0.f, 0, 0};
    if (r < ctl->n_rows) {
        const int slot = ctl->row_slot[r];
        const StepState& s = st[slot];
        o.token = s.token;
        o.done = s.done;
        o.pos = s.pos;
        const int k = s.out_idx - 1;
        o.logprob = (k >= 0 && k < max_out) ? out_lps[(size_t)slot * max_out + k] : 0.f;
    }
    out[r] = o;
}

__global__ void __launch_bounds__(256) batch_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, int n, float eps,
                                                            __half* __restrict__ y) {
    pdl_launch_dependents();
    pdl_wait();
    const int r = blockIdx.x;
    __shared__ float red[8];
    const float* xr = x + (size_t)r * n;
    __half* yr = y + (size_t)r * n;
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) { const float v = xr[i]; ss += v * v; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += red[k];
    const float rstd = 1.0f / sqrtf(tot / (float)n + eps);
    for (int i = threadIdx.x; i < n; i += 256) yr[i] = __float2half_rn((xr[i] * rstd) * w[i]);
}

// launch with the programmatic-dependent-launch attribute: the kernel may become resident while its predecessor in the stream
// is still running and blocks in pdl_wait() before it touches anything (GL_BATCH_PDL=0: plain stream order, for A/B runs)
template <typename... Args>
cudaError_t launch_dep(void (*kern)(Args...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = batch_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

}  // namespace

bool batch_pdl_enabled() {
    static const bool on = []() { const char* e = getenv("GL_BATCH_PDL"); return !(e && e[0] == '0'); }();
    return on;
}

cudaError_t batch_gather_tokens_launch(const BatchCtl* ctl, const StepState* st, int* ids, int bucket, cudaStream_t s) {
    batch_gather_tokens_kernel<<<1, MAX_BATCH, 0, s>>>(ctl, st, ids, bucket);
    return cudaGetLastError();
}

cudaError_t batch_rope_kv_launch(const float* qkv, int bucket, const BatchCtl* ctl, const StepState* st, const int* tables, int table_stride,
                                 int n_head, int n_kv, int hd, const float* cos_t, const float* sin_t, float* q_out, __half* k_cache,
                                 __half* v_cache, cudaStream_t s) {
    const int slices = std::max(1, std::min(8, ((n_head + n_kv) * hd / 2 + 255) / 256));
    return launch_dep(batch_rope_kv_kernel, dim3((unsigned)bucket, (unsigned)slices), dim3(256), 0, s, qkv, ctl, st, tables, table_stride, n_head, n_kv, hd,
                      cos_t, sin_t, q_out, k_cache, v_cache);
}

cudaError_t batch_attn_configure() {
    cudaError_t e = cudaFuncSetAttribute(batch_attn_mma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BamCfg<128>::SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(batch_attn_mma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BamCfg<64>::SMEM);
    return e;
}

static bool batch_attn_use_mma() {
    static const bool on = []() { const char* e = getenv("GL_BATCH_ATTN_MMA"); return !(e && e[0] == '0'); }();
    return on;
}
bool batch_attn_fuses_rope(int head_dim) {
    static const bool on = []() { const char* e = getenv("GL_BATCH_FUSE_ROPE"); return !(e && e[0] == '0'); }();
    return on && batch_attn_use_mma() && (head_dim == 128 || head_dim == 64);
}

cudaError_t batch_attn_launch(const BatchAttnParams& p, int bucket, cudaStream_t s) {
    const int grp = p.n_head / p.n_kv_heads;
    if (grp < 1 || grp > B_MAX_GRP || p.n_head % p.n_kv_heads || p.n_splits < 1 || p.n_splits > 32) return cudaErrorInvalidValue;
    const dim3 grid((unsigned)p.n_kv_heads, (unsigned)p.n_splits, (unsigned)bucket);
    const bool use_mma = batch_attn_use_mma();
    if (p.qkv != nullptr && !use_mma) return cudaErrorInvalidValue;          // only the tensor-core kernel rotates and appends
    if (use_mma) {       // tensor-core kernel (default); GL_BATCH_ATTN_MMA=0 keeps the scalar one for A/B runs
        if (p.head_dim == 128) return launch_dep(batch_attn_mma_kernel<128>, grid, dim3(128), (size_t)BamCfg<128>::SMEM, s, p);
        if (p.head_dim == 64) return launch_dep(batch_attn_mma_kernel<64>, grid, dim3(128), (size_t)BamCfg<64>::SMEM, s, p);
        return cudaErrorInvalidValue;
    }
    if (p.head_dim == 128) batch_attn_kernel<4><<<grid, 32 * grp, 0, s>>>(p);
    else if (p.head_dim == 64) batch_attn_kernel<2><<<grid, 32 * grp, 0, s>>>(p);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t batch_sample_greedy_launch(const float* logits, int n_vocab, int bucket, const BatchCtl* ctl, StepState* st, int* out_ids,
                                       float* out_lps, int max_out, float* scratch, cudaStream_t s) {
    batch_sample_greedy_kernel<<<dim3((unsigned)bucket, BS_PARTS), BS_THREADS, 0, s>>>(logits, n_vocab, ctl, st, out_ids, out_lps, max_out, scratch);
    return cudaGetLastError();
}

cudaError_t batch_collect_launch(const BatchCtl* ctl, const StepState* st, const float* out_lps, int max_out, BatchOut* out, int bucket,
                                 cudaStream_t s) {
    batch_collect_kernel<<<1, MAX_BATCH, 0, s>>>(ctl, st, out_lps, max_out, out, bucket);
    return cudaGetLastError();
}

cudaError_t batch_rmsnorm_launch(const float* x, const float* w, int rows, int n, float eps, __half* y, cudaStream_t s) {
    if (rows <= 0) return cudaSuccess;
    return launch_dep(batch_rmsnorm_kernel, dim3((unsigned)rows), dim3(256), 0, s, x, w, n, eps, y);
}

}  // namespace gl
