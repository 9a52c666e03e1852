// Batched decode GEMM on QUANTISED weights: C[b][n] = sum_k act[b][k] * dequant(W)[n][k] for the B <= 64 sequences of one batched
// decode step (continuous batching, SURVEY.md section 8f.1).  The weights stay in their GGUF bit budget in HBM (Q4_K 4.5 /
// Q6_K 6.5625 bits per weight) and are read ONCE per step for all sequences; they become fp16 tensor-core operands tile by
// tile inside the kernel.  Reference side: the decode loop of several concurrent requests inside Ollama behind
// OllamaService.generate*Response (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237) once the worker holds
// more than one job (WorkerClientService.ts:500-505; MAX_CONCURRENT_JOBS_PER_WORKER, server/src/config/index.ts:31).
//
// Bound: HBM.  A step streams the model's 4.6 GB once; at B = 32 the tensor work is 128 x 32 x 64 MACs per 16 KB of weights
// (a few dozen tensor-core cycles against ~1 000 cycles of HBM time per qtile and SM), so the tensor pipe idles and the CUDA cores'
// job -- ~2.3 lane-operations per weight to unpack nibbles into fp16 -- is what has to keep up with the memory pipe.
//
// Shape of the kernel (persistent, one CTA per SM, 16 warps, hand-written PTX; layouts and the per-thread unpack program in
// qgemm_layout.h, which the CPU suite runs bit for bit):
//   the weights of a GEMM are a stream of QTILES (128 rows x 256 columns, one contiguous 18 / 26 KB range each); the U = tiles x
//   K-blocks qtiles are dealt to the G CTAs as contiguous ranges [c U / G, (c+1) U / G) ("stream-K": perfect balance for every
//   shape -- 32 tiles x 16 blocks on 132 SMs as well as 1002 x 16 -- and every CTA streams ONE contiguous byte range);
//   warp 0 / one lane : weight producer -- per qtile one 1-D TMA bulk copy of the raw bytes into a 2-8 stage ring (the shared
//                       memory the operands leave);
//   warp 1 / one lane : activation producer -- four 2-D TMA boxes [B x 64] fp16 per qtile (L2-resident);
//   warps 4..11       : unpack -- thread (row, half) turns 128 columns of its row into 2 x 32 packed half2 registers and stores
//                       them into the A operand of the qtile in shared memory (four K-steps [128 rows x 64] fp16, 128-byte
//                       swizzle); the next qtile's first K-step is unpacked into registers while the MMAs of this one run;
//   warps 12..15      : one warpgroup: MMA and epilogue -- per qtile 32 wgmma.m64nBk16 (two 64-row halves x 16 K-steps of 16,
//                       A and B from shared memory, fp32 accumulator in registers); after the last qtile of an output tile the
//                       accumulator is staged in the consumed A operand (row-contiguous per batch column) and each thread runs
//                       the fused epilogue of one weight row (fp32 store, residual add, SiLU*mul -> fp16).  An output tile
//                       whose K range is shared with neighbouring CTAs is finished by the lowest-numbered of them (its part of
//                       the tile is the END of its range, the others' the START of theirs): the others store their partial to
//                       scratch and count themselves in, the finisher adds the partials IN CTA ORDER (deterministic) to its
//                       accumulator and runs the epilogue.
// SASS to look for: HGMMA (wgmma), UBLKCP (1-D bulk copy), UTMALDG (2-D TMA).
#include <cuda.h>
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "batch.h"
#include "common.cuh"
#include "qgemm.h"
#include "qgemm_layout.h"
#include "wgmma.cuh"

namespace gl {

namespace {

constexpr int QG_THREADS = 16 * 32;
constexpr int QG_W_UNPACK0 = 4, QG_N_UNPACK = 8, QG_W_EPI0 = 12;    // the MMA / epilogue warps are one warpgroup (warp index % 4 == 0)
constexpr int QG_A_BYTES = 4 * QG_ROWS * QG_KSTEP * 2;               // the A operand of one qtile: four K-steps [128 x 64] fp16 (64 KB)
constexpr int QG_STG_LD = QG_ROWS + 4;                               // accumulator staging: [NB][132] fp32, row-contiguous per batch column
constexpr size_t QG_SMEM = 227 * 1024;               // the whole opt-in shared memory; the raw ring takes what the operands leave

template <int NB> struct QCfg {
    static constexpr int B_TILE = NB * 128;          // activations [NB rows x 64] fp16, 128-byte swizzle
    static constexpr int ACT_BYTES = 4 * B_TILE;
    static constexpr int BAR_BYTES = 1536;         // mbarriers, folded-RMSNorm scratch (64 + 128 floats)
    static constexpr int CK_BYTES = 2 * 4 * NB * 32 * 4;       // cluster mode: two rounds x four source ranks x [NB columns][32 rows] fp32
    static constexpr int RAW_BUDGET = (int)QG_SMEM - 1024 /* alignment */ - BAR_BYTES - ACT_BYTES - QG_A_BYTES;
    static_assert(NB * QG_STG_LD * 4 <= QG_A_BYTES, "the accumulator staging lives in the A operand");
};
constexpr int QG_MAX_RAW_STAGES = 8;

struct QParams {
    CUtensorMap tb;              // activations: dims {K, rows_alloc}, box {64, NB}, 128-byte swizzle
    const uint8_t* w;
    const uint64_t* tile_off;    // per-tile tables: only when the GEMM's tiles are not "type0 up to tile_split, then type1"
    const uint8_t* tile_type;
    unsigned* counters;
    float* partial;              // [grid][NB * 128]: a CTA's part of the tile it shares with lower-numbered CTAs
    void* c;
    int ldc, epi, n, n_tiles, nkb;
    int type0, type1, tile_split;          // tiles [0, tile_split) are type0, the rest type1 (Q | K | V with a Q6_K V); tile_split = n_tiles when uniform
    unsigned long long off_split;          // byte offset of tile tile_split
    int raw_stride, raw_stages;            // raw ring geometry: stride = the largest qtile of this GEMM (18 432 or 27 648)
    int ck_s;                              // 0: stream-K over the whole grid; 4: clusters of four CTAs share tiles, K split in quarters
    // folded RMSNorm (qgemm.h, QGemmNorm)
    const float* gamma_next;
    __half* xg_out;
    int ldxg;
    float* ssq_out;
    const float* ssq_in;
    int ssq_parts, n_norm;
    float eps;
    unsigned long long* trace;             // GL_QGEMM_TRACE=1: [grid][QG_TRACE_SLOTS] %globaltimer stamps of this launch (tools/qgemm_trace.py); else null
};
constexpr int QG_TRACE_SLOTS = 10, QG_TRACE_LAUNCHES = 1024;
__device__ __forceinline__ void q_stamp(const QParams& p, int slot) {
    if (p.trace) p.trace[(size_t)blockIdx.x * QG_TRACE_SLOTS + slot] = globaltimer_ns();
}

__device__ __forceinline__ void tma_load_2d_q(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// the range of qtile units CTA c owns, and who shares an output tile with whom
__device__ __forceinline__ long long q_range_start(int c, long long U, int G) { return (long long)c * U / G; }
// largest c with range_start(c) <= x
__device__ __forceinline__ int q_owner_of(long long x, long long U, int G) { return (int)(((x + 1) * G + U - 1) / U) - 1; }

// type and byte offset of a tile: arithmetic for the common shapes (no dependent global loads in front of the first TMA)
__device__ __forceinline__ int q_tile_type(const QParams& p, int tile) {
    if (p.tile_type != nullptr) return __ldg(p.tile_type + tile);
    return tile < p.tile_split ? p.type0 : p.type1;
}
__device__ __forceinline__ unsigned long long q_tile_off(const QParams& p, int tile) {
    if (p.tile_off != nullptr) return __ldg(p.tile_off + tile);
    return tile < p.tile_split ? (unsigned long long)tile * p.nkb * (unsigned)qg_qtile_bytes(p.type0)
                               : p.off_split + (unsigned long long)(tile - p.tile_split) * p.nkb * (unsigned)qg_qtile_bytes(p.type1);
}

// fused epilogue of 16 batch columns [b0, b0 + 16) of output feature n (v[i] = C[b0 + i][n])
__device__ __forceinline__ void q_epilogue16(const QParams& p, int n, int lane, int b0, float* v, const float* inv) {
    if (inv != nullptr) {                // folded RMSNorm: the activations carried x * gamma / 16, the token's 16 / rms comes here
#pragma unroll
        for (int b = 0; b < 16; ++b) v[b] *= inv[b0 + b];
    }
    if (p.epi == GEMM_EPI_SILU) {
        // weight rows are interleaved [8 gate | 8 up] at load: lane l of a 16-lane group holds gate (l < 8) or up (l >= 8) of
        // hidden column (n / 16) * 8 + l % 8
        __half* out = reinterpret_cast<__half*>(p.c);
        const int hcol = (n >> 4) * 8 + (n & 7);
#pragma unroll
        for (int b = 0; b < 16; ++b) {
            const float up = __shfl_xor_sync(0xffffffffu, v[b], 8);
            if ((lane & 8) == 0 && n < p.n) {
                const float g = v[b];
                out[(size_t)(b0 + b) * p.ldc + hcol] = __float2half_rn((g / (1.0f + expf(-g))) * up);
            }
        }
        return;
    }
    if (n >= p.n) return;
    float* out = reinterpret_cast<float*>(p.c) + (size_t)b0 * p.ldc + n;
    if (p.epi == GEMM_EPI_ADD_F32) {
        // all sixteen loads first: written as load / add / store per element the compiler must keep them in order (it cannot
        // prove the rows distinct), and sixteen L2 round trips in a row are 15 us per launch
        float old[16];
#pragma unroll
        for (int b = 0; b < 16; ++b) old[b] = __ldcg(out + (size_t)b * p.ldc);
#pragma unroll
        for (int b = 0; b < 16; ++b) out[(size_t)b * p.ldc] = old[b] + v[b];
    } else {
#pragma unroll
        for (int b = 0; b < 16; ++b) out[(size_t)b * p.ldc] = v[b];
    }
}

// ---- the CTA's sequence of qtiles ------------------------------------------------------------------------------------------------
// stream-K   : a contiguous range of the GEMM's U = tiles x K-blocks units: (tile, kb) advances kb-first through whole tiles;
// cluster    : (QParams::ck_s = 4) the four CTAs of a thread-block cluster share output tiles: rank r owns K-blocks
//              [r nkb / 4, (r + 1) nkb / 4) of the tiles cluster, cluster + n_clusters, ... -- tile-aligned split-K, the partials
//              meet in DISTRIBUTED SHARED MEMORY (below) instead of going through L2.
struct QWalk {
    int n;                       // units of this CTA
    int tile0, kb0;              // first unit
    int kb_begin, kb_end;        // K-block range of every segment after the first
    int tile_step;
    __device__ __forceinline__ void advance(int& tile, int& kb, int steps) const {
        kb += steps;
        while (kb >= kb_end) { kb -= kb_end - kb_begin; tile += tile_step; }
    }
};
__device__ __forceinline__ uint32_t q_cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t q_mapa(uint32_t local_smem_addr, uint32_t rank) {      // the same location in CTA `rank` of the cluster
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_smem_addr), "r"(rank));
    return ra;
}
__device__ __forceinline__ void q_st_cluster_f32(uint32_t cluster_addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void q_arrive_cluster(uint32_t cluster_bar_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar_addr) : "memory");
}
__device__ __forceinline__ void q_wait_cluster(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    uint32_t done = 0, spins = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(a), "r"(parity) : "memory");
        if (!done && ++spins > (1u << 22)) __trap();
    }
}
constexpr int QG_CK = 4;                                       // cluster size of the tile-aligned split-K mode

template <int NB>
__global__ void __launch_bounds__(QG_THREADS, 1) qgemm_kernel(const __grid_constant__ QParams p) {
    using Cfg = QCfg<NB>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* act_ring = smem;                                                 // [4][NB x 64 fp16]          TMA (L2)      -> tensor core
    uint8_t* a_op = act_ring + Cfg::ACT_BYTES;                                // [4][128 x 64 fp16]         unpack warps  -> tensor core
    float* stg = reinterpret_cast<float*>(a_op);                              // [NB][QG_STG_LD] fp32       accumulator staging (A consumed)
    float* recv = reinterpret_cast<float*>(a_op + QG_A_BYTES);                // cluster mode: [2 rounds][4 ranks][NB][32 rows] partial slices
    uint8_t* raw_ring = a_op + QG_A_BYTES + (p.ck_s ? Cfg::CK_BYTES : 0);     // [raw_stages][raw_stride]  TMA (HBM)     -> unpack warps
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (QG_SMEM - 1024 - Cfg::BAR_BYTES));
    uint64_t* raw_full = bars;                               // [8]  producer (tx bytes)                     -> unpack warps
    uint64_t* raw_empty = raw_full + QG_MAX_RAW_STAGES;      // [8]  the unpack warps                        -> producer
    uint64_t* unit_full = raw_empty + QG_MAX_RAW_STAGES;     // [1]  unpack warps + activations (tx bytes)   -> MMA warpgroup
    uint64_t* unit_empty = unit_full + 1;                    // [1]  MMA warpgroup                           -> unpack warps, activation producer
    uint64_t* recv_bar = unit_empty + 1;                     // [2]  cluster mode: 4 ranks' epilogue warps    -> this rank's epilogue
    float* inv_s = reinterpret_cast<float*>(recv_bar + 2);   // [64] folded RMSNorm: 16 / rms of every token of the step

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = gridDim.x, cta = blockIdx.x;
    const int nkb = p.nkb;
    if (threadIdx.x == 0) q_stamp(p, 0);                                      // CTA entry
    const int U = p.n_tiles * nkb;                                            // < 2^31 / 132 for every matrix of these models
    const bool ck = p.ck_s != 0;
    const int rank = ck ? (int)q_cluster_rank() : 0, cluster = cta / QG_CK;
    QWalk wk;
    int u0 = 0;
    if (!ck) {
        u0 = (int)q_range_start(cta, U, G);
        const int u1 = (int)q_range_start(cta + 1, U, G);
        wk.n = u1 - u0; wk.tile0 = u0 / nkb; wk.kb0 = u0 - wk.tile0 * nkb; wk.kb_begin = 0; wk.kb_end = nkb; wk.tile_step = 1;
    } else {
        const int n_clusters = G / QG_CK;
        const int rounds = cluster < p.n_tiles ? (p.n_tiles - cluster + n_clusters - 1) / n_clusters : 0;
        wk.kb_begin = rank * nkb / QG_CK; wk.kb_end = (rank + 1) * nkb / QG_CK;
        wk.n = rounds * (wk.kb_end - wk.kb_begin); wk.tile0 = cluster; wk.kb0 = wk.kb_begin; wk.tile_step = n_clusters;
    }
    const int R = p.raw_stages;

    if (warp == 1 && lane == 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tb) : "memory");
    if (warp == 0 && lane == 0) {
        for (int i = 0; i < QG_MAX_RAW_STAGES; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&raw_empty[i], QG_N_UNPACK); }
        mbar_init(&unit_full[0], QG_N_UNPACK + 1);
        mbar_init(&unit_empty[0], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&recv_bar[i], QG_CK);
        fence_mbar_init();
    }
    __syncthreads();
    if (ck) {       // nobody may arrive on a peer's barrier before that peer has initialised it
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    if (threadIdx.x == 0) q_stamp(p, 1);                                      // barriers ready

    // Programmatic dependent launch: everything up to here, the weight stream and the unpacking of the first qtile need nothing
    // from the kernel before -- only the activations (read) and C / the split-tile scratch (written) do.
    pdl_launch_dependents();
    if (warp == 0) {
        if (lane == 0) {
            // ===== weight producer: one 1-D bulk copy per qtile, as far ahead as the raw ring is deep =====
            int tile = wk.tile0, kb = wk.kb0, s = 0, cur = -1;
            uint32_t ph = 0, qb = 0;
            const uint8_t* base = nullptr;
            for (int i = 0; i < wk.n; ++i) {
                if (tile != cur) {                                            // next output tile: its type may differ (Q | K | V)
                    cur = tile;
                    qb = (uint32_t)qg_qtile_bytes(q_tile_type(p, tile));
                    base = p.w + q_tile_off(p, tile);
                }
                mbar_wait(&raw_empty[s], ph ^ 1u);
                mbar_expect_tx(&raw_full[s], qb);
                tma_load_1d(raw_ring + (size_t)s * p.raw_stride, base + (size_t)kb * qb, qb, &raw_full[s]);
                if (i == 0) q_stamp(p, 2);                                    // first weight copy issued
                if (++s == R) { s = 0; ph ^= 1u; }
                wk.advance(tile, kb, 1);
            }
        }
    } else if (warp == 1) {
        if (lane == 0) {
            // ===== activation producer: the four [NB x 64] boxes of a qtile's K range (L2-resident) =====
            int tile = wk.tile0, kb = wk.kb0;
            pdl_wait();                                               // the activations are the output of the kernel before
            q_stamp(p, 8);                                                    // the kernel before has completed
            for (int i = 0; i < wk.n; ++i) {
                mbar_wait(&unit_empty[0], (uint32_t)(i & 1) ^ 1u);
                mbar_expect_tx(&unit_full[0], 4u * Cfg::B_TILE);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) tma_load_2d_q(act_ring + kk * Cfg::B_TILE, &p.tb, kb * QG_COLS + kk * QG_KSTEP, 0, &unit_full[0]);
                wk.advance(tile, kb, 1);
            }
        }
    } else if (warp >= QG_W_UNPACK0 && warp < QG_W_EPI0) {
        // ===== unpack warps: thread (row r, half h) turns 128 columns of its row into two K-steps (2 x 32 registers) and stores
        // them into the A operand: row r of K-step kk at kk * 16 KB + 128 r, 16-byte chunk c at position c ^ (r % 8) (the 128-byte
        // swizzle the MMA's descriptor names; the eight rows of a quarter-warp store to eight different bank groups).
        const int t = (warp - QG_W_UNPACK0) * 32 + lane, r = t & 127, h = t >> 7;
        uint8_t* arow = a_op + (size_t)r * 128;
        auto store = [&](int kk, const uint32_t* w) {
#pragma unroll
            for (int c = 0; c < 8; ++c)
                *reinterpret_cast<uint4*>(arow + kk * (QG_ROWS * QG_KSTEP * 2) + ((c ^ (r & 7)) << 4)) = make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
        };
        int tile = wk.tile0, kb = wk.kb0, s = 0, cur = -1, type = 12;
        uint32_t ph = 0;
        for (int i = 0; i < wk.n; ++i) {
            if (tile != cur) { cur = tile; type = q_tile_type(p, tile); }
            const uint8_t* raw = raw_ring + (size_t)s * p.raw_stride;
            mbar_wait(&raw_full[s], ph);
            if (i == 0 && t == 0) q_stamp(p, 3);                              // first qtile has landed
            uint32_t w[32];
            qg_dequant_kstep(type, raw, r, 2 * h, [&](int c, QgU4 v) { w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w; });
            // the first 32 words sit in registers: only now does the thread need the A operand (the MMAs of the previous qtile
            // are done and its accumulator staging has been read)
            mbar_wait(&unit_empty[0], (uint32_t)(i & 1) ^ 1u);
            store(2 * h, w);
            qg_dequant_kstep(type, raw, r, 2 * h + 1, [&](int c, QgU4 v) { w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w; });
            __syncwarp();
            if (lane == 0) mbar_arrive(&raw_empty[s]);                // this warp has read all it needs of the raw bytes
            store(2 * h + 1, w);
            fence_proxy_async();                                      // generic-proxy stores -> the tensor core's (async-proxy) reads
            __syncwarp();
            if (lane == 0) mbar_arrive(&unit_full[0]);
            if (++s == R) { s = 0; ph ^= 1u; }
            wk.advance(tile, kb, 1);
        }
        if (t == 0) q_stamp(p, 4);                                            // the last qtile is unpacked
    } else if (warp >= QG_W_EPI0) {
        // ===== MMA and epilogue warpgroup =====
        const int q = warp & 3;                                       // rows 32q..32q+31 of the tile in the epilogue
        const int nl = q * 32 + lane;                                 // row inside the tile
        const int et = threadIdx.x - QG_W_EPI0 * 32;
        int seg = 0, tile = wk.tile0, kb = wk.kb0;
        const uint32_t act_u32 = smem_u32(act_ring), a_u32 = smem_u32(a_op);
        // the MMAs of qtiles [i0, i0 + n_kb) (one output tile) into the registers, then the accumulator into the staging rows: after
        // this stg[b * QG_STG_LD + row] = C[b][row] of the CTA's part of the tile; the A operand stays claimed until release()
        auto mma_segment = [&](int i0, int n_kb) {
            float acc[2][NB / 2];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                for (int x = 0; x < NB / 2; ++x) acc[hf][x] = 0.f;
            for (int j = 0; j < n_kb; ++j) {
                const int i = i0 + j;
                mbar_wait(&unit_full[0], (uint32_t)(i & 1));          // A operand (unpack warps) and activation boxes (TMA) are there
                wgmma_fence_acc<NB / 2>(acc[0]);
                wgmma_fence_acc<NB / 2>(acc[1]);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const uint64_t bdesc = wgmma_desc_sw128(act_u32 + (uint32_t)(kk * Cfg::B_TILE));
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        const uint64_t adesc = wgmma_desc_sw128(a_u32 + (uint32_t)(kk * (QG_ROWS * QG_KSTEP * 2) + hf * (64 * QG_KSTEP * 2)));
#pragma unroll
                        for (int k = 0; k < 4; ++k) wgmma_m64k16<NB, false>(acc[hf], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc<NB / 2>(acc[0]);
                wgmma_fence_acc<NB / 2>(acc[1]);
                if (j < n_kb - 1) {
                    named_bar_sync(1, 128);                           // every thread's MMAs of this qtile are complete
                    if (et == 0) mbar_arrive(&unit_empty[0]);
                }
            }
            if (i0 + n_kb >= wk.n && et == 0) q_stamp(p, 9);          // last MMA complete
            named_bar_sync(1, 128);
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                for (int x = 0; x < NB / 8; ++x) {
                    const int row = hf * 64 + q * 16 + (lane >> 2), b = 8 * x + 2 * (lane & 3);
                    stg[b * QG_STG_LD + row] = acc[hf][4 * x];
                    stg[(b + 1) * QG_STG_LD + row] = acc[hf][4 * x + 1];
                    stg[b * QG_STG_LD + row + 8] = acc[hf][4 * x + 2];
                    stg[(b + 1) * QG_STG_LD + row + 8] = acc[hf][4 * x + 3];
                }
            named_bar_sync(1, 128);
        };
        auto staged16 = [&](int c, float* v) {
#pragma unroll
            for (int b = 0; b < 16; ++b) v[b] = stg[(c * 16 + b) * QG_STG_LD + nl];
        };
        auto release = [&]() {                                        // the staging has been read: the A operand may be refilled
            named_bar_sync(1, 128);
            if (et == 0) mbar_arrive(&unit_empty[0]);
        };
        pdl_wait();                                                   // C, the scratch and the tickets may still be in use by the kernel before
        const float* inv = nullptr;
        if (p.ssq_in != nullptr) {
            // folded RMSNorm, consumer side: token b's sum of squares = the parts the GEMM before wrote, added in part order by ONE
            // thread per token (every CTA computes the same 64 numbers; the loads hit L2 and hide behind the first qtiles)
            constexpr int GROUPS = 128 / NB;                          // threads per token: each sums every GROUPS-th part
            const int b = et % NB, g = et / NB;
            float acc = 0.f;
            for (int pt = g; pt < p.ssq_parts; pt += GROUPS * 8) {    // eight loads in flight per thread and round trip
                float t8[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) t8[k] = pt + k * GROUPS < p.ssq_parts ? __ldcg(p.ssq_in + (size_t)(pt + k * GROUPS) * 64 + b) : 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) acc += t8[k];
            }
            float* red = inv_s + 64;                                  // [GROUPS][NB] partial sums
            red[g * NB + b] = acc;
            named_bar_sync(1, 128);
            if (et < NB) {
                float ss = 0.f;
#pragma unroll
                for (int k = 0; k < GROUPS; ++k) ss += red[k * NB + et];
                // the parts hold sums of x^2; the activations carried x * gamma * PRESCALE
                inv_s[et] = rsqrtf(ss / (float)p.n_norm + p.eps) * (1.0f / QGEMM_NORM_PRESCALE);
            }
            named_bar_sync(1, 128);
            inv = inv_s;
        }
        for (int i = 0; i < wk.n; ++seg, tile += wk.tile_step) {
            const int n_kb = min(wk.kb_end - kb, wk.n - i);
            kb = wk.kb_begin;
            const int i0 = i;
            i += n_kb;
            if (ck) {
                // ---- cluster mode: this CTA's accumulator is one K-quarter of the tile.  Warp q holds rows 32q..32q+31 of it: they
                // belong to the slice rank q finishes, so the warp stores them straight into rank q's shared memory (slot = own rank)
                // and counts itself in on rank q's barrier; then the four warps reduce the slice this rank owns (ranks in order:
                // deterministic) and run the epilogue.  One DSMEM hop instead of store -> fence -> signal -> poll -> load through L2.
                constexpr int SLOT = NB * 32;                          // floats of one source rank's slice: [NB columns][32 rows]
                constexpr int CPT = NB / 4;                            // batch columns per thread in the reduction: warp q takes columns q CPT ..
                const int par = seg & 1;
                const int n = tile * QG_ROWS + rank * 32 + lane;       // the output feature this thread finishes
                const bool fold = p.xg_out != nullptr;                 // folded RMSNorm, producer side (this GEMM adds to the residual)
                const float gam = fold && n < p.n ? __ldg(p.gamma_next + n) * QGEMM_NORM_PRESCALE : 0.f;
                float old[CPT];
                if (p.epi == GEMM_EPI_ADD_F32) {                       // the residual's old values: requested before anything is waited for
#pragma unroll
                    for (int b = 0; b < CPT; ++b) old[b] = n < p.n ? __ldcg(reinterpret_cast<const float*>(p.c) + (size_t)(q * CPT + b) * p.ldc + n) : 0.f;
                }
                mma_segment(i0, n_kb);
                if (i >= wk.n && warp == QG_W_EPI0 && lane == 0) q_stamp(p, 6);
                const uint32_t dst = q_mapa(smem_u32(recv + (size_t)(par * QG_CK + rank) * SLOT), (uint32_t)q) + (uint32_t)lane * 4u;
#pragma unroll
                for (int c = 0; c < NB / 16; ++c) {
                    float v[16];
                    staged16(c, v);
#pragma unroll
                    for (int b = 0; b < 16; ++b) q_st_cluster_f32(dst + (uint32_t)((c * 16 + b) * 32 * 4), v[b]);
                }
                release();
                __syncwarp();
                if (lane == 0) q_arrive_cluster(q_mapa(smem_u32(&recv_bar[par]), (uint32_t)q));
                q_wait_cluster(&recv_bar[par], (uint32_t)(seg >> 1) & 1u);
                const float* mine = recv + (size_t)par * QG_CK * SLOT + (size_t)(q * CPT) * 32 + lane;
                float* out = reinterpret_cast<float*>(p.c) + (size_t)(q * CPT) * p.ldc + n;
                const int hcol = (n >> 4) * 8 + (n & 7);               // SiLU*mul: rows are [8 gate | 8 up] groups, lane ^ 8 is the partner
#pragma unroll
                for (int b = 0; b < CPT; ++b) {
                    float v = 0.f;
#pragma unroll
                    for (int src = 0; src < QG_CK; ++src) v += mine[(size_t)src * SLOT + b * 32];
                    if (inv != nullptr) v *= inv[q * CPT + b];
                    if (p.epi == GEMM_EPI_SILU) {
                        const float up = __shfl_xor_sync(0xffffffffu, v, 8);
                        if ((lane & 8) == 0 && n < p.n)
                            reinterpret_cast<__half*>(p.c)[(size_t)(q * CPT + b) * p.ldc + hcol] = __float2half_rn((v / (1.0f + expf(-v))) * up);
                        continue;
                    }
                    const float xn = p.epi == GEMM_EPI_ADD_F32 ? old[b] + v : v;
                    if (n < p.n) out[(size_t)b * p.ldc] = xn;
                    if (fold) {
                        if (n < p.n) p.xg_out[(size_t)(q * CPT + b) * p.ldxg + n] = __float2half_rn(xn * gam);
                        // sum of squares of this slice's 32 rows for token q CPT + b: lanes in a fixed butterfly order
                        float sq = n < p.n ? xn * xn : 0.f;
                        sq += __shfl_xor_sync(0xffffffffu, sq, 16);
                        sq += __shfl_xor_sync(0xffffffffu, sq, 8);
                        sq += __shfl_xor_sync(0xffffffffu, sq, 4);
                        sq += __shfl_xor_sync(0xffffffffu, sq, 2);
                        sq += __shfl_xor_sync(0xffffffffu, sq, 1);
                        if (lane == 0) p.ssq_out[(size_t)(tile * QG_CK + rank) * 64 + q * CPT + b] = sq;
                    }
                }
                continue;
            }
            const int n = tile * QG_ROWS + nl;
            const bool whole = n_kb == nkb;                           // the whole K range of this tile is ours
            // Shared tile.  Its FIRST units are the END of CTA c_first's range, its later units the START of the ranges of
            // c_first + 1 .. c_last: those CTAs store their part to scratch and count themselves in; c_first gets there last (or
            // together with the CTAs whose whole range lies inside the tile), so it is the designated finisher -- it keeps its own
            // part in registers, adds the others' (CTA order: deterministic) and runs the epilogue.  (All CTAs of the grid are
            // resident -- one per SM -- and nobody waits for a lower-numbered CTA, so the wait cannot deadlock.)
            const int t0 = tile * nkb;
            const int c_first = whole ? cta : q_owner_of(t0, U, G), c_last = whole ? cta : q_owner_of(t0 + nkb - 1, U, G);
            const bool finisher = !whole && cta == c_first;
            float* mine = p.partial + (size_t)cta * (NB * QG_ROWS) + nl;
            constexpr bool PRE = NB <= 32;                            // the others' sum fits the registers beside the accumulator chunk
            float ps[PRE ? NB : 1];
            mma_segment(i0, n_kb);
            if (finisher) {
                if (warp == QG_W_EPI0 && lane == 0) {
                    const unsigned need = (unsigned)(c_last - c_first);
                    unsigned got;
                    while (true) {
                        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(got) : "l"(p.counters + tile) : "memory");
                        if (got >= need) break;
                        __nanosleep(32);
                    }
                    p.counters[tile] = 0;                             // ready for the next launch (everybody has counted in)
                }
                named_bar_sync(1, 128);
                if (PRE) {
#pragma unroll
                    for (int b = 0; b < (PRE ? NB : 1); ++b) ps[b] = 0.f;
                    for (int c = c_first + 1; c <= c_last; ++c) {
                        const float* pc = p.partial + (size_t)c * (NB * QG_ROWS) + nl;
                        float tv[PRE ? NB : 1];
#pragma unroll
                        for (int b = 0; b < (PRE ? NB : 1); ++b) tv[b] = __ldcg(pc + b * QG_ROWS);
#pragma unroll
                        for (int b = 0; b < (PRE ? NB : 1); ++b) ps[b] += tv[b];
                    }
                }
            }
            if (i >= wk.n && warp == QG_W_EPI0 && lane == 0) q_stamp(p, 6);   // last accumulator complete
#pragma unroll
            for (int c = 0; c < NB / 16; ++c) {
                float v[16];
                staged16(c, v);
                if (whole) q_epilogue16(p, n, lane, c * 16, v, inv);
                else if (finisher) {
                    if (PRE) {
#pragma unroll
                        for (int b = 0; b < 16; ++b) v[b] += ps[PRE ? c * 16 + b : 0];
                    } else {
                        for (int cc = c_first + 1; cc <= c_last; ++cc) {
                            const float* pc = p.partial + (size_t)cc * (NB * QG_ROWS) + (size_t)(c * 16) * QG_ROWS + nl;
                            float tv[16];
#pragma unroll
                            for (int b = 0; b < 16; ++b) tv[b] = __ldcg(pc + b * QG_ROWS);
#pragma unroll
                            for (int b = 0; b < 16; ++b) v[b] += tv[b];
                        }
                    }
                    q_epilogue16(p, n, lane, c * 16, v, inv);
                } else {
#pragma unroll
                    for (int b = 0; b < 16; ++b) mine[(c * 16 + b) * QG_ROWS] = v[b];
                }
            }
            release();
            if (whole || finisher) continue;
            __threadfence();
            named_bar_sync(1, 128);
            if (warp == QG_W_EPI0 && lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.counters + tile) : "memory");
        }
        if (warp == QG_W_EPI0 && lane == 0) q_stamp(p, 7);                    // epilogue done
    }
}

// ---- load time: native GGUF rows -> QG qtile stream -----------------------------------------------------------------------
struct PackParams {
    QGemmSource src[3];
    int nsrc, mode, nkb, n_rows;
    const uint64_t* tile_off;
    uint8_t* dst;
};
__global__ void __launch_bounds__(128) qgemm_pack_kernel(const PackParams p) {
    const int row = blockIdx.x * 128 + threadIdx.x;       // output row of the GEMM
    const int kb = blockIdx.y;
    if (row >= p.n_rows) return;
    int si = 0, srow = row;
    if (p.mode == 1) {                                     // [8 gate | 8 up] groups
        si = (row & 15) >> 3;
        srow = (row >> 4) * 8 + (row & 7);
    } else {
        while (si < p.nsrc - 1 && srow >= p.src[si].rows) { srow -= p.src[si].rows; ++si; }
    }
    const int type = p.src[si].type;
    const int bb = type == 12 ? 144 : 210;
    const uint8_t* blk = p.src[si].w + ((size_t)srow * p.nkb + kb) * bb;
    const int tile = row >> 7;
    qg_pack_block(type, blk, p.dst + p.tile_off[tile] + (size_t)kb * qg_qtile_bytes(type), row & 127);
}

typedef CUresult (*EncodeTiledFnQ)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFnQ encode_fn_q() {
    static EncodeTiledFnQ fn = []() -> EncodeTiledFnQ {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
        return reinterpret_cast<EncodeTiledFnQ>(f);
    }();
    return fn;
}

// clusters of four CTAs (227 KB of shared memory each) the device can keep resident at once, per kernel variant
template <int NB>
int max_clusters_nb() {
    static const int n = []() {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)(QGEMM_MAX_GRID / QG_CK * QG_CK));
        cfg.blockDim = dim3(QG_THREADS);
        cfg.dynamicSmemBytes = QG_SMEM;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = QG_CK; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        int k = 0;
        if (cudaOccupancyMaxActiveClusters(&k, qgemm_kernel<NB>, &cfg) != cudaSuccess) { cudaGetLastError(); k = 0; }
        return k;
    }();
    return n;
}
// Cluster mode pays where tiles are few and deep.  With many tiles per cluster (gate/up: 7 rounds, lm_head: 31) the rounds
// quantise (7 x 4 qtiles against 24.2 under stream-K) and a 4-qtile segment per tile leaves the accumulator hand-off no slack.  Default: at
// most two rounds (QKV, attn_output, ffn_down of the Llama shapes); GL_QGEMM_CLUSTER_ROUNDS overrides.
int cluster_max_rounds() {
    static const int r = []() { const char* e = getenv("GL_QGEMM_CLUSTER_ROUNDS"); const int v = e ? atoi(e) : 2; return v < 1 ? 1 : v; }();
    return r;
}
bool cluster_mode_enabled() {
    static const bool on = []() { const char* e = getenv("GL_QGEMM_CLUSTER"); return !(e && e[0] == '0'); }();
    return on;
}

template <int NB>
cudaError_t launch_nb(QParams& qp, int grid, int n_sm, cudaStream_t s) {
    // Tile-aligned split-K inside clusters of four.  Under stream-K a tile of QKV / attn_output / ffn_down (32-48 tiles of 16-56
    // K-blocks on 132 SMs) is shared by 4-6 CTAs that all finish at the same moment, and the partial sums cross L2 on the
    // critical path; a cluster exchanges them through distributed shared memory.  Stream-K remains
    // for GEMMs with many tiles per cluster (gate/up, lm_head: cluster_max_rounds()), for matrices with fewer than four K-blocks
    // per row and for GL_QGEMM_CLUSTER=0.
    qp.ck_s = 0;
    if (cluster_mode_enabled() && qp.nkb >= QG_CK) {                     // the same rule as qgemm_uses_cluster()
        const int cap = std::min(max_clusters_nb<NB>(), std::min(n_sm, QGEMM_MAX_GRID) / QG_CK);
        const int n_clusters = std::min(cap, qp.n_tiles);
        if (n_clusters > 0 && qp.n_tiles <= cluster_max_rounds() * n_clusters) {
            // Any number of rounds on two receive buffers: a rank sends round r only after its own wait for round r - 1, which
            // needs every peer's round r - 1 arrival, and a peer arrives for r - 1 only after it has read round r - 2.
            qp.ck_s = QG_CK;
            grid = n_clusters * QG_CK;
        }
    }
    qp.raw_stages = std::min(QG_MAX_RAW_STAGES, (QCfg<NB>::RAW_BUDGET - (qp.ck_s ? QCfg<NB>::CK_BYTES : 0)) / qp.raw_stride);
    if (qp.raw_stages < 2) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(QG_THREADS);
    cfg.dynamicSmemBytes = QG_SMEM;
    cfg.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (batch_pdl_enabled()) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    if (qp.ck_s) {
        at[na].id = cudaLaunchAttributeClusterDimension;
        at[na].val.clusterDim.x = QG_CK; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1;
        ++na;
    }
    cfg.attrs = at;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, qgemm_kernel<NB>, qp);
}

}  // namespace

// ---- GL_QGEMM_TRACE=1: per-launch, per-CTA %globaltimer stamps (profiling aid; tools/qgemm_trace.py reads them back) ----
namespace {
unsigned long long* g_trace = nullptr;
int g_trace_launch = 0;
bool trace_on() {
    static const bool on = []() { const char* e = getenv("GL_QGEMM_TRACE"); return e && e[0] == '1'; }();
    return on;
}
}  // namespace
extern "C" int gl_dbg_qgemm_trace(unsigned long long* out, int max_launches, int reset) {
    const int n = std::min(std::min(g_trace_launch, QG_TRACE_LAUNCHES), max_launches);
    if (out && g_trace && n > 0) cudaMemcpy(out, g_trace, (size_t)n * QGEMM_MAX_GRID * QG_TRACE_SLOTS * 8, cudaMemcpyDeviceToHost);
    const int total = g_trace_launch;
    if (reset) { g_trace_launch = 0; if (g_trace) cudaMemset(g_trace, 0, (size_t)QG_TRACE_LAUNCHES * QGEMM_MAX_GRID * QG_TRACE_SLOTS * 8); }
    return std::min(total, QG_TRACE_LAUNCHES);
}

size_t qgemm_partial_floats(int nb) { return (size_t)QGEMM_MAX_GRID * 2 * nb * QG_ROWS; }
bool qgemm_batch_ok(int nb) { return nb == 16 || nb == 32 || nb == 64; }

cudaError_t qgemm_configure() {
    cudaError_t e = cudaFuncSetAttribute(qgemm_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QG_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(qgemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QG_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(qgemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QG_SMEM);
    return e;
}

cudaError_t qgemm_pack_launch(const QGemmSource* src, int nsrc, int mode, int k, uint8_t* dst, uint64_t* tile_off_host, uint8_t* tile_type_host,
                              cudaStream_t s) {
    if (nsrc < 1 || nsrc > 3 || (mode == 1 && nsrc != 2) || k % QG_COLS) return cudaErrorInvalidValue;
    int n_rows = 0;
    for (int i = 0; i < nsrc; ++i) {
        if (!qg_type_ok(src[i].type) || src[i].rows % (mode == 1 ? 64 : QG_ROWS)) return cudaErrorInvalidValue;
        n_rows += src[i].rows;
    }
    if (mode == 1 && (src[0].rows != src[1].rows || src[0].type != src[1].type)) return cudaErrorInvalidValue;
    const int nkb = k / QG_COLS, n_tiles = n_rows / QG_ROWS;
    uint64_t off = 0;
    for (int t = 0; t < n_tiles; ++t) {
        int type;
        if (mode == 1) type = src[0].type;
        else {
            int row = t * QG_ROWS, si = 0;
            while (si < nsrc - 1 && row >= src[si].rows) { row -= src[si].rows; ++si; }
            type = src[si].type;
        }
        tile_off_host[t] = off;
        tile_type_host[t] = (uint8_t)type;
        off += (uint64_t)nkb * qg_qtile_bytes(type);
    }
    uint64_t* d_off = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_off, (size_t)n_tiles * 8);
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(d_off, tile_off_host, (size_t)n_tiles * 8, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        PackParams pp{};
        for (int i = 0; i < nsrc; ++i) pp.src[i] = src[i];
        pp.nsrc = nsrc; pp.mode = mode; pp.nkb = nkb; pp.n_rows = n_rows; pp.tile_off = d_off; pp.dst = dst;
        qgemm_pack_kernel<<<dim3((unsigned)n_tiles, (unsigned)nkb), 128, 0, s>>>(pp);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFree(d_off);
    return e;
}

bool qgemm_uses_cluster(const QGemmWeights& wt, int nb, int epi, int n_sm) {
    (void)epi;
    if (!cluster_mode_enabled() || wt.nkb < QG_CK) return false;
    const int mc = nb == 16 ? max_clusters_nb<16>() : nb == 32 ? max_clusters_nb<32>() : max_clusters_nb<64>();
    const int cap = std::min(mc, std::min(n_sm, QGEMM_MAX_GRID) / QG_CK);
    const int n_clusters = std::min(cap, wt.n_tiles);
    return n_clusters > 0 && wt.n_tiles <= cluster_max_rounds() * n_clusters;
}

cudaError_t qgemm_launch(const QGemmWeights& wt, const __half* act, int act_rows_alloc, int nb, void* c, int ldc, int epi, float* partial,
                         int n_sm, cudaStream_t s, const QGemmNorm* norm) {
    if (!qgemm_batch_ok(nb) || act_rows_alloc < nb || !wt.w || (wt.k % QG_COLS) || ((uintptr_t)act % 16)) return cudaErrorInvalidValue;
    if (epi != GEMM_EPI_F32 && epi != GEMM_EPI_ADD_F32 && epi != GEMM_EPI_SILU) return cudaErrorInvalidValue;
    EncodeTiledFnQ fn = encode_fn_q();
    if (!fn) return cudaErrorInvalidValue;
    QParams qp{};
    const cuuint64_t dims[2] = {(cuuint64_t)wt.k, (cuuint64_t)act_rows_alloc};
    const cuuint64_t strides[1] = {(cuuint64_t)wt.k * 2};
    const cuuint32_t box[2] = {(cuuint32_t)QG_KSTEP, (cuuint32_t)nb};
    const cuuint32_t estr[2] = {1, 1};
    if (fn(&qp.tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(act), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return cudaErrorInvalidValue;
    qp.w = wt.w; qp.counters = wt.counters; qp.partial = partial;
    // tile addressing: arithmetic when the tiles are "type0, then type1" (every Llama GEMM: uniform, or Q | K | V with another V
    // type); the per-tile tables only for anything else
    qp.type0 = wt.type0; qp.type1 = wt.type1; qp.tile_split = wt.tile_split; qp.off_split = wt.off_split;
    qp.tile_off = wt.two_segment ? nullptr : wt.tile_off;
    qp.tile_type = wt.two_segment ? nullptr : wt.tile_type;
    qp.raw_stride = wt.has_q6k ? QG_Q6K_BYTES + 768 : QG_Q4K_BYTES;      // 27 648 / 18 432: multiples of 1024
    qp.c = c; qp.ldc = ldc; qp.epi = epi; qp.n = wt.n; qp.n_tiles = wt.n_tiles; qp.nkb = wt.nkb;
    if (norm != nullptr) {
        if (norm->xg_out != nullptr && !(epi == GEMM_EPI_ADD_F32 && qgemm_uses_cluster(wt, nb, epi, n_sm) && norm->gamma_next && norm->ssq_out))
            return cudaErrorInvalidValue;                                // the producer side exists in the cluster epilogue only
        qp.gamma_next = norm->gamma_next; qp.xg_out = norm->xg_out; qp.ldxg = norm->ldxg; qp.ssq_out = norm->ssq_out;
        qp.ssq_in = norm->ssq_in; qp.ssq_parts = norm->ssq_parts; qp.n_norm = norm->n_norm; qp.eps = norm->eps;
    }
    const long long U = (long long)wt.n_tiles * wt.nkb;
    const int grid = (int)std::min<long long>(std::min(n_sm, QGEMM_MAX_GRID), U);
    if (trace_on()) {       // NOTE: a captured graph keeps the slot of the capture: trace with plain launches (gl_time_batch_step's warm pass)
        if (!g_trace) {
            if (cudaMalloc((void**)&g_trace, (size_t)QG_TRACE_LAUNCHES * QGEMM_MAX_GRID * QG_TRACE_SLOTS * 8) != cudaSuccess) return cudaErrorMemoryAllocation;
            cudaMemset(g_trace, 0, (size_t)QG_TRACE_LAUNCHES * QGEMM_MAX_GRID * QG_TRACE_SLOTS * 8);
        }
        if (g_trace_launch < QG_TRACE_LAUNCHES) qp.trace = g_trace + (size_t)g_trace_launch * QGEMM_MAX_GRID * QG_TRACE_SLOTS;
        ++g_trace_launch;
    }
    if (nb == 16) return launch_nb<16>(qp, grid, n_sm, s);
    if (nb == 32) return launch_nb<32>(qp, grid, n_sm, s);
    return launch_nb<64>(qp, grid, n_sm, s);
}

}  // namespace gl
