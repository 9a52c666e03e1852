// Decode GEMV: y = dequant(W)[rows x K] * x[K], the kernel that bounds Llama decode on H100.
//
// Replaces the quantised mat-vec that, in the reference, runs inside the Ollama daemon behind
// OllamaService.generateResponse / generateStreamResponse
// (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237).
//
// Design (DESIGN.md section 4.1; building blocks in gemv_core.cuh).  HBM-bound: every weight byte is used
// once per token, so the kernel is a byte-streaming pipeline, not a GEMM.
//   * persistent grid, one CTA per SM; each CTA owns a contiguous, balanced range of the phase's ITEMS
//     (4 rows x K; 2 rows where 4 do not fit a slot), so there is no tail wave and no atomics;
//   * one producer warp (lane w feeds consumer warp w) streams row segments with 1-D TMA bulk copies (cp.async.bulk, SASS UBLKCP) into an
//     mbarrier-guarded FIFO ring of small shared-memory slots (weights are static, so the ring is filled
//     BEFORE griddepcontrol.wait: under programmatic dependent launch the next kernel's weights are
//     already in flight while the previous kernel drains);
//   * NW consumer warps, each owning whole items: dp4a block decode straight out of shared memory against
//     the activation vector held in shared memory as two int8 planes (15-bit fixed point per 32-column
//     block; rowdot.h), fp32 accumulate, warp-shuffle reduction -- no barrier between warps, ever;
//   * fused prologue: RMSNorm + activation snap; fused epilogues: residual add, RoPE + KV-page
//     append, SiLU*mul.
#include "gemv_core.cuh"

namespace gl {

namespace {

// PRO selects the ONE prologue variant a kernel carries (gemv_core.cuh): 0 coalesced float4 loads (any shape), 1 raw staging by
// bulk copy + half-block snap (narrow rows), 2 half-block snap with 256-bit loads (wide rows).  One variant per kernel keeps the
// code small: with all three inlined the latency-bound single-item phases slowed by 20 % (instruction cache, run 51).
template <int ABITS, int NW, int PRO>
__global__ void __launch_bounds__((NW + 1) * 32, 1) gemv_kernel(const __grid_constant__ GemvParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    Ring ring;
    const float* xraw = reinterpret_cast<const float*>(smem + gemv_fixed_smem(p.cols));       // raw x staging (xraw_bytes, may be 0)
    uint64_t* xbar = reinterpret_cast<uint64_t*>(smem + SM_MISC + 16);                          // two mbarriers
    ring.init(smem, smem + gemv_fixed_smem(p.cols) + p.xraw_bytes, p.n_tracks, p.depth, p.slot_bytes);
    ring.init_barriers(tid);
    if (tid == 0) {
        reinterpret_cast<volatile int*>(smem + SM_MISC)[2] = 0;
        mbar_init(&xbar[0], 1);
        mbar_init(&xbar[1], 1);
    }
    if (tid < RING_MAX_SLOTS) fence_mbar_init();
    __syncthreads();
    pdl_launch_dependents();

    // optional device-side timeline (GL_TRACE=1): entry / upstream wait over / planes ready / this warp's items done,
    // for the first and the last CTA of the grid
    unsigned long long* tr = nullptr;
    if (p.trace != nullptr && tid == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) tr = p.trace + (blockIdx.x == 0 ? 0 : 8);
    if (tr) tr[0] = globaltimer_ns();
    if (warp == NW) {
        // producer: weights are static, so streaming starts before the upstream kernel has finished
        // A kernel whose CTAs become resident beside the upstream kernel's (attn_output beside the attention CTAs) must not
        // flood the SM's request queue while those are still on their latency-critical tail: the attention merge took
        // 4.4 us instead of ~1.5 behind 110 KB of early weight prefetch (run 43).  Such a launch lets only a few lanes
        // prefetch early; the others start when the upstream kernel is done.
        if (p.polite_tracks > 0 && lane >= p.polite_tracks) pdl_wait();
        Track trk{0u, 0u};
        gemv_produce(p.pd, ring, trk, lane, blockIdx.x, gridDim.x);
        if (p.epi == EPI_QKV && lane == 31) {
            pdl_wait();                                  // the position belongs to the upstream chain (sampler of the previous step)
            volatile int* box = reinterpret_cast<volatile int*>(smem + SM_MISC);
            const int pos = __ldcg(&p.st->pos);
            box[0] = pos;
            box[1] = __ldcg(p.page_table + pos / KV_PAGE_TOKENS);
            __threadfence_block();
            box[2] = 1;
        }
        return;
    }
    float scale;
    if constexpr (PRO == 2) {
        PrologueStaticHB ps;
        gemv_prologue_static_hb(p, tid, ps);      // RMSNorm weights: static, requested while the upstream kernel drains
        pdl_wait();   // x (and the residual / KV pages we write) belong to the upstream kernel
        if (tr) tr[1] = globaltimer_ns();
        scale = gemv_prologue_hb256<ABITS, NW>(p, smem, tid, ps, tr);
    } else if constexpr (PRO == 1) {
        PrologueStaticHB ps;
        gemv_prologue_static_hb(p, tid, ps);
        pdl_wait();
        if (tr) tr[1] = globaltimer_ns();
        scale = gemv_prologue_tma<ABITS, NW>(p, smem, xraw, xbar, tid, ps, tr);
    } else {
        PrologueStatic ps;
        gemv_prologue_static<NW>(p, tid, ps);
        pdl_wait();
        if (tr) tr[1] = globaltimer_ns();
        scale = gemv_prologue<ABITS, NW>(p, smem, tid, ps, tr);
    }
    // the QKV epilogue needs (position, physical KV page): two dependent loads, fetched by an idle lane of the producer
    // warp and handed over through shared memory, so that no consumer warp ever stalls on them
    EpiCtx ec{0, 0};
    if (p.epi == EPI_QKV) {
        volatile int* box = reinterpret_cast<volatile int*>(smem + SM_MISC);
        while (box[2] == 0) { }
        ec.pos = box[0];
        ec.page = box[1];
    }
    if (tr) tr[2] = globaltimer_ns();
    Track trk{0u, 0u};
    gemv_consume<ABITS>(p, ring, trk, smem, tid, scale, ec, blockIdx.x, gridDim.x);
    if (tr) tr[3] = globaltimer_ns();
}

}  // namespace

size_t gemv_smem_bytes(int cols, int n_slots, int slot_bytes) {
    return (size_t)gemv_fixed_smem(cols) + (size_t)n_slots * slot_bytes;
}

bool gemv_plan(GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, int slot_bytes) {
    if (nmat < 1 || nmat > 3 || cols <= 0 || cols > 32768 || (cols & 255)) return false;
    if (slot_bytes <= 0 || (slot_bytes & 127)) return false;
    const KSplit ks = ksplit(cols);
    if (!ks.nks) return false;
    ProdDesc d{};
    d.nseg = (unsigned char)nmat;
    d.pair = pair ? 1 : 0;
    d.nks = (unsigned char)ks.nks;
    d.seg_nb = (unsigned char)ks.seg_nb;
    for (int s = 0; s < nmat; ++s) {
        const GemvMat& m = mats[s];
        if (m.type != T_Q4_K && m.type != T_Q6_K && m.type != T_Q8_0) return false;
        if (m.rows <= 0 || ((uintptr_t)m.w & 15)) return false;
        const int sb = kseg_bytes(m.type, ks.seg_nb);
        // Q4_K items are 4 rows; the wider formats take 2 (item_rows(), rowdot.h)
        const int rpi = item_rows(m.type);
        if (rpi * sb > slot_bytes) return false;
        // with more than one K-segment the matrix must have been stored with this item's rows as its tile
        if (ks.nks > 1 && m.tile_rows != (pair ? rpi / 2 : rpi)) return false;
        d.seg[s].w = m.w;
        d.seg[s].rows = m.rows;
        const int rows_per_item = pair ? rpi / 2 : rpi;
        d.seg[s].n_items = (m.rows + rows_per_item - 1) / rows_per_item;
        d.seg_bytes[s] = (unsigned short)sb;
        d.rpi[s] = (unsigned char)rpi;
        d.type[s] = (unsigned char)m.type;
    }
    if (pair && (nmat != 2 || mats[0].type != mats[1].type || mats[0].rows != mats[1].rows)) return false;
    p.pd = d;
    p.cols = cols;
    return true;
}

int gemv_geometry(GemvParams& p, const GemvMat* mats, int nmat, bool pair, int cols, const GemvGeomOpts& o, int n_ctas) {
    // slot size: what the widest item of this kernel needs (Q4_K: 4 row segments, Q6_K / Q8_0: 2), ring depth: whatever
    // shared memory is left, capped so that the bytes in flight stay near what the HBM pipe needs
    const KSplit ks = ksplit(cols);
    if (!ks.nks || nmat < 1 || nmat > 3) return GEMV_GEOM_SHAPE;
    int need = 0;
    for (int i = 0; i < nmat; ++i) need = std::max(need, item_rows(mats[i].type) * kseg_bytes(mats[i].type, ks.seg_nb));
    p.slot_bytes = (need + 127) & ~127;
    if (!gemv_plan(p, mats, nmat, pair, cols, p.slot_bytes)) return GEMV_GEOM_SHAPE;
    // prologue variant (= which kernel): by default the 256-bit-load half-block prologue for every width, so that all GEMV
    // launches of a step are one kernel; xraw stages narrow rows raw by one bulk copy instead (16 KB of ring)
    const int nw = o.nw;
    p.xraw_bytes = 0;
    p.xraw_nseg = 1;
    const bool variants = gemv_prologue_variants(nw);
    p.hb256 = (variants && o.hb256 && (cols > GEMV_XRAW_MAX_COLS || !o.xraw) && cols <= 16 * nw * 32 * (nw >= 12 ? 3 : 4)) ? 1 : 0;
    if (variants && o.xraw && !p.hb256) {
        if (cols <= GEMV_XRAW_MAX_COLS && cols / 16 <= nw * 32) {
            p.xraw_bytes = cols * 4;
        } else if (o.xraw_wide && ks.nks > 1 && cols / ks.nks / 16 <= nw * 32) {     // wide rows: K-segment pieces, two buffers
            p.xraw_nseg = ks.nks;
            p.xraw_bytes = 2 * (cols / ks.nks) * 4;
        }
    }
    const size_t fixed = gemv_smem_bytes(cols, 0, 0) + (size_t)p.xraw_bytes;
    const int ns = std::min(RING_MAX_SLOTS, (int)(((size_t)o.smem_kb * 1024 - fixed) / p.slot_bytes));
    // as many consumer warps as there are, each with >= 2 slots; spare slots deepen the tracks (small slots: more bytes in flight)
    // tracks x depth: as many bytes in flight as the ring can hold, giving up at most two consumer warps for depth
    // (small slots -- Q6_K pairs -- would otherwise leave a third of the shared memory unused: lm_head 0.94 -> 0.86 of peak)
    p.n_tracks = std::min(nw, ns / 2);
    p.depth = p.n_tracks > 0 ? std::min(o.ring_depth_max, ns / p.n_tracks) : 0;
    for (int t = std::max(1, nw - 2); p.pd.nks > 1 && t < std::min(nw, ns / 2); ++t) {      // (narrow rows keep every warp: lm_head is issue-bound at 10)
        const int dd = std::min(o.ring_depth_max, ns / t);
        if (dd >= 2 && t * dd > p.n_tracks * p.depth) { p.n_tracks = t; p.depth = dd; }
    }
    // a phase in which no warp gets a second slot (one round of items, one K-segment) needs one slot per warp: the smaller
    // footprint (121 KB instead of 232 KB) lets the next kernel's CTAs become resident -- and start their own prefetch --
    // while this one is still running (programmatic dependent launch)
    if (o.lean_rings && p.n_tracks > 0 && p.pd.nks == 1) {
        int items = 0;
        for (int i = 0; i < (pair ? 1 : nmat); ++i) items += p.pd.seg[i].n_items;
        if ((items + n_ctas - 1) / n_ctas <= p.n_tracks) p.depth = 1;
    }
    return p.n_tracks < 1 ? GEMV_GEOM_SMEM : GEMV_GEOM_OK;
}

bool gemv_variant_ok(int abits, int nw) { return (abits == 16 || abits == 8) && (nw == 8 || nw == 12 || nw == 16); }

namespace {
template <int ABITS, int NW, int PRO>
cudaError_t configure_one() {
    return cudaFuncSetAttribute(gemv_kernel<ABITS, NW, PRO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
}
template <int ABITS, int NW, int PRO>
cudaError_t launch_one(const cudaLaunchConfig_t& cfg, const GemvParams& p) {
    return cudaLaunchKernelEx(&cfg, gemv_kernel<ABITS, NW, PRO>, p);
}
template <int ABITS>
cudaError_t configure_abits() {
    cudaError_t e = configure_one<ABITS, 8, 0>();
    if (e == cudaSuccess) e = configure_one<ABITS, 16, 0>();
    if (e == cudaSuccess) e = configure_one<ABITS, 12, 0>();
    if (e == cudaSuccess) e = configure_one<ABITS, 12, 1>();
    if (e == cudaSuccess) e = configure_one<ABITS, 12, 2>();
    return e;
}
template <int ABITS>
cudaError_t launch_abits(const cudaLaunchConfig_t& cfg, const GemvParams& p, int nw, int pro) {
    if (nw == 8) return launch_one<ABITS, 8, 0>(cfg, p);
    if (nw == 16) return launch_one<ABITS, 16, 0>(cfg, p);
    if (pro == 2) return launch_one<ABITS, 12, 2>(cfg, p);
    if (pro == 1) return launch_one<ABITS, 12, 1>(cfg, p);
    return launch_one<ABITS, 12, 0>(cfg, p);
}
}  // namespace

// the specialised prologues are compiled for 12 consumer warps only
bool gemv_prologue_variants(int consumer_warps) { return consumer_warps == 12; }

cudaError_t gemv_configure() {
    cudaError_t e = configure_abits<16>();
    if (e == cudaSuccess) e = configure_abits<8>();
    return e;
}

cudaError_t gemv_launch(const GemvParams& p, int abits, int nw, int n_ctas, bool pdl, cudaStream_t s) {
    if (!gemv_variant_ok(abits, nw) || p.n_tracks < 1 || p.n_tracks > nw || p.depth < 1 || p.n_tracks * p.depth > RING_MAX_SLOTS) return cudaErrorInvalidValue;
    if (p.hb256 && (p.xraw_bytes != 0 || p.cols > 16 * nw * 32 * (nw >= 12 ? 3 : 4) || ((uintptr_t)p.x & 31))) return cudaErrorInvalidValue;
    if (p.xraw_bytes != 0) {
        const int ns = p.xraw_nseg;
        if (ns < 1 || p.cols % (ns * 16) || p.cols / ns / 16 > nw * 32 || ((uintptr_t)p.x & 15) || ((p.cols / ns * 4) & 15) ||
            p.xraw_bytes != (ns == 1 ? 1 : 2) * (p.cols / ns) * 4)
            return cudaErrorInvalidValue;
    }
    if (p.epi == EPI_QKV && ((p.pd.seg[0].rows & 1) || (p.pd.nseg > 1 && (p.pd.seg[1].rows & 1)))) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)n_ctas);
    cfg.blockDim = dim3((unsigned)gemv_threads(nw));
    cfg.dynamicSmemBytes = gemv_smem_bytes(p.cols, p.n_tracks * p.depth, p.slot_bytes) + (size_t)p.xraw_bytes;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    const int pro = p.hb256 ? 2 : (p.xraw_bytes > 0 ? 1 : 0);
    if (pro != 0 && !gemv_prologue_variants(nw)) return cudaErrorInvalidValue;
    return abits == 16 ? launch_abits<16>(cfg, p, nw, pro) : launch_abits<8>(cfg, p, nw, pro);
}

// ------------------------------------------------------------------------------------------------
// fp-weight GEMV (F32 / F16 / BF16): warp per row, 16-B loads, fp32 FMA.  Not the headline path.
// ------------------------------------------------------------------------------------------------
namespace {
template <int TYPE>
__global__ void __launch_bounds__(256) gemv_fp_kernel(const uint8_t* __restrict__ w, int rows, int cols,
                                                      const float* __restrict__ x, float* __restrict__ y) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int r = warp; r < rows; r += nwarps) {
        float acc = 0.f;
        if (TYPE == T_F32) {
            const float* wr = reinterpret_cast<const float*>(w) + (size_t)r * cols;
            for (int c = lane * 4; c < cols; c += 128) {
                const float4 a = *reinterpret_cast<const float4*>(wr + c);
                const float4 b = *reinterpret_cast<const float4*>(x + c);
                acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
            }
        } else {
            const uint16_t* wr = reinterpret_cast<const uint16_t*>(w) + (size_t)r * cols;
            for (int c = lane * 8; c < cols; c += 256) {
                const uint4 a = *reinterpret_cast<const uint4*>(wr + c);
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float f0, f1;
                    if (TYPE == T_F16) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&aw[q]));
                        f0 = f.x; f1 = f.y;
                    } else {
                        f0 = __uint_as_float(aw[q] << 16);
                        f1 = __uint_as_float(aw[q] & 0xFFFF0000u);
                    }
                    acc += f0 * x[c + 2 * q] + f1 * x[c + 2 * q + 1];
                }
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) y[r] = acc;
    }
}
}  // namespace

cudaError_t gemv_fp_launch(const void* w, int type, int rows, int cols, const float* x, float* y, cudaStream_t s) {
    if (cols % 8) return cudaErrorInvalidValue;
    const int blocks = min((rows + 7) / 8, 132 * 8);
    const uint8_t* wb = static_cast<const uint8_t*>(w);
    switch (type) {
        case T_F32: gemv_fp_kernel<T_F32><<<blocks, 256, 0, s>>>(wb, rows, cols, x, y); break;
        case T_F16: gemv_fp_kernel<T_F16><<<blocks, 256, 0, s>>>(wb, rows, cols, x, y); break;
        case T_BF16: gemv_fp_kernel<T_BF16><<<blocks, 256, 0, s>>>(wb, rows, cols, x, y); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace gl
