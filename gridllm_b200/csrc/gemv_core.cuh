// Device-side building blocks of the weight-streaming GEMV, shared by the stand-alone kernel
// (gemv.cu) and the persistent decode-step kernel (decode_mega.cu).
//
//   producer warp : gemv_produce()  -- 1-D TMA bulk copies of row segments into an mbarrier ring of small
//                                      slots; lane w feeds the track of consumer warp w
//   consumer warps: gemv_prologue() -- (RMSNorm) + snap x to int8 planes in shared memory
//                   gemv_consume()  -- every warp owns whole ITEMS (4 rows, or 2 where 4 do not fit a slot):
//                                      dp4a block decode of the item's slots, warp-shuffle reduction, fused
//                                      epilogue (store / residual add / RoPE+KV append / SiLU*mul)
//
// Work decomposition (rowdot.h vocabulary).  The rows of a phase are cut into items; a CTA owns a contiguous,
// balanced range of the flat item list; inside the CTA items are dealt round-robin to the consumer warps, so
// no two warps ever share a row and there is NO barrier of any kind between the prologue and the end of the phase.
// One ring slot = the R row-segments of one (item, K-segment).
//
// Ring discipline: TRACKS.  The ring is n_tracks x depth slots; consumer warp w owns track w (slots w*depth ..
// w*depth+depth-1) and walks it cyclically, and producer lane w feeds exactly that track.  Every mbarrier therefore
// has ONE waiter on each side, each of which completed the previous phase itself before it waits for the next --
// the only situation in which a parity wait cannot alias.  (A shared FIFO of arbitrary depth looks attractive -- 19
// slots for 12 warps -- but a warp can then wait two uses ahead of a slot another warp has not finished, and
// try_wait.parity answers for the wrong phase; found on the GPU in run 20b.)  Warps beyond n_tracks idle in GEMV
// phases; rounds are n_tracks items wide.
//
// Why small slots: the bytes a SM keeps in flight are what the HBM pipe needs (~48-64 KB per SM at 6.5 TB/s x ~1 us),
// and nothing more -- every extra prefetched byte sits in the SM's request FIFO in front of the latency-critical
// loads of a phase change (barrier flag, x), which is what a timeline of the persistent kernel measured
// (prologue 3.2 us at 72 KB in flight, 4.5 us at 144-180 KB).
#pragma once
#include "common.cuh"
#include "gguf_file.h"
#include "kernels.h"
#include "rowdot.h"

namespace gl {

// shared-memory carve-up (bytes from the start of dynamic smem)
constexpr int SM_BARS = 0;                 // full[36], empty[36] mbarriers (576 B)
constexpr int SM_RED = 576;                // 32 floats: RMSNorm partials
constexpr int SM_MISC = 704;               // 64 B scratch (flags)
constexpr int SM_X = 768;                  // x planes start

__host__ __device__ inline int gemv_x_bytes(int cols) { return 2 * cols + cols / 2; }   // hi, lo, sx, sm, s16
__host__ __device__ inline int gemv_fixed_smem(int cols) { return (SM_X + gemv_x_bytes(cols) + 127) & ~127; }

struct Ring {
    uint64_t* full;
    uint64_t* empty;
    uint8_t* slots;
    unsigned n_tracks;      // consumer warps that take items (<= NW)
    unsigned depth;         // slots per track (>= 2)
    unsigned slot_bytes;
    __device__ __forceinline__ void init(uint8_t* smem, uint8_t* slot_base, int tracks, int d, int bytes) {
        full = reinterpret_cast<uint64_t*>(smem + SM_BARS);
        empty = full + RING_MAX_SLOTS;
        slots = slot_base;
        n_tracks = (unsigned)tracks;
        depth = (unsigned)d;
        slot_bytes = (unsigned)bytes;
    }
    // threads 0 .. n_slots-1 of the CTA, one slot each (followed by fence_mbar_init + a CTA barrier in the caller)
    __device__ __forceinline__ void init_barriers(int tid) const {
        if ((unsigned)tid < n_tracks * depth) {
            mbar_init(&full[tid], 1);
            mbar_init(&empty[tid], 1);
        }
    }
};

// Where a warp (or the producer lane that feeds it) stands in its track.
struct Track {
    unsigned d;      // slot inside the track
    unsigned par;    // phase bit of that slot's next use
    __device__ __forceinline__ void advance(unsigned depth) {
        if (++d == depth) { d = 0; par ^= 1u; }
    }
};

struct WorkRange { int a, b; };
__device__ __forceinline__ WorkRange cta_range(int n, int cta, int n_ctas) {
    WorkRange r;
    r.a = (int)(((long long)cta * n) / n_ctas);
    r.b = (int)(((long long)(cta + 1) * n) / n_ctas);
    return r;
}

__device__ __forceinline__ int total_items(const ProdDesc& d) {
    int t = d.seg[0].n_items;
    if (!d.pair) {
        if (d.nseg > 1) t += d.seg[1].n_items;
        if (d.nseg > 2) t += d.seg[2].n_items;
    }
    return t;
}

// flat item index -> (weight segment, item inside it)
__device__ __forceinline__ void item_of(const ProdDesc& d, int flat, int& s, int& it) {
    s = 0;
    it = flat;
    if (!d.pair) {
        if (d.nseg > 1 && it >= d.seg[0].n_items) {
            it -= d.seg[0].n_items;
            s = 1;
            if (d.nseg > 2 && it >= d.seg[1].n_items) {
                it -= d.seg[1].n_items;
                s = 2;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// producer (one WARP): stream this CTA's slots of one phase.  Lane w feeds track w (= consumer warp w): its item of
// every round, K-segment by K-segment, each slot as soon as that track's next slot is free.  tr is the lane's
// position in its track (continues across the phases of the persistent kernel).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void gemv_produce(const ProdDesc& d, const Ring& ring, Track& tr, int lane, int cta, int n_ctas) {
    const WorkRange wr = cta_range(total_items(d), cta, n_ctas);
    const int nks = d.nks;
    const int A = (int)ring.n_tracks;
    if (lane >= A) return;
    for (int i0 = wr.a + lane; i0 < wr.b; i0 += A) {
        // this lane's item.  A matrix is stored [tile][K-segment][row in tile][segment] (rowdot.h) with the item's rows as
        // the tile, so the rows of one (item, K-segment) are ONE contiguous range: one bulk copy per matrix per slot.
        int s, it;
        item_of(d, i0, s, it);
        const uint32_t sb = d.seg_bytes[s];
        const int rpi = d.rpi[s];
        const int tile = d.pair ? (rpi >> 1) : rpi;               // rows of this matrix per item
        const int n = min(tile, d.seg[s].rows - it * tile);        // ragged last item
        const size_t tile_bytes = (size_t)tile * nks * sb;
        const uint8_t* w0 = d.seg[s].w + (size_t)it * tile_bytes;
        const uint8_t* w1 = d.pair ? d.seg[1].w + (size_t)it * tile_bytes : nullptr;
        const uint32_t bytes = (uint32_t)n * sb;
        for (int ks = 0; ks < nks; ++ks) {
            const unsigned pos = (unsigned)lane * ring.depth + tr.d;
            mbar_wait(&ring.empty[pos], tr.par ^ 1u);
            uint8_t* dst = ring.slots + (size_t)pos * ring.slot_bytes;
            uint64_t* bar = &ring.full[pos];
            const size_t ko = (size_t)ks * tile * sb;
            if (d.pair) {
                mbar_expect_tx(bar, 2u * bytes);
                tma_load_1d(dst, w0 + ko, bytes, bar);
                tma_load_1d(dst + tile * sb, w1 + ko, bytes, bar);
            } else {
                mbar_expect_tx(bar, bytes);
                tma_load_1d(dst, w0 + ko, bytes, bar);
            }
            tr.advance(ring.depth);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// consumer prologue: x -> (RMSNorm) -> int8 planes in smem.  All NW*32 consumer threads call it (named barrier 1).
// ---------------------------------------------------------------------------------------------------
// Returns the scalar every row sum of this phase must be multiplied by: 1, or the RMSNorm factor
// rstd = 1/sqrt(mean(x^2)+eps).  The fixed-point integers v = rint(x*w / amax_blk(x*w) * RANGE) do not depend on
// rstd (it cancels), so the planes are built from x*w while the sum of squares is still being reduced, and rstd is
// applied once per output row.  One named barrier in total.
constexpr int PROLOGUE_NB = 5;            // float4 loads in flight per thread (one L2 round trip per batch)

// The static half of the prologue: the RMSNorm weights of this thread's first batch.  They do not depend on the
// upstream kernel / phase, so the caller requests them BEFORE it waits for it (griddepcontrol.wait, grid barrier).
struct PrologueStatic { float4 wv[PROLOGUE_NB]; };
template <int NW>
__device__ __forceinline__ void gemv_prologue_static(const GemvParams& p, int tid, PrologueStatic& ps) {
    constexpr int NT = NW * 32;
    if (p.norm_w == nullptr) return;
    const int nf = p.cols / 4;
    const float4* w4 = reinterpret_cast<const float4*>(p.norm_w);
#pragma unroll
    for (int i = 0; i < PROLOGUE_NB; ++i) {
        const int f = tid + i * NT;
        if (f < nf) ps.wv[i] = __ldg(w4 + f);
    }
}

template <int ABITS, int NW, int NB>
__device__ __forceinline__ float gemv_prologue_nb(const GemvParams& p, uint8_t* smem, int tid, const PrologueStatic& ps, unsigned long long* tr) {
    constexpr int NT = NW * 32;
    const int K = p.cols;
    const int warp = tid >> 5, lane = tid & 31;
    float* red = reinterpret_cast<float*>(smem + SM_RED);
    uint8_t* xhi = smem + SM_X;
    uint8_t* xlo = xhi + K;
    float* sx_arr = reinterpret_cast<float*>(xlo + K);
    float* sm_arr = sx_arr + K / 32;
    int* s16_arr = reinterpret_cast<int*>(sm_arr + K / 32);

    // Thread t owns float4 #(t + i*NT): a warp instruction covers 512 contiguous bytes (= four 32-column blocks, one
    // 128-column unit), eight lanes share a block.  Every read of data produced upstream uses ld.global.cg: this CTA
    // may have been resident (and its SM's L1 populated) before the producer of x finished.
    const int nf = K / 4;                  // K % 256 == 0, so liveness below is uniform over a warp
    const bool norm = p.norm_w != nullptr;
    const float4* x4 = reinterpret_cast<const float4*>(p.x);
    const float4* w4 = reinterpret_cast<const float4*>(p.norm_w);
    float ss = 0.f;
    for (int f0 = tid; f0 < nf; f0 += NB * NT) {
        float4 v[NB], wv[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            const int f = f0 + i * NT;
            if (f < nf) v[i] = __ldcg(x4 + f);
        }
        if (norm) {
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                const int f = f0 + i * NT;
                if (f0 == tid && i < PROLOGUE_NB) wv[i] = ps.wv[i < PROLOGUE_NB ? i : 0];      // first batch: requested before the upstream wait
                else if (f < nf) wv[i] = __ldg(w4 + f);
            }
        }
        if (tr && f0 == tid) {      // (profiling) the first batch's x has arrived when its first value can be consumed
            if (__float_as_uint(v[0].x) != 0x7fc12345u) tr[4] = globaltimer_ns();
        }
        if constexpr (NB > PROLOGUE_NB) {
            // WIDE rows (every iteration of the batch is live): the batch is processed phase by phase across its NB float4s, not float4 by float4: the two shuffle butterflies
            // (block amax, block sums) are 3 dependent shuffles each, and interleaving NB independent chains is what hides their
            // latency (the float4-at-a-time loop spent 1.0 us on K = 4096 and 3.0 us on K = 14336, run 34).  Validity of an
            // iteration is uniform over the warp (nf is a multiple of 32), so the shuffles of invalid iterations are harmless.
            float e[NB][4], amax[NB];
            uint32_t hw[NB], lw[NB];
            int vs[NB], vs32[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                const bool ok = f0 + i * NT < nf;
                e[i][0] = ok ? v[i].x : 0.f; e[i][1] = ok ? v[i].y : 0.f; e[i][2] = ok ? v[i].z : 0.f; e[i][3] = ok ? v[i].w : 0.f;
                if (norm && ok) {
                    ss += e[i][0] * e[i][0] + e[i][1] * e[i][1] + e[i][2] * e[i][2] + e[i][3] * e[i][3];
                    e[i][0] *= wv[i].x; e[i][1] *= wv[i].y; e[i][2] *= wv[i].z; e[i][3] *= wv[i].w;
                }
                amax[i] = fmaxf(fmaxf(fabsf(e[i][0]), fabsf(e[i][1])), fmaxf(fabsf(e[i][2]), fabsf(e[i][3])));
            }
#pragma unroll
            for (int w = 1; w <= 4; w <<= 1) {
#pragma unroll
                for (int i = 0; i < NB; ++i) amax[i] = fmaxf(amax[i], __shfl_xor_sync(0xffffffffu, amax[i], w));
            }
#pragma unroll
            for (int i = 0; i < NB; ++i) snap4<ABITS>(e[i], snap_inv<ABITS>(amax[i]), &hw[i], &lw[i], &vs[i]);
#pragma unroll
            for (int w = 1; w <= 2; w <<= 1) {
#pragma unroll
                for (int i = 0; i < NB; ++i) vs[i] += __shfl_xor_sync(0xffffffffu, vs[i], w);           // sum(v) of the 16-column group
            }
#pragma unroll
            for (int i = 0; i < NB; ++i) vs32[i] = vs[i] + __shfl_xor_sync(0xffffffffu, vs[i], 4);
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                const int f = f0 + i * NT;
                if (f < nf) {
                    // float4 f covers columns 4f..4f+3: unit f>>5, 16-B chunk (f>>2)&7 of the unit, word f&3 of the chunk
                    const int u = f >> 5;
                    const int off = (u << 7) + (((((f >> 2) & 7) ^ (u & 7))) << 4) + ((f & 3) << 2);
                    *reinterpret_cast<uint32_t*>(xhi + off) = hw[i];
                    if (ABITS == 16) *reinterpret_cast<uint32_t*>(xlo + off) = lw[i];
                    if ((f & 3) == 0) s16_arr[f >> 2] = vs[i];
                    if ((f & 7) == 0) {
                        const float sx = amax[i] / (ABITS == 16 ? ACT16_RANGE : ACT8_RANGE);
                        sx_arr[f >> 3] = sx;
                        sm_arr[f >> 3] = sx * (float)vs32[i];
                    }
                }
            }
            } else {
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                const int f = f0 + i * NT;
                if (f < nf) {
                    float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
                    if (norm) {
                        ss += e[0] * e[0] + e[1] * e[1] + e[2] * e[2] + e[3] * e[3];
                        e[0] *= wv[i].x; e[1] *= wv[i].y; e[2] *= wv[i].z; e[3] *= wv[i].w;
                    }
                    float amax = fmaxf(fmaxf(fabsf(e[0]), fabsf(e[1])), fmaxf(fabsf(e[2]), fabsf(e[3])));
                    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
                    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
                    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
                    uint32_t h, l;
                    int vs;
                    snap4<ABITS>(e, snap_inv<ABITS>(amax), &h, &l, &vs);
                    vs += __shfl_xor_sync(0xffffffffu, vs, 1);
                    vs += __shfl_xor_sync(0xffffffffu, vs, 2);           // sum(v) of this 16-column group
                    const int vs32 = vs + __shfl_xor_sync(0xffffffffu, vs, 4);
                    // float4 f covers columns 4f..4f+3: unit f>>5, 16-B chunk (f>>2)&7 of the unit, word f&3 of the chunk
                    const int u = f >> 5;
                    const int off = (u << 7) + (((((f >> 2) & 7) ^ (u & 7))) << 4) + ((f & 3) << 2);
                    *reinterpret_cast<uint32_t*>(xhi + off) = h;
                    if (ABITS == 16) *reinterpret_cast<uint32_t*>(xlo + off) = l;
                    if ((f & 3) == 0) s16_arr[f >> 2] = vs;
                    if ((f & 7) == 0) {
                        const float sx = amax / (ABITS == 16 ? ACT16_RANGE : ACT8_RANGE);
                        sx_arr[f >> 3] = sx;
                        sm_arr[f >> 3] = sx * (float)vs32;
                    }
                }
            }
        }
    }
    if (tr) tr[5] = globaltimer_ns();
    if (norm) {
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
    }
    named_bar_sync(1, NT);
    float scale = 1.f;
    if (norm) {
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) tot += red[w];
        scale = 1.0f / sqrtf(tot / (float)K + p.eps);
    }
    // NOTE: the planes (and red[]) are rewritten only by the NEXT prologue, which every caller separates from this
    // point by a CTA-wide barrier (end of kernel, or the grid barrier of the persistent kernel).
    return scale;
}

// ---------------------------------------------------------------------------------------------------
// Prologue for K <= GEMV_XRAW_MAX_COLS in the stand-alone kernel: x is brought in by ONE bulk copy (TMA) into a raw fp32
// staging buffer, then one thread per HALF BLOCK (16 columns) snaps it out of shared memory; lanes 2k / 2k+1 share a
// 32-column block, so one shuffle gives the block amax and one the block sum.
//   * the float4-per-lane version above needs six shuffles per float4 and recomputes the reciprocal, the addresses and
//     the stores every 4 columns: 21 instructions per column, 1.0 us of arithmetic per K = 4096 prologue (run 45);
//   * reading x with 64-B-per-lane global loads instead (no staging) cut the arithmetic to 0.33 us but multiplied the
//     load requests by eight, and those queue behind the ring's bulk prefetch in the SM's request FIFO: x arrived after
//     3.2 us instead of 0.6 (run 46).  One bulk copy is one request.
// ps carries this thread's RMSNorm weights (its half block), requested before the upstream wait.
// ---------------------------------------------------------------------------------------------------
struct PrologueStaticHB { float4 wv[4]; };
__device__ __forceinline__ void gemv_prologue_static_hb(const GemvParams& p, int tid, PrologueStaticHB& ps) {
    if (p.norm_w == nullptr || tid >= p.cols / 16) return;
    const float4* w4 = reinterpret_cast<const float4*>(p.norm_w) + 4 * tid;
#pragma unroll
    for (int i = 0; i < 4; ++i) ps.wv[i] = __ldg(w4 + i);
}

// ---------------------------------------------------------------------------------------------------
// Prologue, half block per thread straight from global memory: a lane's 16 columns are two whole 32-byte sectors, each read
// with two back-to-back 128-bit loads (Hopper has no 256-bit global load), while the arithmetic keeps the half-block form: one
// shuffle for the block maximum, one for the block sum, reciprocal / addresses / stores once per 16 columns.  Serves every
// width: K = 14336 is 896 half blocks = 2.3 per thread, all of them requested at once.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldcg256(const float* p, float* v) {
    asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p) : "memory");
    asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4 + 16];" : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]) : "l"(p) : "memory");
}

template <int ABITS, int NW>
__device__ __forceinline__ float gemv_prologue_hb256(const GemvParams& p, uint8_t* smem, int tid, const PrologueStaticHB& ps, unsigned long long* tr) {
    constexpr int NT = NW * 32;
    constexpr int MAXR = NW >= 12 ? 3 : 4;          // rounds of half blocks per thread: K <= 16 * NT * MAXR (checked by the host)
    const int K = p.cols;
    const int warp = tid >> 5, lane = tid & 31;
    float* red = reinterpret_cast<float*>(smem + SM_RED);
    uint8_t* xhi = smem + SM_X;
    uint8_t* xlo = xhi + K;
    float* sx_arr = reinterpret_cast<float*>(xlo + K);
    float* sm_arr = sx_arr + K / 32;
    int* s16_arr = reinterpret_cast<int*>(sm_arr + K / 32);
    const int nhb = K / 16;                 // a multiple of 16: a warp whose lower half is live runs with all its lanes
    const bool norm = p.norm_w != nullptr;
    float e[MAXR][16];
#pragma unroll
    for (int r = 0; r < MAXR; ++r) {
        const int hb = tid + r * NT;
        if (hb < nhb) {
            ldcg256(p.x + 16 * (size_t)hb, e[r]);
            ldcg256(p.x + 16 * (size_t)hb + 8, e[r] + 8);
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) e[r][i] = 0.f;
        }
    }
    float ss = 0.f;
#pragma unroll
    for (int r = 0; r < MAXR; ++r) {
        const int hb = tid + r * NT;
        if ((hb & ~31) < nhb) {             // uniform over the warp
            const bool ok = hb < nhb;
            if (tr && r == 0) { if (__float_as_uint(e[0][0]) != 0x7fc12345u) tr[4] = globaltimer_ns(); }
            if (norm && ok) {
                const float4* w4 = reinterpret_cast<const float4*>(p.norm_w) + 4 * hb;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 wv = (r == 0) ? ps.wv[i] : __ldg(w4 + i);
                    ss += e[r][4 * i] * e[r][4 * i] + e[r][4 * i + 1] * e[r][4 * i + 1] + e[r][4 * i + 2] * e[r][4 * i + 2] + e[r][4 * i + 3] * e[r][4 * i + 3];
                    e[r][4 * i] *= wv.x; e[r][4 * i + 1] *= wv.y; e[r][4 * i + 2] *= wv.z; e[r][4 * i + 3] *= wv.w;
                }
            }
            float amax = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(e[r][i]));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));            // the other half of the 32-column block
            const float inv = snap_inv<ABITS>(amax);
            uint32_t hw[4], lw[4];
            int s16 = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int vs;
                snap4<ABITS>(e[r] + 4 * i, inv, &hw[i], &lw[i], &vs);
                s16 += vs;                                                        // sum(v) of this 16-column group
            }
            const int s32 = s16 + __shfl_xor_sync(0xffffffffu, s16, 1);
            if (ok) {
                // half block hb = columns 16 hb ..: unit hb >> 3, 16-B chunk hb & 7 of the unit
                const int u = hb >> 3;
                const int off = (u << 7) + (((hb & 7) ^ (u & 7)) << 4);
                *reinterpret_cast<uint4*>(xhi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                if (ABITS == 16) *reinterpret_cast<uint4*>(xlo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                s16_arr[hb] = s16;
                if ((hb & 1) == 0) {
                    const float sx = amax / (ABITS == 16 ? ACT16_RANGE : ACT8_RANGE);
                    sx_arr[hb >> 1] = sx;
                    sm_arr[hb >> 1] = sx * (float)s32;
                }
            }
        }
    }
    if (tr) tr[5] = globaltimer_ns();
    if (norm) {
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
    }
    named_bar_sync(1, NT);
    float scale = 1.f;
    if (norm) {
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) tot += red[w];
        scale = 1.0f / sqrtf(tot / (float)K + p.eps);
    }
    return scale;
}

// x is staged in nseg pieces of seg_cols columns (narrow rows: one piece = the whole row; wide rows: one K-segment at
// a time through TWO buffers, the bulk copy of piece s+2 issued as soon as piece s has been snapped).
template <int ABITS, int NW>
__device__ __forceinline__ float gemv_prologue_tma(const GemvParams& p, uint8_t* smem, const float* xraw, uint64_t* xbar, int tid,
                                                   const PrologueStaticHB& ps, unsigned long long* tr) {
    constexpr int NT = NW * 32;
    const int K = p.cols;
    const int warp = tid >> 5, lane = tid & 31;
    float* red = reinterpret_cast<float*>(smem + SM_RED);
    uint8_t* xhi = smem + SM_X;
    uint8_t* xlo = xhi + K;
    float* sx_arr = reinterpret_cast<float*>(xlo + K);
    float* sm_arr = sx_arr + K / 32;
    int* s16_arr = reinterpret_cast<int*>(sm_arr + K / 32);
    const int nseg = p.xraw_nseg;
    const int seg_cols = K / nseg;
    const int nhb = seg_cols / 16;          // <= NT (the host only selects this variant then); a multiple of 16
    const uint32_t seg_bytes = (uint32_t)seg_cols * 4u;
    const bool norm = p.norm_w != nullptr;
    if (tid == 0) {
        for (int s = 0; s < min(nseg, 2); ++s) {
            mbar_expect_tx(&xbar[s], seg_bytes);
            tma_load_1d(const_cast<float*>(xraw) + (size_t)s * seg_cols, p.x + (size_t)s * seg_cols, seg_bytes, &xbar[s]);
        }
    }
    float ss = 0.f;
    for (int s = 0; s < nseg; ++s) {
        const int b = s & 1;
        // a warp whose lower half is live runs the body with all its lanes (the two shuffles need them)
        if ((tid & ~31) < nhb) {
            const bool ok = tid < nhb;
            mbar_wait(&xbar[b], (uint32_t)(s >> 1) & 1u);
            if (tr && s == 0) tr[4] = globaltimer_ns();
            const int hb = s * nhb + (ok ? tid : 0);          // half block of the whole row
            float e[16];
            const float4* xr = reinterpret_cast<const float4*>(xraw + (size_t)b * seg_cols) + 4 * (ok ? tid : 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 t = xr[i];
                e[4 * i] = ok ? t.x : 0.f; e[4 * i + 1] = ok ? t.y : 0.f; e[4 * i + 2] = ok ? t.z : 0.f; e[4 * i + 3] = ok ? t.w : 0.f;
            }
            if (norm && ok) {
                const float4* w4 = reinterpret_cast<const float4*>(p.norm_w) + 4 * hb;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 wv = (s == 0) ? ps.wv[i] : __ldg(w4 + i);
                    ss += e[4 * i] * e[4 * i] + e[4 * i + 1] * e[4 * i + 1] + e[4 * i + 2] * e[4 * i + 2] + e[4 * i + 3] * e[4 * i + 3];
                    e[4 * i] *= wv.x; e[4 * i + 1] *= wv.y; e[4 * i + 2] *= wv.z; e[4 * i + 3] *= wv.w;
                }
            }
            float amax = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(e[i]));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));            // the other half of the 32-column block
            const float inv = snap_inv<ABITS>(amax);
            uint32_t hw[4], lw[4];
            int s16 = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int vs;
                snap4<ABITS>(e + 4 * i, inv, &hw[i], &lw[i], &vs);
                s16 += vs;                                                        // sum(v) of this 16-column group
            }
            const int s32 = s16 + __shfl_xor_sync(0xffffffffu, s16, 1);
            if (ok) {
                // half block hb = columns 16 hb ..: unit hb >> 3, 16-B chunk hb & 7 of the unit
                const int u = hb >> 3;
                const int off = (u << 7) + (((hb & 7) ^ (u & 7)) << 4);
                *reinterpret_cast<uint4*>(xhi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                if (ABITS == 16) *reinterpret_cast<uint4*>(xlo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                s16_arr[hb] = s16;
                if ((hb & 1) == 0) {
                    const float sx = amax / (ABITS == 16 ? ACT16_RANGE : ACT8_RANGE);
                    sx_arr[hb >> 1] = sx;
                    sm_arr[hb >> 1] = sx * (float)s32;
                }
            }
        }
        if (s + 1 < nseg) {
            named_bar_sync(1, NT);                              // buffer b has been read by everyone
            if (tid == 0 && s + 2 < nseg) {
                mbar_expect_tx(&xbar[b], seg_bytes);
                tma_load_1d(const_cast<float*>(xraw) + (size_t)b * seg_cols, p.x + (size_t)(s + 2) * seg_cols, seg_bytes, &xbar[b]);
            }
        }
    }
    if (tr) tr[5] = globaltimer_ns();
    if (norm) {
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
    }
    named_bar_sync(1, NT);
    float scale = 1.f;
    if (norm) {
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) tot += red[w];
        scale = 1.0f / sqrtf(tot / (float)K + p.eps);
    }
    return scale;
}

// Wide rows without RMSNorm (ffn_down: K = 14336, 9-14 float4 per thread) take all their loads in ONE round trip.
template <int ABITS, int NW>
__device__ __forceinline__ float gemv_prologue(const GemvParams& p, uint8_t* smem, int tid, const PrologueStatic& ps, unsigned long long* tr = nullptr) {
    if (p.norm_w == nullptr && p.cols > 8192) return gemv_prologue_nb<ABITS, NW, 2 * PROLOGUE_NB>(p, smem, tid, ps, tr);
    return gemv_prologue_nb<ABITS, NW, PROLOGUE_NB>(p, smem, tid, ps, tr);
}

// reduce four per-lane partials over the warp with 6 shuffles.  On return, lane L holds the warp total of row
// ((L >> 3) & 3); i.e. lanes 0-7 -> row 0, 8-15 -> row 1, 16-23 -> row 2, 24-31 -> row 3.
__device__ __forceinline__ float warp_sum4(const float* o, int lane) {
    const bool b4 = lane & 16, b3 = lane & 8;
    float ka = b4 ? o[2] : o[0], kb = b4 ? o[3] : o[1];
    const float sa = b4 ? o[0] : o[2], sb = b4 ? o[1] : o[3];
    ka += __shfl_xor_sync(0xffffffffu, sa, 16);
    kb += __shfl_xor_sync(0xffffffffu, sb, 16);
    float k = b3 ? kb : ka;
    const float snd = b3 ? ka : kb;
    k += __shfl_xor_sync(0xffffffffu, snd, 8);
    k += __shfl_xor_sync(0xffffffffu, k, 4);
    k += __shfl_xor_sync(0xffffffffu, k, 2);
    k += __shfl_xor_sync(0xffffffffu, k, 1);
    return k;
}
// two partials, 5 shuffles: lanes 0-15 -> row 0, 16-31 -> row 1
__device__ __forceinline__ float warp_sum2(const float* o, int lane) {
    const bool b4 = lane & 16;
    float k = b4 ? o[1] : o[0];
    const float snd = b4 ? o[0] : o[1];
    k += __shfl_xor_sync(0xffffffffu, snd, 16);
    k += __shfl_xor_sync(0xffffffffu, k, 8);
    k += __shfl_xor_sync(0xffffffffu, k, 4);
    k += __shfl_xor_sync(0xffffffffu, k, 2);
    k += __shfl_xor_sync(0xffffffffu, k, 1);
    return k;
}

struct EpiCtx {      // per-step constants of the QKV epilogue (position, physical KV page of that position)
    int pos;
    int page;
};
// two dependent loads: the caller issues them right after the upstream wait so that they travel with the prologue's x
__device__ __forceinline__ EpiCtx load_epi_ctx(const GemvParams& p) {
    EpiCtx ec{0, 0};
    if (p.epi == EPI_QKV) {
        ec.pos = __ldcg(&p.st->pos);
        ec.page = __ldcg(p.page_table + ec.pos / KV_PAGE_TOKENS);
    }
    return ec;
}

// ---------------------------------------------------------------------------------------------------
// one item of TYPE with R rows: all its K-segments, reduction, epilogue.  Warp-private.
// ---------------------------------------------------------------------------------------------------
template <int ABITS, int TYPE, int R>
__device__ __forceinline__ void consume_item(const GemvParams& p, const Ring& ring, Track& tr, int warp, int s, int it, uint8_t* smem,
                                             int lane, float scale, const EpiCtx& ec) {
    const ProdDesc& d = p.pd;
    const int K = p.cols;
    const int nks = d.nks, n = 2 * d.seg_nb;
    const int sb = d.seg_bytes[s];
    const int rows = d.seg[s].rows;
    const bool pair = d.pair != 0;
    const bool rope = (p.epi == EPI_QKV && s < 2);
    constexpr int LPR = 32 / R;                 // lanes per row after the reduction (8 or 16)
    const int j = lane / LPR;                   // local row this lane reports
    // rows of the item and the epilogue's operands (requested before the dot products)
    const int h = R / 2;
    const int base_row = pair ? it * h : it * R;
    const int my_row = base_row + (pair ? (j % h) : j);
    bool my_ok = (lane % LPR) == 0 && my_row < rows;
    if (pair) my_ok = my_ok && j < h;
    else if (rope) my_ok = my_ok && (j & 1) == 0;
    float pre0 = 0.f, pre1 = 0.f;
    if (my_ok) {
        if (p.epi == EPI_ADD) pre0 = __ldcg(p.resid + my_row);
        else if (rope) {
            const int d2 = (my_row % p.head_dim) >> 1;
            pre0 = __ldg(p.rope_cos + (size_t)ec.pos * (p.head_dim / 2) + d2);
            pre1 = __ldg(p.rope_sin + (size_t)ec.pos * (p.head_dim / 2) + d2);
        }
    }
    float acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.f;
    const uint8_t* xhi = smem + SM_X;
    const float* sx_arr = reinterpret_cast<const float*>(xhi + 2 * K);
    const bool valid = lane < n;
    for (int ks = 0; ks < nks; ++ks) {
        const unsigned pos = (unsigned)warp * ring.depth + tr.d, par = tr.par;
        tr.advance(ring.depth);
        const uint8_t* slot = ring.slots + (size_t)pos * ring.slot_bytes;
        XPlanes xp;
        {
            const int ug = ks * n + (valid ? lane : 0);
            xp.hi = xhi + ug * 128;
            xp.lo = xhi + K + ug * 128;
            xp.sx = sx_arr + 4 * ug;
            xp.sm = sx_arr + K / 32 + 4 * ug;
            xp.s16 = reinterpret_cast<const int*>(sx_arr + 2 * (K / 32)) + 8 * ug;
            xp.sw = ug & 7;
        }
        mbar_wait(&ring.full[pos], par);
        if (valid) {
            if (TYPE == T_Q4_K) item_dot_q4k<ABITS, R>(slot, sb, lane, xp, acc);
            else if (TYPE == T_Q6_K) item_dot_q6k<ABITS, R>(slot, sb, n, lane, xp, acc);
            else item_dot_q80<ABITS, R>(slot, sb, n, lane, xp, acc);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[pos]);      // this warp was the slot's only reader
    }
    const float tot = (R == 4) ? warp_sum4(acc, lane) : warp_sum2(acc, lane);
    // partner row of a pair: adjacent row (RoPE) or the up row (gate/up, h local rows further)
    const float other = __shfl_xor_sync(0xffffffffu, tot, pair ? h * LPR : LPR);
    if (!my_ok) return;
    const float v0 = tot * scale, v1 = other * scale;      // RMSNorm factor of the fused prologue (1 if none)
    if (p.epi == EPI_STORE) {
        p.out[my_row] = v0;
    } else if (p.epi == EPI_ADD) {
        p.out[my_row] = pre0 + v0;
    } else if (p.epi == EPI_SILU) {
        p.out[my_row] = (v0 / (1.0f + expf(-v0))) * v1;
    } else {   // EPI_QKV
        const int kvh = my_row / p.head_dim, dd = my_row % p.head_dim;
        const size_t off = (((size_t)ec.page * p.n_kv_heads + kvh) * KV_PAGE_TOKENS + (ec.pos % KV_PAGE_TOKENS)) * p.head_dim + dd;
        if (s < 2) {
            const float o0 = v0 * pre0 - v1 * pre1, o1 = v0 * pre1 + v1 * pre0;      // pre0 = cos, pre1 = sin
            if (s == 0) *reinterpret_cast<float2*>(p.out + my_row) = make_float2(o0, o1);
            else *reinterpret_cast<__half2*>(p.k_cache + off) = __floats2half2_rn(o0, o1);
        } else {
            p.v_cache[off] = __float2half_rn(v0);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// consumer main loop over this CTA's items.  All consumer warps call it; tr is the warp's position in its track.
// ---------------------------------------------------------------------------------------------------
template <int ABITS>
__device__ __forceinline__ void gemv_consume(const GemvParams& p, const Ring& ring, Track& tr, uint8_t* smem, int tid, float scale,
                                             const EpiCtx& ec, int cta, int n_ctas) {
    const ProdDesc& d = p.pd;
    const int warp = tid >> 5, lane = tid & 31;
    const WorkRange wr = cta_range(total_items(d), cta, n_ctas);
    const int A = (int)ring.n_tracks;
    if (warp >= A) return;
    for (int i0 = wr.a + warp; i0 < wr.b; i0 += A) {
        int s, it;
        item_of(d, i0, s, it);
        const int type = d.type[s];      // rows per item follow from the type (gemv_plan): Q4_K 4, Q6_K / Q8_0 2
        if (type == T_Q4_K) consume_item<ABITS, T_Q4_K, 4>(p, ring, tr, warp, s, it, smem, lane, scale, ec);
        else if (type == T_Q6_K) consume_item<ABITS, T_Q6_K, 2>(p, ring, tr, warp, s, it, smem, lane, scale, ec);
        else consume_item<ABITS, T_Q8_0, 2>(p, ring, tr, warp, s, it, smem, lane, scale, ec);
    }
}

}  // namespace gl
