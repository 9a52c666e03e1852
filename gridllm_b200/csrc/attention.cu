// Paged-KV decode attention (one query token, GQA), split over KV pages -- stand-alone kernel of the per-op path.
//
// Stands in for the attention inside Ollama's decode step, reached in the reference only through
// OllamaService.generate*Response (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237).
// Bound: HBM (KV pages) in principle, latency in practice at the 512+128-token workloads of BASELINE.json (2.6 MB
// of KV per layer), so everything is arranged to shorten the dependent chain after griddepcontrol.wait:
// * one launch; the S splits of a KV head are ONE thread-block cluster; split s owns pages s, s+S, ... (independent of the
//   context length), so every row that is already final -- whole pages and the leading rows of the newest page -- is
//   staged with 1-D TMA bulk copies BEFORE the wait, while the QKV GEMV that appends the newest row is still running;
// * after the wait ONE round trip: q, the position and the newest K / V row (the one the QKV epilogue just appended,
//   fetched at the position read before the wait) are requested together;
// * two warps per query head, each walking half of the split's pages, merged in shared memory; the splits merge through
//   distributed shared memory (every split sends each rank the slice of its partial that rank merges, one cluster
//   barrier): no global partials, no atomic ticket, no last-CTA merge.  Splits are merged in rank order: deterministic.
// The grid is fixed (it lives in a CUDA graph); surplus splits only join the barrier, and a context of one page is
// written straight to the output by split 0 without any merge.
#include "attn_core.cuh"

namespace gl {

namespace {

constexpr int STAGE_PAGES = 8;      // pages per split staged at once (before the wait: every final page up to 16 * S * 8 tokens)
constexpr int MAX_GRP = 8;
constexpr int WPH = 2;              // warps per query head
constexpr int MAX_CL = 16;          // splits of one KV head = CTAs of one cluster

__device__ __forceinline__ uint32_t attn_mapa(uint32_t local_smem_addr, uint32_t rank) {      // the same location in CTA `rank` of the cluster
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_smem_addr), "r"(rank));
    return ra;
}

template <int DPL>
__device__ __forceinline__ uint2 ld_row(const __half* p) {      // this lane's DPL dims of one K / V row, through L2
    if (DPL == 4) return __ldcg(reinterpret_cast<const uint2*>(p));
    return make_uint2(__ldcg(reinterpret_cast<const unsigned*>(p)), 0u);
}
template <int DPL>
__device__ __forceinline__ uint2 lds_row(const __half* p) {
    if (DPL == 4) return *reinterpret_cast<const uint2*>(p);
    return make_uint2(*reinterpret_cast<const unsigned*>(p), 0u);
}

// One page against one query head, rows from shared memory except row `jn` (-1: none), which this lane holds in kn / vn.
template <int DPL>
__device__ __forceinline__ void page_math(const __half* kb, const __half* vb, int npos, int jn, uint2 kn, uint2 vn, const float* q, float* o,
                                          float& m_run, float& l_run) {
    constexpr int HD = DPL * 32;
    uint2 kk[KV_PAGE_TOKENS];
#pragma unroll
    for (int j = 0; j < KV_PAGE_TOKENS; ++j) kk[j] = j == jn ? kn : lds_row<DPL>(kb + j * HD);
    const float w = attn_page_scores<DPL>(kk, npos, q, o, m_run, l_run);
#pragma unroll
    for (int j = 0; j < KV_PAGE_TOKENS; ++j) {
        if (j >= npos) break;                                      // warp-uniform; rows beyond npos may hold anything
        attn_pv_row<DPL>(w, j, j == jn ? vn : lds_row<DPL>(vb + j * HD), o);
    }
}

// grid (n_kv_heads, S), cluster (1, S, 1), 32 * WPH * grp threads: warp = half * grp + head of the group
template <int DPL>
__global__ void __launch_bounds__(32 * WPH * MAX_GRP) attn_decode_kernel(const __grid_constant__ AttnParams p) {
    constexpr int HD = DPL * 32;
    constexpr int PAGE_ELEMS = KV_PAGE_TOKENS * HD;
    constexpr uint32_t ROW_BYTES = HD * sizeof(__half);
    extern __shared__ __align__(128) __half stage_buf[];           // [STAGE_PAGES][K page, V page]
    __shared__ __align__(8) uint64_t bar;
    __shared__ __align__(16) float pair_o[MAX_GRP][HD];             // the second warp of each head: its partial
    __shared__ float pair_ml[MAX_GRP][2];
    __shared__ __align__(16) float rx_o[MAX_CL][128];               // [split][this rank's slice of the group's output]
    __shared__ __align__(8) float rx_ml[MAX_CL][MAX_GRP][2];        // [split][head of the group](max, sum)

    const int kvh = blockIdx.x, split = blockIdx.y;                 // cluster (1, S, 1): split = rank in the cluster
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = p.n_head / p.n_kv_heads;
    const int hw = warp % grp, half = warp / grp;
    const int head = kvh * grp + hw;
    const int S = p.n_splits;

    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    unsigned long long* tr = nullptr;
    if (p.trace != nullptr && threadIdx.x == 0 && blockIdx.y == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) tr = p.trace + (blockIdx.x == 0 ? 0 : 8);
    if (tr) tr[0] = globaltimer_ns();
    __syncthreads();
    pdl_launch_dependents();

    // Within a step the position counter only grows (a context shift lowers it, but kv_shift.cu runs BETWEEN steps, launched
    // without programmatic dependent launch and never releasing its dependants early, so no kernel of the next step starts
    // before the lowered position is visible).  A value read before the wait is therefore a lower bound pos_lb: every
    // row below it was appended by an earlier step, whose kernels have completed, and is final.  Only rows < pos_lb are
    // requested here.  Row pos_lb is written by the upstream QKV epilogue (or, if pos_lb is stale, by an earlier step that
    // may still be running); it is read only after the wait, and used only when the position read after the wait is pos_lb.
    const int pos_lb = __ldcg(&p.st->pos);
    const int lb_pages = (pos_lb + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;      // pages holding at least one row < pos_lb
    const int npre = split < lb_pages ? min(STAGE_PAGES, (lb_pages - split + S - 1) / S) : 0;
    const int new_pg = pos_lb / KV_PAGE_TOKENS;                     // page of row pos_lb
    const bool own_new = new_pg % S == split;
    const int new_entry = own_new ? __ldcg(p.page_table + min(new_pg, p.n_table - 1)) : 0;
    int my_entry = 0;                                               // lane i of warp 0: this split's i-th page
    if (warp == 0 && lane < STAGE_PAGES) my_entry = __ldcg(p.page_table + min(split + lane * S, p.n_table - 1));
    auto stage = [&](int slot, int page, int rows) {                // one lane: two bulk copies of the first `rows` rows of a page
        const size_t off = ((size_t)page * p.n_kv_heads + kvh) * PAGE_ELEMS;
        tma_load_1d(stage_buf + slot * 2 * PAGE_ELEMS, p.k_cache + off, rows * ROW_BYTES, &bar);
        tma_load_1d(stage_buf + slot * 2 * PAGE_ELEMS + PAGE_ELEMS, p.v_cache + off, rows * ROW_BYTES, &bar);
    };
    if (warp == 0 && npre > 0) {
        const int rows = lane < npre ? min(KV_PAGE_TOKENS, pos_lb - (split + lane * S) * KV_PAGE_TOKENS) : 0;
        const unsigned total = __reduce_add_sync(0xffffffffu, (unsigned)rows);
        if (lane == 0) mbar_expect_tx(&bar, 2u * total * ROW_BYTES);
        __syncwarp();
        if (lane < npre) stage(lane, my_entry, rows);
    }
    pdl_wait();
    if (tr) tr[1] = globaltimer_ns();

    // one round trip: q, the position and (speculatively, at pos_lb) the newest K / V row travel together
    float q[DPL], o[DPL];
    {
        const float* qp = p.q + (size_t)head * HD + lane * DPL;
        if (DPL == 4) {
            const float4 t = __ldcg(reinterpret_cast<const float4*>(qp));
            q[0] = t.x; q[1] = t.y; q[DPL - 2] = t.z; q[DPL - 1] = t.w;
        } else {
            const float2 t = __ldcg(reinterpret_cast<const float2*>(qp));
            q[0] = t.x; q[1] = t.y;
        }
#pragma unroll
        for (int d = 0; d < DPL; ++d) o[d] = 0.f;
    }
    uint2 kn = make_uint2(0u, 0u), vn = make_uint2(0u, 0u);
    if (own_new) {
        const size_t off = ((size_t)new_entry * p.n_kv_heads + kvh) * PAGE_ELEMS + (size_t)(pos_lb % KV_PAGE_TOKENS) * HD + lane * DPL;
        kn = ld_row<DPL>(p.k_cache + off);
        vn = ld_row<DPL>(p.v_cache + off);
    }
    const int pos = __ldcg(&p.st->pos);
    const int L = pos + 1;
#pragma unroll
    for (int d = 0; d < DPL; ++d) q[d] *= p.scale;
    const int n_pages = (L + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    const int active = min(n_pages, S);
    const int my_pages = split < active ? (n_pages - split + S - 1) / S : 0;
    const bool fresh = pos == pos_lb;                               // else rows >= pos_lb are (re)fetched after the wait

    float m_run = -INFINITY, l_run = 0.f;
    uint32_t ph = 0;
    for (int t0 = 0; t0 < my_pages; t0 += STAGE_PAGES) {
        const int np = min(STAGE_PAGES, my_pages - t0);
        const int have = t0 == 0 ? npre : 0;                        // pages of this tile requested before the wait
        // pages still to fetch: every page of a later tile; in the first tile none when the position is pos_lb (row pos_lb
        // is in registers), else each page holding a row >= pos_lb, whole (its pre-wait rows are fetched again)
        const int first = t0 > 0 ? 0 : fresh ? np : min(np, max(0, (pos_lb / KV_PAGE_TOKENS - split + S - 1) / S));
        if (have > 0) { mbar_wait(&bar, ph); ph ^= 1; }
        if (first < np) {
            // every thread must have seen the previous phase complete before the barrier is armed again (parity aliasing),
            // and the staging slots of the previous tile must be consumed
            if (have > 0 || t0 > 0) __syncthreads();
            if (warp == 0) {
                const int i = t0 + lane;
                const int pg = split + i * S;
                const int rows = lane >= first && lane < np ? min(KV_PAGE_TOKENS, L - pg * KV_PAGE_TOKENS) : 0;
                const unsigned total = __reduce_add_sync(0xffffffffu, (unsigned)rows);
                if (lane == 0) mbar_expect_tx(&bar, 2u * total * ROW_BYTES);
                __syncwarp();
                if (rows > 0) stage(lane, t0 == 0 ? my_entry : __ldcg(p.page_table + pg), rows);
            }
            mbar_wait(&bar, ph);
            ph ^= 1;
        }
        for (int i = half; i < np; i += WPH) {
            const int pg = split + (t0 + i) * S;
            const int jn = (t0 == 0 && fresh && pg == new_pg) ? pos_lb % KV_PAGE_TOKENS : -1;
            const __half* kb = stage_buf + i * 2 * PAGE_ELEMS + lane * DPL;
            page_math<DPL>(kb, kb + PAGE_ELEMS, min(KV_PAGE_TOKENS, L - pg * KV_PAGE_TOKENS), jn, kn, vn, q, o, m_run, l_run);
        }
        if (t0 + STAGE_PAGES < my_pages) __syncthreads();           // slots are re-filled by the next tile's copies
    }

    // the two warps of a head: the second hands its partial to the first through shared memory
    if (half == 1) {
        if (DPL == 4) *reinterpret_cast<float4*>(&pair_o[hw][lane * DPL]) = make_float4(o[0], o[1], o[DPL - 2], o[DPL - 1]);
        else *reinterpret_cast<float2*>(&pair_o[hw][lane * DPL]) = make_float2(o[0], o[1]);
        if (lane == 0) { pair_ml[hw][0] = m_run; pair_ml[hw][1] = l_run; }
    }
    __syncthreads();
    if (tr) tr[2] = globaltimer_ns();
    if (half == 0 && split < active) {
        const float m1 = pair_ml[hw][0], l1 = pair_ml[hw][1];
        const float M = fmaxf(m_run, m1);                           // split < active: this split has a page, so M is finite
        const float w0 = m_run == -INFINITY ? 0.f : expf(m_run - M), w1 = m1 == -INFINITY ? 0.f : expf(m1 - M);
#pragma unroll
        for (int d = 0; d < DPL; ++d) o[d] = o[d] * w0 + pair_o[hw][lane * DPL + d] * w1;
        m_run = M;
        l_run = l_run * w0 + l1 * w1;
    }
    if (active == 1) {                                              // one page: split 0 holds the result, no merge
        if (split == 0 && half == 0) {
            const float inv = 1.0f / l_run;
            float* out = p.out + (size_t)head * HD + lane * DPL;
#pragma unroll
            for (int d = 0; d < DPL; ++d) out[d] = o[d] * inv;
        }
        return;
    }
    const int G = grp * HD, slice = G / S;                          // rank r merges outputs [r * slice, (r + 1) * slice) of the group
    if (half == 0 && split < active) {
        const int f = hw * HD + lane * DPL;                         // this lane's dims in the group's flat output
        const uint32_t dst = attn_mapa(smem_u32(&rx_o[split][f % slice]), (uint32_t)(f / slice));
        if (DPL == 4) asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(o[0]), "f"(o[1]), "f"(o[DPL - 2]), "f"(o[DPL - 1]) : "memory");
        else asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dst), "f"(o[0]), "f"(o[1]) : "memory");
        if (lane < S) {                                             // (max, sum) of this head to every rank
            const uint32_t dml = attn_mapa(smem_u32(&rx_ml[split][hw][0]), (uint32_t)lane);
            asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dml), "f"(m_run), "f"(l_run) : "memory");
        }
    }
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    const int t = threadIdx.x;
    if (t < slice) {
        const int f = split * slice + t, hh = f / HD;
        float M = -INFINITY;
        for (int sp = 0; sp < active; ++sp) M = fmaxf(M, rx_ml[sp][hh][0]);
        float acc = 0.f, den = 0.f;
        for (int sp = 0; sp < active; ++sp) {                       // splits in rank order: deterministic
            const float w = expf(rx_ml[sp][hh][0] - M);
            den += w * rx_ml[sp][hh][1];
            acc += w * rx_o[sp][t];
        }
        p.out[(size_t)kvh * G + f] = acc / den;
    }
    if (tr) tr[3] = globaltimer_ns();
}

size_t attn_stage_bytes(int head_dim) { return (size_t)STAGE_PAGES * 2 * KV_PAGE_TOKENS * head_dim * sizeof(__half); }

}  // namespace

// 8 or 16 splits (16 = a non-portable cluster size), and a slice of the group's output per rank that is a whole number of
// lanes' dims and fits the receive buffer
bool attn_splits_ok(int n_head, int n_kv_heads, int head_dim, int n_splits) {
    if (n_kv_heads < 1 || n_head % n_kv_heads || (n_splits != 8 && n_splits != 16) || (head_dim != 64 && head_dim != 128)) return false;
    const int grp = n_head / n_kv_heads, G = grp * head_dim;
    if (grp > MAX_GRP || G % n_splits) return false;
    const int slice = G / n_splits;
    return slice % (head_dim / 32) == 0 && slice <= 128;
}

cudaError_t attn_decode_configure() {
    cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel<4>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_decode_kernel<2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_decode_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_stage_bytes(128));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_decode_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_stage_bytes(64));
    return e;
}

cudaError_t attn_decode_launch(const AttnParams& p, bool pdl, cudaStream_t s) {
    if (!attn_splits_ok(p.n_head, p.n_kv_heads, p.head_dim, p.n_splits)) return cudaErrorInvalidValue;
    const int grp = p.n_head / p.n_kv_heads;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)p.n_kv_heads, (unsigned)p.n_splits);
    cfg.blockDim = dim3(32u * WPH * grp);
    cfg.dynamicSmemBytes = attn_stage_bytes(p.head_dim);
    cfg.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (pdl) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = 1; at[na].val.clusterDim.y = (unsigned)p.n_splits; at[na].val.clusterDim.z = 1;
    ++na;
    cfg.attrs = at;
    cfg.numAttrs = na;
    return p.head_dim == 128 ? cudaLaunchKernelEx(&cfg, attn_decode_kernel<4>, p) : cudaLaunchKernelEx(&cfg, attn_decode_kernel<2>, p);
}

}  // namespace gl
