// Paged-KV decode attention (one query token, GQA), split over KV pages -- stand-alone kernel of the per-op path.
//
// Stands in for the attention inside Ollama's decode step, reached in the reference only through
// OllamaService.generate*Response (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237).
// Bound: HBM (KV pages) in principle, latency in practice at the 512+128-token workloads of BASELINE.json (2.6 MB
// of KV per layer), so everything is arranged to shorten the dependent chain: one launch; split s owns pages s, s+S,
// ... (independent of the context length), so the pages that are already final are staged with 1-D TMA bulk copies
// BEFORE griddepcontrol.wait, while the QKV GEMV that appends the newest row is still running (a 16-token page of one
// KV head is one contiguous 4 KB block); after the wait only the page holding the newest rows is fetched; per page a
// transposing 16-shuffle score reduction; partials merged by the last CTA of each KV head (atomic ticket) with
// batched loads -- no second kernel.  The grid is fixed (it lives in a CUDA graph); surplus splits leave at once,
// and a context of one page is written straight to the output without partials, ticket or merge.
#include "attn_core.cuh"

namespace gl {

namespace {

constexpr int TILE_PAGES = 4;
constexpr int MAX_GRP = 8;

constexpr int MAX_CL = 16;          // splits of one KV head in one thread-block cluster (cluster mode)

__device__ __forceinline__ uint32_t attn_mapa(uint32_t local_smem_addr, uint32_t rank) {      // the same location in CTA `rank` of the cluster
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_smem_addr), "r"(rank));
    return ra;
}

// CL = false: partials through global memory, merged by the last CTA of each KV head (atomic ticket).
// CL = true : the n_splits CTAs of a KV head are ONE thread-block cluster.  Every split sends each rank the slice of its partial
//             output that rank owns (st.shared::cluster into the rank's receive buffer: distributed shared memory) with its
//             (max, sum); one cluster barrier; every rank merges its slice of the head group's output -- no global round trip,
//             no ticket, and the merge is spread over the cluster (the ticket path: partial store 0.9 us + ticket 0.8 us + the
//             last CTA's 32 partial loads 2.0 us per layer).
template <int DPL, bool CL>   // dims per lane = head_dim / 32
__global__ void __launch_bounds__(32 * MAX_GRP) attn_decode_kernel(const __grid_constant__ AttnParams p) {
    constexpr int HD = DPL * 32;
    constexpr int PAGE_ELEMS = KV_PAGE_TOKENS * HD;
    constexpr uint32_t PAGE_BYTES = PAGE_ELEMS * sizeof(__half);
    __shared__ __align__(128) __half ks[TILE_PAGES * PAGE_ELEMS];
    __shared__ __align__(128) __half vs[TILE_PAGES * PAGE_ELEMS];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int is_last;
    __shared__ __align__(16) float rx_o[CL ? MAX_CL : 1][CL ? 128 : 4];      // [split][this rank's slice of the group's output]
    __shared__ __align__(8) float rx_ml[CL ? MAX_CL : 1][2];                 // [split](max, sum) of the head the slice belongs to

    const int kvh = blockIdx.x, split = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = p.n_head / p.n_kv_heads;
    const int head = kvh * grp + warp;
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

    // Split s owns pages s, s + S, s + 2S, ... -- a mapping that does not depend on the context length, so the pages
    // that are already FINAL can be requested before the upstream kernel (this layer's QKV GEMV, which appends the
    // newest row) has finished: the position counter only grows inside a sequence, so any value read here is a lower
    // bound, and a page whose 16 rows all lie below it was completed by earlier steps.
    const int pos_lb = __ldcg(&p.st->pos);
    const int final_pages = pos_lb / KV_PAGE_TOKENS;
    int npre = 0;
    if (split < final_pages) npre = min(TILE_PAGES, (final_pages - split + S - 1) / S);
    // lane i's page-table entry of this split's i-th page: static, requested before the wait (clamped to the table)
    int my_entry = 0;
    if (warp == 0 && lane < TILE_PAGES) my_entry = __ldcg(p.page_table + min(split + lane * S, p.n_table - 1));
    auto stage = [&](int slot, int page) {        // one lane: two bulk copies of a physical page
        const size_t off = ((size_t)page * p.n_kv_heads + kvh) * PAGE_ELEMS;
        tma_load_1d(ks + slot * PAGE_ELEMS, p.k_cache + off, PAGE_BYTES, &bar);
        tma_load_1d(vs + slot * PAGE_ELEMS, p.v_cache + off, PAGE_BYTES, &bar);
    };
    if (warp == 0 && npre > 0) {
        if (lane == 0) mbar_expect_tx(&bar, 2u * npre * PAGE_BYTES);
        __syncwarp();
        if (lane < npre) stage(lane, my_entry);
    }
    pdl_wait();
    if (tr) tr[1] = globaltimer_ns();

    // q and the position travel together (a warp issues in order: nothing below may consume the position before q is requested)
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
    const int L = __ldcg(&p.st->pos) + 1;
#pragma unroll
    for (int d = 0; d < DPL; ++d) q[d] *= p.scale;
    const int n_pages = (L + KV_PAGE_TOKENS - 1) / KV_PAGE_TOKENS;
    const int active = min(n_pages, S);
    if (!CL && split >= active) return;             // (then nothing was staged either: final_pages <= n_pages)
    const int my_pages = split < active ? (n_pages - split + S - 1) / S : 0;      // cluster mode: idle splits stay for the barrier

    float m_run = -INFINITY, l_run = 0.f;
    uint32_t ph = 0;
    for (int t0 = 0; t0 < my_pages; t0 += TILE_PAGES) {
        const int np = min(TILE_PAGES, my_pages - t0);
        const int have = t0 == 0 ? npre : 0;        // pages of this tile already requested before the wait
        if (have > 0) { mbar_wait(&bar, ph); ph ^= 1; }
        if (np > have) {                            // the rest: the page holding the newest rows (and long contexts)
            // every thread must have seen the previous phase complete before the barrier is armed again: a straggler
            // that still waits for parity p when phase p+1 completes would wait for ever (parity aliasing)
            if (have > 0) __syncthreads();
            if (warp == 0) {
                if (lane == 0) mbar_expect_tx(&bar, 2u * (np - have) * PAGE_BYTES);
                __syncwarp();
                if (lane >= have && lane < np) stage(lane, t0 == 0 ? my_entry : __ldcg(p.page_table + split + (t0 + lane) * S));
            }
            mbar_wait(&bar, ph);
            ph ^= 1;
        }
        for (int i = 0; i < np; ++i) {
            uint2 kk[KV_PAGE_TOKENS], vv[KV_PAGE_TOKENS];
            const __half* kb = ks + i * PAGE_ELEMS + lane * DPL;
            const __half* vb = vs + i * PAGE_ELEMS + lane * DPL;
#pragma unroll
            for (int j = 0; j < KV_PAGE_TOKENS; ++j) {
                if (DPL == 4) {
                    kk[j] = *reinterpret_cast<const uint2*>(kb + j * HD);
                    vv[j] = *reinterpret_cast<const uint2*>(vb + j * HD);
                } else {
                    kk[j] = make_uint2(*reinterpret_cast<const unsigned*>(kb + j * HD), 0u);
                    vv[j] = make_uint2(*reinterpret_cast<const unsigned*>(vb + j * HD), 0u);
                }
            }
            const int pg = split + (t0 + i) * S;
            attn_page_math<DPL>(kk, vv, min(KV_PAGE_TOKENS, L - pg * KV_PAGE_TOKENS), q, o, m_run, l_run);
        }
        if (t0 + TILE_PAGES < my_pages) __syncthreads();   // tile buffers are re-filled by the next TMA
    }

    if (tr) tr[2] = globaltimer_ns();
    if constexpr (CL) {
        const int G = grp * HD, slice = G / S;      // rank r merges outputs [r * slice, (r + 1) * slice) of this KV head's group
        if (split < active) {
            const int f = warp * HD + lane * DPL;   // this lane's dims in the group's flat output
            const uint32_t dst = attn_mapa(smem_u32(&rx_o[split][f % slice]), (uint32_t)(f / slice));
            if (DPL == 4) asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(o[0]), "f"(o[1]), "f"(o[DPL - 2]), "f"(o[DPL - 1]) : "memory");
            else asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dst), "f"(o[0]), "f"(o[1]) : "memory");
            const int per_head = HD / slice;        // ranks that hold slices of this warp's head
            if (lane < per_head) {
                const uint32_t dml = attn_mapa(smem_u32(&rx_ml[split][0]), (uint32_t)(warp * per_head + lane));
                asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dml), "f"(m_run), "f"(l_run) : "memory");
            }
        }
        asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
        const int t = threadIdx.x;
        if (t < slice) {
            float M = -INFINITY;
            for (int sp = 0; sp < active; ++sp) M = fmaxf(M, rx_ml[sp][0]);
            float acc = 0.f, den = 0.f;
            for (int sp = 0; sp < active; ++sp) {   // splits in order: deterministic
                const float w = expf(rx_ml[sp][0] - M);
                den += w * rx_ml[sp][1];
                acc += w * rx_o[sp][t];
            }
            p.out[(size_t)kvh * G + split * slice + t] = acc / den;
        }
        return;
    }
    if (active == 1) {
        const float inv = 1.0f / l_run;
        float* out = p.out + (size_t)head * HD + lane * DPL;
#pragma unroll
        for (int d = 0; d < DPL; ++d) out[d] = o[d] * inv;
        return;
    }
    // partial result of (head, split)
    {
        float* po = p.part_o + ((size_t)head * p.n_splits + split) * HD + lane * DPL;
        if (DPL == 4) *reinterpret_cast<float4*>(po) = make_float4(o[0], o[1], o[DPL - 2], o[DPL - 1]);
        else *reinterpret_cast<float2*>(po) = make_float2(o[0], o[1]);
        if (lane == 0) {
            p.part_ml[((size_t)head * p.n_splits + split) * 2] = m_run;
            p.part_ml[((size_t)head * p.n_splits + split) * 2 + 1] = l_run;
        }
    }
    __syncthreads();
    if (p.trace != nullptr && threadIdx.x == 0) atomicMax(p.trace + 5, globaltimer_ns());      // (profiling) last partial written
    if (threadIdx.x == 0) {
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(p.counters + kvh) : "memory");
        if (p.trace != nullptr) atomicMax(p.trace + 6, globaltimer_ns());                           // (profiling) last ticket drawn
        is_last = (ticket == (unsigned)active - 1);
        if (is_last) p.counters[kvh] = 0;      // ready for the next launch
    }
    __syncthreads();
    if (!is_last) return;
    attn_merge_head<DPL, 32>(p.part_o, p.part_ml, p.out, head, p.n_splits, active, lane);      // all 32 partials in one round trip
    if (p.trace != nullptr && lane == 0) atomicMax(p.trace + 7, globaltimer_ns());                  // (profiling) last merge done
}

}  // namespace

// cluster mode needs: 8 or 16 splits (16 = a non-portable cluster size), and a slice of the group's output per rank that lies
// inside one head and is at least one lane's dims wide
bool attn_cluster_ok(int n_head, int n_kv_heads, int head_dim, int n_splits) {
    if (n_kv_heads < 1 || n_head % n_kv_heads || (n_splits != 8 && n_splits != 16)) return false;
    const int grp = n_head / n_kv_heads, G = grp * head_dim;
    if (grp > MAX_GRP || G % n_splits) return false;
    const int slice = G / n_splits, dpl = head_dim / 32;
    return slice <= head_dim && head_dim % slice == 0 && slice % dpl == 0 && slice <= 32 * grp && slice <= 128;
}

cudaError_t attn_decode_configure() {
    cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel<4, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attn_decode_kernel<2, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    return e;
}

cudaError_t attn_decode_launch(const AttnParams& p, bool pdl, cudaStream_t s) {
    const int grp = p.n_head / p.n_kv_heads;
    if (grp < 1 || grp > MAX_GRP || p.n_head % p.n_kv_heads || p.n_splits < 1 || p.n_splits > 32) return cudaErrorInvalidValue;
    if (p.cluster && !attn_cluster_ok(p.n_head, p.n_kv_heads, p.head_dim, p.n_splits)) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)p.n_kv_heads, (unsigned)p.n_splits);
    cfg.blockDim = dim3(32u * grp);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (pdl) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    if (p.cluster) {
        at[na].id = cudaLaunchAttributeClusterDimension;
        at[na].val.clusterDim.x = 1; at[na].val.clusterDim.y = (unsigned)p.n_splits; at[na].val.clusterDim.z = 1;
        ++na;
    }
    cfg.attrs = at;
    cfg.numAttrs = na;
    if (p.cluster) {
        if (p.head_dim == 128) return cudaLaunchKernelEx(&cfg, attn_decode_kernel<4, true>, p);
        if (p.head_dim == 64) return cudaLaunchKernelEx(&cfg, attn_decode_kernel<2, true>, p);
        return cudaErrorInvalidValue;
    }
    if (p.head_dim == 128) return cudaLaunchKernelEx(&cfg, attn_decode_kernel<4, false>, p);
    if (p.head_dim == 64) return cudaLaunchKernelEx(&cfg, attn_decode_kernel<2, false>, p);
    return cudaErrorInvalidValue;
}

}  // namespace gl
