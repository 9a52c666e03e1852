// Seeded temperature / top-k / top-p sampling of one token from the lm_head logits (InferenceRequest.options.temperature,
// top_k, top_p, seed: /root/reference/client/src/types/index.ts:1-27; forwarded by OllamaService.generateResponse,
// /root/reference/client/src/services/OllamaService.ts:101-134).  The arithmetic lives in Ollama in the reference [external];
// the order followed here is top-k -> temperature -> softmax -> top-p -> min-p -> inverse-CDF draw, restated in
// oracle/sampler.py (min-p: tests/penalty_oracle.py).  Repetition penalties (penalty.cu) have already been applied to the
// logits when a request has them.
//
// One CTA of 1024 threads, all passes over the 0.5 MB of logits out of L2:
//   pass 0   online max / sum of exp (log-softmax of the drawn token at T = 1, the same logprob the greedy sampler reports);
//   select   the k best (logit descending, index ascending) by an 8-bit radix select over the 64-bit key
//            (orderable(logit) << 32 | ~index): keys are unique, so ties are broken identically everywhere; per-warp
//            histograms with match.any aggregation (no shared-memory atomics); stops at the first digit whose bin is
//            taken whole -- four passes when the k-th logit is unique;
//   sort     bitonic over <= 1024 candidates in shared memory;
//   draw     w_j = exp((l_j - l_0) / T), running sum in candidate order, top-p cut, u from a counter-based generator
//            (splitmix64 of seed and output index: a request is reproducible whatever the chunking of the host loop).
// Bound: latency.  Measured in a request (run 59): 0.17 ms per token -- one load in flight per thread and pass -- so requests
// with top_k <= 64 (Ollama's default is 40) take a two-stage path instead, sample_topk_fast_kernel below: <= 64 CTAs each sort
// a 2048-logit slice in shared memory and publish their 64 best keys, the last CTA (atomic ticket) merges the sorted lists and
// draws.  The host picks the kernel by the request's top_k (a captured graph per sampler).  Greedy requests launch neither.
#include "common.cuh"
#include "kernels.h"

namespace gl {

namespace {

constexpr int TS_THREADS = 1024;
constexpr int TS_WARPS = TS_THREADS / 32;

__device__ __forceinline__ uint32_t orderable(float v) {
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float from_orderable(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ unsigned long long key_of(float v, int i) {
    return ((unsigned long long)orderable(v) << 32) | (unsigned long long)(~(uint32_t)i);
}

struct MS { float m, s; };
__device__ __forceinline__ MS ms_merge(MS a, MS b) {
    MS r;
    r.m = fmaxf(a.m, b.m);
    const float ea = (a.m == -INFINITY) ? 0.f : expf(a.m - r.m), eb = (b.m == -INFINITY) ? 0.f : expf(b.m - r.m);
    r.s = a.s * ea + b.s * eb;
    return r;
}

// ---- the draw itself (one thread): weights in cum[0..k), candidates sorted in cand[0..k) ------------------------------
__device__ __forceinline__ void draw_and_advance(const SampleParams& p, StepState* st, int out_idx, const unsigned long long* cand, float* cum,
                                                 int k_sel, MS tot) {
    // min-p: the prefix of candidates whose weight w_j = exp((l_j - l_0) / T) is >= min_p (weights do not increase along the
    // candidate order, and w_0 = 1, so this is a prefix of at least one); applied after top-p, both cuts are prefixes
    const float min_p = __ldcg(&st->min_p);
    int n_minp = k_sel;
    if (min_p > 0.f)
        for (int j = 1; j < k_sel; ++j)
            if (!(cum[j] >= min_p)) { n_minp = j; break; }
    float run = 0.f;
    for (int j = 0; j < k_sel; ++j) { run += cum[j]; cum[j] = run; }
    // top-p: the shortest prefix whose mass reaches top_p of the candidates' mass
    const float top_p = __ldcg(&st->top_p);
    int n_keep = k_sel;
    if (top_p > 0.f && top_p < 1.f) {
        const float lim = top_p * run;
        for (int j = 0; j < k_sel; ++j)
            if (cum[j] >= lim) { n_keep = j + 1; break; }
    }
    n_keep = min(n_keep, n_minp);
    // u in [0, 1): 24 bits of splitmix64(seed, output index)
    unsigned long long z = (((unsigned long long)__ldcg(&st->seed_hi) << 32) | __ldcg(&st->seed_lo)) + 0x9E3779B97F4A7C15ull * (unsigned long long)(out_idx + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const float u = (float)(z >> 40) * (1.0f / 16777216.0f);
    const float r = u * cum[n_keep - 1];
    int pick = n_keep - 1;
    for (int j = 0; j < n_keep; ++j)
        if (cum[j] > r) { pick = j; break; }
    const int id = (int)(~(uint32_t)(cand[pick] & 0xffffffffull));
    const float logit = from_orderable((uint32_t)(cand[pick] >> 32));
    if (out_idx < p.max_out) {
        p.out_ids[out_idx] = id;
        p.out_logprobs[out_idx] = (logit - tot.m) - logf(tot.s);
    }
    st->token = id;
    st->pos = st->pos + 1;
    st->out_idx = out_idx + 1;
    if (!st->ignore_eos) {
        for (int q = 0; q < st->n_stop; ++q)
            if (st->stop_ids[q] == id) st->done = 1;
    }
}

// ---- two-stage path for top_k <= TOPK_FAST_K --------------------------------------------------------------------------
constexpr int TF_THREADS = 256;
constexpr int TF_SLICE = 2048;          // logits per CTA (sorted in shared memory)
constexpr int TF_PER_THREAD = TF_SLICE / TF_THREADS;

__device__ __forceinline__ bool topk_fast_applies(int top_k, int n_vocab) {
    return top_k >= 1 && top_k <= TOPK_FAST_K && n_vocab <= TOPK_FAST_MAX_CTAS * TF_SLICE;
}

// descending bitonic sort of P (power of two) keys in shared memory by NT threads
template <int NT>
__device__ __forceinline__ void bitonic_desc(unsigned long long* a, int P, int tid) {
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = tid; t < P / 2; t += NT) {
                const int i = 2 * t - (t & (stride - 1)), j = i + stride;
                const bool desc = (i & size) == 0;
                const unsigned long long x = a[i], y = a[j];
                if ((x < y) == desc) { a[i] = y; a[j] = x; }
            }
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(TF_THREADS) sample_topk_fast_kernel(const __grid_constant__ SampleParams p) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ unsigned long long keys[TOPK_FAST_MAX_CTAS * TOPK_FAST_K];      // 32 KB: stage 1 sorts its slice in the first 2048
    __shared__ float cum[TOPK_FAST_K];
    __shared__ unsigned long long sel[TOPK_FAST_K];
    __shared__ MS red[TF_THREADS / 32];
    __shared__ int is_last;
    static_assert(TOPK_FAST_MAX_CTAS * TOPK_FAST_K >= TF_SLICE, "stage-1 sort buffer");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    StepState* st = p.st;
    if (__ldcg(&st->done)) return;
    const int n = p.n_vocab;
    const int top_k = __ldcg(&st->top_k);
    if (!topk_fast_applies(top_k, n)) __trap();                  // the host picks the kernel by the request's top_k (sample_topk_fast_applies)
    const int out_idx = __ldcg(&st->out_idx);
    const int n_ctas = gridDim.x;                                // = ceil(n / TF_SLICE)
    const bool keep = p.logits_keep != nullptr && out_idx < p.max_out;
    float* dst = keep ? p.logits_keep + (size_t)out_idx * n : nullptr;
    unsigned long long* g_cand = p.topk_scratch;                                   // [n_ctas][TOPK_FAST_K] sorted keys
    float* g_m = reinterpret_cast<float*>(p.topk_scratch + TOPK_FAST_MAX_CTAS * TOPK_FAST_K);
    float* g_s = g_m + TOPK_FAST_MAX_CTAS;
    unsigned* ticket_ctr = reinterpret_cast<unsigned*>(g_s + TOPK_FAST_MAX_CTAS);

    // ---- stage 1: this CTA's slice -> keys in shared memory, (max, sum exp), sort, publish the 64 best ----
    const int base = blockIdx.x * TF_SLICE;
    float v[TF_PER_THREAD];
#pragma unroll
    for (int j = 0; j < TF_PER_THREAD; ++j) {                    // all loads of a thread in flight together
        const int i = base + tid + j * TF_THREADS;
        v[j] = i < n ? __ldcg(p.logits + i) : -INFINITY;
    }
    MS a{-INFINITY, 0.f};
#pragma unroll
    for (int j = 0; j < TF_PER_THREAD; ++j) {
        const int i = base + tid + j * TF_THREADS;
        keys[tid + j * TF_THREADS] = i < n ? key_of(v[j], i) : 0ull;
        if (i < n) {
            if (keep) dst[i] = v[j];
            if (v[j] > a.m) { a.s = (a.m == -INFINITY ? 0.f : a.s * expf(a.m - v[j])) + 1.0f; a.m = v[j]; }
            else if (v[j] != -INFINITY) a.s += expf(v[j] - a.m);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        MS t;
        t.m = __shfl_xor_sync(0xffffffffu, a.m, o);
        t.s = __shfl_xor_sync(0xffffffffu, a.s, o);
        a = ms_merge(a, t);
    }
    if (lane == 0) red[warp] = a;
    bitonic_desc<TF_THREADS>(keys, TF_SLICE, tid);               // (starts with a CTA barrier: keys and red are visible)
    if (tid < TOPK_FAST_K) g_cand[blockIdx.x * TOPK_FAST_K + tid] = keys[tid];
    if (tid == 0) {
        MS t = red[0];
        for (int w = 1; w < TF_THREADS / 32; ++w) t = ms_merge(t, red[w]);
        g_m[blockIdx.x] = t.m;
        g_s[blockIdx.x] = t.s;
    }
    __syncthreads();
    if (tid == 0) {
        unsigned ticket;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(ticket_ctr) : "memory");
        is_last = (ticket == (unsigned)n_ctas - 1);
        if (is_last) *ticket_ctr = 0;
    }
    __syncthreads();
    if (!is_last) return;

    // ---- stage 2 (last CTA): merge the sorted lists, draw ----
    for (int i = tid; i < n_ctas * TOPK_FAST_K; i += TF_THREADS) keys[i] = __ldcg(g_cand + i);
    __syncthreads();
    if (warp != 0) return;
    MS tot{-INFINITY, 0.f};
    for (int c = lane; c < n_ctas; c += 32) tot = ms_merge(tot, MS{__ldcg(g_m + c), __ldcg(g_s + c)});
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        MS t;
        t.m = __shfl_xor_sync(0xffffffffu, tot.m, o);
        t.s = __shfl_xor_sync(0xffffffffu, tot.s, o);
        tot = ms_merge(tot, t);
    }
    const int k_sel = min(top_k, n);
    // lane l owns lists l and l + 32; every round the warp takes the largest head (keys are unique)
    int h0 = 0, h1 = 0;
    const bool has0 = lane < n_ctas, has1 = lane + 32 < n_ctas;
    for (int r = 0; r < k_sel; ++r) {
        const unsigned long long k0 = (has0 && h0 < TOPK_FAST_K) ? keys[lane * TOPK_FAST_K + h0] : 0ull;
        const unsigned long long k1 = (has1 && h1 < TOPK_FAST_K) ? keys[(lane + 32) * TOPK_FAST_K + h1] : 0ull;
        const unsigned long long mine = k0 > k1 ? k0 : k1;
        unsigned long long best = mine;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
            best = t > best ? t : best;
        }
        if (mine == best) {                                       // exactly one lane (a real key is never 0 here: k_sel <= n)
            if (k0 == best) ++h0; else ++h1;
            sel[r] = best;
        }
        __syncwarp();
    }
    const float inv_t = 1.0f / __ldcg(&st->temperature);
    const float top = from_orderable((uint32_t)(sel[0] >> 32));
    for (int j = lane; j < k_sel; j += 32) cum[j] = expf((from_orderable((uint32_t)(sel[j] >> 32)) - top) * inv_t);
    __syncwarp();
    if (lane == 0) draw_and_advance(p, st, out_idx, sel, cum, k_sel, tot);
}

__global__ void __launch_bounds__(TS_THREADS) sample_topk_kernel(const __grid_constant__ SampleParams p) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ unsigned hist[TS_WARPS][256];
    __shared__ unsigned long long cand[SAMPLE_MAX_K];
    __shared__ float cum[SAMPLE_MAX_K];
    __shared__ MS red[TS_WARPS];
    __shared__ unsigned long long s_prefix, s_mask;
    __shared__ int s_need, s_stop, s_ncand;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    StepState* st = p.st;
    const int done = __ldcg(&st->done);
    if (done) return;
    const int out_idx = __ldcg(&st->out_idx);
    const int n = p.n_vocab;
    const bool keep = p.logits_keep != nullptr && out_idx < p.max_out;
    float* dst = keep ? p.logits_keep + (size_t)out_idx * n : nullptr;

    // ---- pass 0: max and sum of exp over the whole vocabulary ----
    MS a{-INFINITY, 0.f};
    for (int i = tid; i < n; i += TS_THREADS) {
        const float v = __ldcg(p.logits + i);
        if (keep) dst[i] = v;
        if (v > a.m) { a.s = (a.m == -INFINITY ? 0.f : a.s * expf(a.m - v)) + 1.0f; a.m = v; }
        else if (v != -INFINITY) a.s += expf(v - a.m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        MS t;
        t.m = __shfl_xor_sync(0xffffffffu, a.m, o);
        t.s = __shfl_xor_sync(0xffffffffu, a.s, o);
        a = ms_merge(a, t);
    }
    if (lane == 0) red[warp] = a;
    if (tid == 0) {
        int k = __ldcg(&st->top_k);
        if (k <= 0 || k > SAMPLE_MAX_K) k = SAMPLE_MAX_K;
        s_need = min(k, n);
        s_prefix = 0ull;
        s_mask = 0ull;
        s_stop = 0;
        s_ncand = 0;
    }
    __syncthreads();
    const int k_sel = s_need;

    // ---- radix select of the k_sel largest keys ----
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = tid; i < TS_WARPS * 256; i += TS_THREADS) (&hist[0][0])[i] = 0u;
        __syncthreads();
        const unsigned long long prefix = s_prefix, mask = s_mask;
        for (int base = 0; base < n; base += TS_THREADS) {
            const int i = base + tid;
            unsigned bin = 0xffffu;
            if (i < n) {
                const unsigned long long key = key_of(__ldcg(p.logits + i), i);
                if ((key & mask) == prefix) bin = (unsigned)(key >> shift) & 255u;
            }
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (bin != 0xffffu && lane == (__ffs(peers) - 1)) hist[warp][bin] += __popc(peers);     // one writer per (warp, bin)
            __syncwarp();
        }
        __syncthreads();
        if (tid < 256) {
            unsigned tot = 0;
            for (int w = 0; w < TS_WARPS; ++w) tot += hist[w][tid];
            hist[0][tid] = tot;
        }
        __syncthreads();
        if (warp == 0) {
            // lane L owns bins 8L .. 8L+7; above = elements in higher bins
            unsigned c = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) c += hist[0][lane * 8 + j];
            unsigned incl = c;                      // suffix sum over lanes >= L
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_down_sync(0xffffffffu, incl, o);
                if (lane + o < 32) incl += t;
            }
            const unsigned above = incl - c;
            const unsigned need = (unsigned)s_need;
            __syncwarp();
            if (above < need && need <= incl) {     // exactly one lane
                unsigned ab = above;
                for (int j = 7; j >= 0; --j) {
                    const unsigned h = hist[0][lane * 8 + j];
                    if (ab + h >= need) {
                        s_prefix = prefix | ((unsigned long long)(lane * 8 + j) << shift);
                        s_mask = mask | (0xffull << shift);
                        s_need = (int)(need - ab);
                        s_stop = (h == need - ab) ? 1 : 0;
                        break;
                    }
                    ab += h;
                }
            }
        }
        __syncthreads();
        if (s_stop) break;
    }

    // ---- gather the selected keys, pad to a power of two, sort descending ----
    int P = 1;
    while (P < k_sel) P <<= 1;
    for (int i = tid; i < P; i += TS_THREADS) cand[i] = 0ull;
    __syncthreads();
    {
        const unsigned long long prefix = s_prefix, mask = s_mask;
        for (int i = tid; i < n; i += TS_THREADS) {
            const unsigned long long key = key_of(__ldcg(p.logits + i), i);
            if ((key & mask) >= prefix) {
                const int j = atomicAdd(&s_ncand, 1);
                if (j < SAMPLE_MAX_K) cand[j] = key;
            }
        }
    }
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            if (tid < P / 2) {
                const int i = 2 * tid - (tid & (stride - 1)), j = i + stride;
                const bool desc = (i & size) == 0;
                const unsigned long long x = cand[i], y = cand[j];
                if ((x < y) == desc) { cand[i] = y; cand[j] = x; }
            }
        }
    }
    __syncthreads();

    // ---- weights at temperature T (relative to the best candidate) ----
    const float inv_t = 1.0f / __ldcg(&st->temperature);
    const float top = from_orderable((uint32_t)(cand[0] >> 32));
    if (tid < k_sel) cum[tid] = expf((from_orderable((uint32_t)(cand[tid] >> 32)) - top) * inv_t);
    __syncthreads();
    if (tid != 0) return;

    MS tot = red[0];
    for (int w = 1; w < TS_WARPS; ++w) tot = ms_merge(tot, red[w]);
    draw_and_advance(p, st, out_idx, cand, cum, k_sel, tot);
}

}  // namespace

bool sample_topk_fast_applies(int top_k, int n_vocab) {
    return top_k >= 1 && top_k <= TOPK_FAST_K && n_vocab <= TOPK_FAST_MAX_CTAS * TF_SLICE;
}

// fast: the two-stage kernel (the caller has checked sample_topk_fast_applies for the request's top_k), else the single-CTA one
cudaError_t sample_topk_launch(const SampleParams& p, bool fast, bool pdl, cudaStream_t s) {
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    if (fast) {
        if (p.topk_scratch == nullptr || p.n_vocab > TOPK_FAST_MAX_CTAS * TF_SLICE) return cudaErrorInvalidValue;
        cfg.gridDim = dim3((unsigned)((p.n_vocab + TF_SLICE - 1) / TF_SLICE));
        cfg.blockDim = dim3(TF_THREADS);
        return cudaLaunchKernelEx(&cfg, sample_topk_fast_kernel, p);
    }
    cfg.gridDim = dim3(1);
    cfg.blockDim = dim3(TS_THREADS);
    return cudaLaunchKernelEx(&cfg, sample_topk_kernel, p);
}

}  // namespace gl
