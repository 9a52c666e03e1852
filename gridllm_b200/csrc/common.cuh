// Device helpers shared by the sm_90a kernels: mbarrier / TMA-bulk PTX, programmatic dependent
// launch, warp reductions.  sm_90a only -- there is no fallback path.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gl {

// State of the sequence being decoded; lives in device memory so that a captured CUDA graph can be
// replayed step after step without host patching (the sampler advances it on the device).
struct StepState {
    int pos;           // position of the token this step processes
    int token;         // token id this step processes
    int n_prompt;      // sequential-prefill mode: prompt length (tokens come from prompt_ids while pos < n_prompt)
    int out_idx;       // next slot in out_ids / out_logprobs
    int done;          // 1 once a stop token was sampled (and !ignore_eos): later steps are no-ops
    int ignore_eos;
    int n_stop;
    int stop_ids[8];
    unsigned bar_base;  // epoch of the persistent kernel's grid barrier (decode_mega.cu)
    // sampling (sampler.cu); temperature 0 = greedy
    float temperature;
    int top_k;          // <= 0 or > SAMPLE_MAX_K: the SAMPLE_MAX_K best logits
    float top_p;        // 1 = off
    unsigned seed_lo, seed_hi;
    float min_p;        // 0 = off (temperature > 0 only)
    // repetition penalties (penalty.cu); pen_last_n = 0: none (the host also sets it to 0 when every penalty is a no-op)
    int pen_last_n;     // window: > 0 the last N history ids, -1 the whole history
    float repeat_penalty;     // 1 = off
    float presence_penalty, frequency_penalty;
    // 1: the JSON grammar mask runs on this sequence (schema_mask.cu; its automaton state lives in its SchemaSlot); 0: none
    int json;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (cudaErrorLaunchFailure), never as
// a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 22)) __trap();
    }
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Programmatic dependent launch (PDL): let the next kernel in the stream start its weight prefetch
// while this one is still running; it blocks in pdl_wait() before touching anything we produce.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace gl
