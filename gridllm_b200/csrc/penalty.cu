// Repetition / presence / frequency penalties on the device (InferenceRequest.options.repeat_penalty, repeat_last_n,
// presence_penalty, frequency_penalty: validated by the reference gateway, server/src/routes/ollama.ts:26-39, and forwarded by
// OllamaService, /root/reference/client/src/services/OllamaService.ts:121-125).  Semantics: gl_sample_opts in
// include/gridllm_native.h and tests/penalty_oracle.py::penalize.  The arithmetic is that of llama.cpp's penalties sampler, which
// Ollama's runner uses [external, unpinned], in single fp32 operations rounded to nearest with no contraction, so that numpy
// float32 reproduces the result bit for bit.
//
// One CTA per sequence row, no sort: pass 1 atomically counts the window's ids into the row's int32[n_vocab] scratch; after a
// CTA barrier pass 2 walks the window again with atomicExch(count[id], 0), and the one thread that gets a non-zero count back
// rewrites logit[id].  Every distinct id is written exactly once whichever thread wins, and the scratch is zero again on exit.
// Cost O(W) for any window up to the context: 2 W L2 atomics and at most W logit read-modify-writes (a few KB at Ollama's
// default window of 64).  Bound: latency -- one small launch, a couple of dependent L2 round trips per thread and pass.  The
// penalty parameters live in StepState, so the captured graphs do not change with the request; rows without penalties and
// finished rows return at once, and the host only puts the kernel into steps where some row has penalties.
#include "common.cuh"
#include "kernels.h"
#include "batch.h"

namespace gl {

namespace {

constexpr int PEN_THREADS = 512;

__global__ void __launch_bounds__(PEN_THREADS) penalty_kernel(const __grid_constant__ PenaltyParams p) {
    pdl_launch_dependents();
    pdl_wait();                                      // the logits come from the lm_head kernel before
    const int row = blockIdx.x;
    int slot = 0;
    if (p.ctl) {
        if (row >= __ldcg(&p.ctl->n_rows)) return;
        slot = __ldcg(&p.ctl->row_slot[row]);
    }
    const StepState* st = p.st + slot;
    const int last_n = __ldcg(&st->pen_last_n);
    if (last_n == 0 || __ldcg(&st->done)) return;
    const int np = __ldcg(&st->n_prompt);
    const int h = np + __ldcg(&st->out_idx);        // history: the prompt, then every token drawn so far
    const int w = last_n < 0 ? h : min(last_n, h);
    const float rp = __ldcg(&st->repeat_penalty), pp = __ldcg(&st->presence_penalty), fp = __ldcg(&st->frequency_penalty);
    const int* prompt = p.prompt + (size_t)slot * p.prompt_stride;
    const int* outs = p.out_ids + (size_t)slot * p.out_stride;
    int* cnt = p.counts + (size_t)slot * p.n_vocab;
    float* lg = p.logits + (size_t)row * p.n_vocab;
    const unsigned nv = (unsigned)p.n_vocab;

    for (int j = h - w + (int)threadIdx.x; j < h; j += PEN_THREADS) {
        const int id = j < np ? __ldcg(prompt + j) : __ldcg(outs + (j - np));
        if ((unsigned)id < nv) atomicAdd(cnt + id, 1);
    }
    __syncthreads();
    for (int j = h - w + (int)threadIdx.x; j < h; j += PEN_THREADS) {
        const int id = j < np ? __ldcg(prompt + j) : __ldcg(outs + (j - np));
        if ((unsigned)id >= nv) continue;
        const int c = atomicExch(cnt + id, 0);
        if (c == 0) continue;                        // another position of the same id took it
        float a = lg[id];
        if (rp != 1.f) a = a <= 0.f ? __fmul_rn(a, rp) : __fdiv_rn(a, rp);
        lg[id] = __fsub_rn(a, __fadd_rn(__fmul_rn((float)c, fp), pp));
    }
}

}  // namespace

cudaError_t penalty_launch(const PenaltyParams& p, int rows, bool pdl, cudaStream_t s) {
    if (!p.logits || !p.st || !p.prompt || !p.out_ids || !p.counts || rows < 1) return cudaErrorInvalidValue;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)rows);
    cfg.blockDim = dim3(PEN_THREADS);
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, penalty_kernel, p);
}

}  // namespace gl
