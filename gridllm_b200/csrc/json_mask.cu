// JSON grammar mask on the device (InferenceRequest format: "json" -- validated by the reference gateway,
// server/src/routes/ollama.ts:23-25, 88-90, and forwarded to Ollama by the reference worker,
// client/src/services/OllamaService.ts:209-211).  Language: json_fsm.h; semantics: gl_sample_opts.format in include/gridllm_native.h; restated in
// tests/json_oracle.py.
//
// Grid (vocabulary chunks of JM_THREADS) x rows, one thread per token.  Thread 0 of every CTA rebuilds the row's automaton state
// for this draw: the entry its previous output left (json_st[(i - 1) & 1]) advanced by the piece of the token drawn last
// (StepState.token); output 0 starts from the initial state.  CTA 0 of the row stores the result as entry i & 1, which only the
// next launch reads: no CTA reads what another CTA of the same launch writes, and a captured graph replays with no host.  Every
// thread then runs its token's piece through json_step from that state and writes -inf on rejection.  Stop tokens (the row's
// stop_ids: eos / eot / the request's) are allowed exactly when the root object has closed (json_done); other empty pieces
// (control tokens) never.  Tokens whose piece is plain string text (JSON_CLS_PLAIN) pass the string-body state without the
// byte loop.
//
// Bound: latency -- one launch, one L2 round trip for the offsets and a few for the piece bytes (1-2 MB of table for a 128 k
// vocabulary, resident in L2 after the first step), n_vocab logit writes at most.  Rows without JSON and finished rows return
// at once, and the host only puts the kernel into steps where some row has JSON: one extra launch per draw.
#include "common.cuh"
#include "kernels.h"
#include "batch.h"
#include "json_fsm.h"

namespace gl {

namespace {

constexpr int JM_THREADS = 256;

__device__ __forceinline__ JsonState load_state(const unsigned* w) {
    JsonState s;
    unsigned* d = reinterpret_cast<unsigned*>(&s);
#pragma unroll
    for (int k = 0; k < 4; ++k) d[k] = __ldcg(w + k);
    return s;
}

__device__ __forceinline__ void store_state(unsigned* w, const JsonState& s) {
    const unsigned* d = reinterpret_cast<const unsigned*>(&s);
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = d[k];
}

__device__ __forceinline__ bool run_piece(JsonState& s, const JsonMaskParams& p, int t) {
    const uint32_t a = __ldg(p.offsets + t), b = __ldg(p.offsets + t + 1);
    for (uint32_t i = a; i < b; ++i)
        if (!json_step(s, __ldg(p.bytes + i))) return false;
    return true;
}

__global__ void __launch_bounds__(JM_THREADS) json_mask_kernel(const __grid_constant__ JsonMaskParams p) {
    pdl_launch_dependents();
    pdl_wait();                                      // the logits come from the lm_head (or the penalty kernel) before
    __shared__ JsonState s_state;
    __shared__ int s_stop[8];
    __shared__ int s_nstop;
    const int row = blockIdx.y;
    int slot = 0;
    if (p.ctl) {
        if (row >= __ldcg(&p.ctl->n_rows)) return;
        slot = __ldcg(&p.ctl->row_slot[row]);
    }
    StepState* st = p.st + slot;
    if (!__ldcg(&st->json) || __ldcg(&st->done)) return;
    const int out_idx = __ldcg(&st->out_idx);
    if (threadIdx.x == 0) {
        JsonState s{};
        if (out_idx > 0) {
            s = load_state(st->json_st[(out_idx - 1) & 1]);
            const int prev = __ldcg(&st->token);
            if ((unsigned)prev < (unsigned)p.n_vocab) run_piece(s, p, prev);      // accepted when it was drawn
        }
        if (blockIdx.x == 0) store_state(st->json_st[out_idx & 1], s);
        s_state = s;
        const int ns = min(__ldcg(&st->n_stop), 8);
        s_nstop = ns;
        for (int k = 0; k < ns; ++k) s_stop[k] = __ldcg(&st->stop_ids[k]);
    }
    __syncthreads();
    const int t = blockIdx.x * JM_THREADS + threadIdx.x;
    if (t >= p.n_vocab) return;
    JsonState s = s_state;
    bool stop = false;
    for (int k = 0; k < s_nstop; ++k) stop = stop || s_stop[k] == t;
    bool ok;
    if (stop) ok = json_done(s);
    else if (__ldg(p.offsets + t) == __ldg(p.offsets + t + 1)) ok = false;             // control token
    else if (s.mode == JM_STR && (__ldg(p.cls + t) & JSON_CLS_PLAIN)) ok = true;
    else ok = run_piece(s, p, t);
    if (!ok) p.logits[(size_t)row * p.n_vocab + t] = -INFINITY;
}

__global__ void json_replay_kernel(StepState* st, const int* ids, int n, const uint32_t* offsets, const uint8_t* bytes) {
    JsonState s{};
    for (int j = 0; j + 1 < n; ++j) {
        const int t = ids[j];
        json_run(s, bytes + offsets[t], (int)(offsets[t + 1] - offsets[t]));
    }
    store_state(st->json_st[(n - 1) & 1], s);
}

}  // namespace

cudaError_t json_mask_launch(const JsonMaskParams& p, int rows, bool pdl, cudaStream_t s) {
    if (!p.logits || !p.st || !p.offsets || !p.bytes || !p.cls || rows < 1 || p.n_vocab < 1) return cudaErrorInvalidValue;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)((p.n_vocab + JM_THREADS - 1) / JM_THREADS), (unsigned)rows);
    cfg.blockDim = dim3(JM_THREADS);
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, json_mask_kernel, p);
}

cudaError_t json_replay_launch(StepState* st, const int* ids, int n, const uint32_t* offsets, const uint8_t* bytes, cudaStream_t s) {
    if (!st || !ids || n < 1 || !offsets || !bytes) return cudaErrorInvalidValue;
    json_replay_kernel<<<1, 1, 0, s>>>(st, ids, n, offsets, bytes);
    return cudaGetLastError();
}

}  // namespace gl
