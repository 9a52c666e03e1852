// JSON grammar mask on the device: Ollama's `format`, either "json" or a JSON schema.  Language: schema_fsm.h over json_fsm.h;
// semantics: gl_sample_opts.format and gl_format_schema in include/gridllm_native.h; restated in tests/json_oracle.py and
// tests/schema_oracle.py.  Format json is the built-in any-object schema, so one kernel masks both kinds of row.
//
// Grid (vocabulary chunks of SM_THREADS) x rows, one thread per token.  A masked row (StepState.json = 1) keeps its automaton
// state in its SchemaSlot (two entries by output parity) and finds its tables through the slot's pointer, so one captured graph
// serves any mix of schemas.  The CTA loads the row's state into shared memory, thread 0 advances it by the piece of the token
// drawn last (StepState.token; output 0 starts from the initial state), and CTA 0 stores the result as the entry of this
// output, which only the next launch reads: no CTA reads what another CTA of the same launch writes, and a captured graph
// replays with no host.  Every thread then walks its token's piece from the shared state with a private JsonState and cursor
// and a private overlay of the frames it touches (it copies a frame from shared memory the first time it needs it; it only ever
// needs the top one or pushes a new one), which is exact for any piece length, and writes -inf on rejection.  Stop tokens (the
// row's stop_ids: eos / eot / the request's) are allowed exactly when the document has closed; other empty pieces (control
// tokens) never.  Plain string text (JSON_CLS_PLAIN) passes an unbounded string without the byte loop.
//
// Bound: latency -- one launch, one L2 round trip for the offsets and a few for the piece bytes (1-2 MB of table for a 128 k
// vocabulary, resident in L2 after the first step), n_vocab logit writes at most.  The host only puts the kernel into steps
// where some row is masked: one extra launch per draw.
#include "common.cuh"
#include "kernels.h"
#include "batch.h"
#include "schema_fsm.h"

namespace gl {

namespace {

constexpr int SM_THREADS = 256;
constexpr int SM_STATE_WORDS = (int)(sizeof(SchemaState) / 4);

struct OverlayFrames {
    const SchemaFrame* sh;       // the row's frames in shared memory
    SchemaFrame pv[JSON_MAX_DEPTH];
    int lo;                      // pv[d] is this thread's frame d for every d >= lo below the depth
    __device__ __forceinline__ SchemaFrame& at(int d) {
        while (lo > d) { --lo; pv[lo] = sh[lo]; }
        return pv[d];
    }
};

__device__ __forceinline__ bool run_piece_schema(const SchemaView& v, JsonState& js, SchemaCursor& cur, SchemaArrayFrames& fr,
                                                 const SchemaMaskParams& p, int t) {
    const uint32_t a = __ldg(p.offsets + t), b = __ldg(p.offsets + t + 1);
    for (uint32_t i = a; i < b; ++i)
        if (!schema_step(v, js, cur, fr, __ldg(p.bytes + i))) return false;
    return true;
}

__global__ void __launch_bounds__(SM_THREADS) schema_mask_kernel(const __grid_constant__ SchemaMaskParams p) {
    pdl_launch_dependents();
    pdl_wait();                                      // the logits come from the lm_head (or the penalty kernel) before
    __shared__ SchemaState s_state;
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
    SchemaSlot* e = p.ctl ? p.ss + slot : p.ss;
    const int out_idx = __ldcg(&st->out_idx);
    const SchemaView v = schema_view((const uint8_t*)__ldcg((const unsigned long long*)&e->tab));
    if (out_idx > 0) {
        const unsigned* src = reinterpret_cast<const unsigned*>(&e->st[(out_idx - 1) & 1]);
        unsigned* dst = reinterpret_cast<unsigned*>(&s_state);
        for (int k = threadIdx.x; k < SM_STATE_WORDS; k += SM_THREADS) dst[k] = __ldcg(src + k);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int prev = out_idx > 0 ? __ldcg(&st->token) : -1;
        if (out_idx == 0) {
            schema_init(s_state.js, s_state.cur, v);
        } else if ((unsigned)prev < (unsigned)p.n_vocab) {
            SchemaArrayFrames fr{s_state.fr};
            run_piece_schema(v, s_state.js, s_state.cur, fr, p, prev);     // accepted when it was drawn
        }
        const int ns = min(__ldcg(&st->n_stop), 8);
        s_nstop = ns;
        for (int k = 0; k < ns; ++k) s_stop[k] = __ldcg(&st->stop_ids[k]);
    }
    __syncthreads();
    if (blockIdx.x == 0) {
        const unsigned* src = reinterpret_cast<const unsigned*>(&s_state);
        unsigned* dst = reinterpret_cast<unsigned*>(&e->st[out_idx & 1]);
        for (int k = threadIdx.x; k < SM_STATE_WORDS; k += SM_THREADS) dst[k] = src[k];
    }
    const int t = blockIdx.x * SM_THREADS + threadIdx.x;
    if (t >= p.n_vocab) return;
    JsonState js = s_state.js;
    SchemaCursor cur = s_state.cur;
    bool stop = false;
    for (int k = 0; k < s_nstop; ++k) stop = stop || s_stop[k] == t;
    bool ok;
    const uint32_t a = __ldg(p.offsets + t), b = __ldg(p.offsets + t + 1);
    if (stop) ok = schema_done(js);
    else if (a == b) ok = false;                                      // control token
    else if (js.mode == JM_STR && (__ldg(p.cls + t) & JSON_CLS_PLAIN) &&
             (cur.phase == SP_ANY || (cur.phase == SP_STR && v.nodes[cur.node].hi == SCHEMA_UNBOUNDED)))
        ok = true;
    else {
        OverlayFrames fr;
        fr.sh = s_state.fr;
        fr.lo = js.depth;
        ok = true;
        for (uint32_t i = a; i < b && ok; ++i) ok = schema_step(v, js, cur, fr, __ldg(p.bytes + i));
    }
    if (!ok) p.logits[(size_t)row * p.n_vocab + t] = -INFINITY;
}

__global__ void schema_replay_kernel(SchemaSlot* e, const int* ids, int n, const uint32_t* offsets, const uint8_t* bytes) {
    SchemaState s;
    const SchemaView v = schema_view(e->tab);
    schema_init(s.js, s.cur, v);
    SchemaArrayFrames fr{s.fr};
    for (int j = 0; j + 1 < n; ++j) {
        const int t = ids[j];
        schema_run(v, s.js, s.cur, fr, bytes + offsets[t], (int)(offsets[t + 1] - offsets[t]));
    }
    e->st[(n - 1) & 1] = s;
}

}  // namespace

cudaError_t schema_mask_launch(const SchemaMaskParams& p, int rows, bool pdl, cudaStream_t s) {
    if (!p.logits || !p.st || !p.ss || !p.offsets || !p.bytes || !p.cls || rows < 1 || p.n_vocab < 1) return cudaErrorInvalidValue;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)((p.n_vocab + SM_THREADS - 1) / SM_THREADS), (unsigned)rows);
    cfg.blockDim = dim3(SM_THREADS);
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, schema_mask_kernel, p);
}

cudaError_t schema_replay_launch(SchemaSlot* e, const int* ids, int n, const uint32_t* offsets, const uint8_t* bytes, cudaStream_t s) {
    if (!e || !ids || n < 1 || !offsets || !bytes) return cudaErrorInvalidValue;
    schema_replay_kernel<<<1, 1, 0, s>>>(e, ids, n, offsets, bytes);
    return cudaGetLastError();
}

}  // namespace gl
