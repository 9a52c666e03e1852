// JSON schema mask on the device (Ollama's `format` as a JSON schema).  Language: schema_fsm.h over json_fsm.h; semantics:
// gl_format_schema in include/gridllm_native.h; restated in tests/schema_oracle.py.
//
// The grid of json_mask_kernel: vocabulary chunks of SM_THREADS x rows, one thread per token.  A row with a schema
// (StepState.json = 2) keeps its automaton state in its SchemaSlot (two entries by output parity, like StepState.json_st) and
// finds its tables through the slot's pointer, so one captured graph serves any mix of schemas.  A row with format json
// (StepState.json = 1) is the built-in any-object schema: its state stays the JsonState in StepState.json_st (the one
// json_mask_kernel keeps), from which the cursor follows, so the two kernels can take turns on the same row and give identical
// masks.
//
// The CTA loads the row's state into shared memory, thread 0 advances it by the piece of the token drawn last, and CTA 0 stores
// the result as the entry of this output.  Every thread then walks its token's piece from the shared state with a private
// JsonState and cursor and a private overlay of the frames it touches (it copies a frame from shared memory the first time it
// needs it; it only ever needs the top one or pushes a new one), which is exact for any piece length.  Plain string text takes
// the fast path of json_mask_kernel where the string is unbounded.
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
    const int kind = __ldcg(&st->json);
    if (!kind || __ldcg(&st->done)) return;
    SchemaSlot* e = p.ctl ? p.ss + slot : p.ss;
    const int out_idx = __ldcg(&st->out_idx);
    const uint8_t* tab = kind == 1 ? p.json_tab : (const uint8_t*)__ldcg((const unsigned long long*)&e->tab);
    const SchemaView v = schema_view(tab);
    if (kind == 2 && out_idx > 0) {
        const unsigned* src = reinterpret_cast<const unsigned*>(&e->st[(out_idx - 1) & 1]);
        unsigned* dst = reinterpret_cast<unsigned*>(&s_state);
        for (int k = threadIdx.x; k < SM_STATE_WORDS; k += SM_THREADS) dst[k] = __ldcg(src + k);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int prev = out_idx > 0 ? __ldcg(&st->token) : -1;
        if (kind == 1) {                                             // format json: the JsonState of json_mask_kernel
            JsonState js{};
            if (out_idx > 0) {
                unsigned* d = reinterpret_cast<unsigned*>(&js);
                for (int k = 0; k < 4; ++k) d[k] = __ldcg(&st->json_st[(out_idx - 1) & 1][k]);
                if ((unsigned)prev < (unsigned)p.n_vocab) {
                    const uint32_t a = __ldg(p.offsets + prev), b = __ldg(p.offsets + prev + 1);
                    json_run(js, p.bytes + a, (int)(b - a));
                }
            }
            if (blockIdx.x == 0) {
                const unsigned* d = reinterpret_cast<const unsigned*>(&js);
                for (int k = 0; k < 4; ++k) st->json_st[out_idx & 1][k] = d[k];
            }
            s_state.js = js;
            schema_cursor_of_json(js, v, s_state.cur);
        } else if (out_idx == 0) {
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
    if (kind == 2 && blockIdx.x == 0) {
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
    if (!p.logits || !p.st || !p.ss || !p.json_tab || !p.offsets || !p.bytes || !p.cls || rows < 1 || p.n_vocab < 1) return cudaErrorInvalidValue;
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
