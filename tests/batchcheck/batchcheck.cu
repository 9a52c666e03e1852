// Test-only launcher shim: lets tests/test_gpu_batch_kernels.py run the per-row kernels of the batched decode step (batch.cu,
// and the embedding gather of prefill.cu) alone on host buffers.  Every entry point copies its host buffers in, runs the
// launch(es), synchronises, copies back every buffer the kernels may touch (sentinels included) and returns the cudaError_t.
// Not part of the C ABI of libgridllm_native.so.
#include <cuda_runtime.h>
#include <stdint.h>

#include "batch.h"
#include "common.cuh"
#include "kernels.h"
#include "prefill.h"

using namespace gl;

namespace {

struct Dev {                         // device copy of one host buffer (null / zero bytes: no buffer)
    void* d = nullptr;
    size_t bytes = 0;
    cudaError_t in(const void* host, size_t n) {
        bytes = n;
        if (!host || !n) return cudaSuccess;
        cudaError_t e = cudaMalloc(&d, n);
        return e == cudaSuccess ? cudaMemcpy(d, host, n, cudaMemcpyHostToDevice) : e;
    }
    cudaError_t fill(size_t n, int byte) {       // a fresh buffer of n bytes, every byte `byte`
        bytes = n;
        cudaError_t e = cudaMalloc(&d, n);
        return e == cudaSuccess ? cudaMemset(d, byte, n) : e;
    }
    cudaError_t out(void* host) const { return d ? cudaMemcpy(host, d, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    ~Dev() { if (d) cudaFree(d); }
    template <typename T> T* p() const { return reinterpret_cast<T*>(d); }
};

#define KC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// The kernel in front of the step's first dependant: lets it start at once, waits ~delay_ns, and only then writes the QKV rows
// (n floats from src to dst), as the QKV GEMM does.  A dependant that reads them before griddepcontrol.wait reads the NaN the
// buffer held before.
__global__ void late_qkv_kernel(const float* src, float* dst, size_t n, unsigned delay_ns) {
    pdl_launch_dependents();
    const unsigned long long t0 = globaltimer_ns();
    while (globaltimer_ns() - t0 < delay_ns) { }
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}

}  // namespace

extern "C" {

int bc_state_bytes() { return (int)sizeof(StepState); }
int bc_ctl_bytes() { return (int)sizeof(BatchCtl); }

// One batched attention launch per replay behind late_qkv_kernel, on fresh copies of the caches, the output, the scratch and the
// counters.  fused = 1: batch_attn_launch with qkv set (it rotates q and appends the step's K / V rows itself); fused = 0:
// batch_rope_kv_launch into q_out, then batch_attn_launch on q.  qkv [bucket][ld] fp32 (the device buffer starts as NaN);
// st [MAX_BATCH] StepState; tables [MAX_BATCH][table_stride]; out16 holds bucket * n_head * hd halves starting out_off halves
// into a buffer of out_halves (the rest: sentinels).  Per replay r, written at offset r of each *_all buffer: the output
// buffer, both caches, the counters ([bucket][n_kv]) and (unfused) q_out ([bucket][n_head * hd] fp32, NaN where not written).
int bc_attn(int fused, int reps, unsigned delay_ns, const float* qkv, int ld, const void* ctl, const void* st, const int* tables,
            int table_stride, const float* cos_t, const float* sin_t, size_t rope_floats, const void* kc, const void* vc, size_t cache_bytes,
            int bucket, int n_head, int n_kv, int hd, int n_splits, float scale, const void* out16, size_t out_halves, size_t out_off,
            void* out_all, void* kc_all, void* vc_all, unsigned* ctr_all, float* q_all) {
    static const cudaError_t conf = batch_attn_configure();
    KC(conf);
    const size_t qkv_floats = (size_t)bucket * ld, q_floats = (size_t)bucket * n_head * hd;
    const size_t part = (size_t)bucket * n_head * n_splits;
    Dev dsrc, dctl, dst, dtab, dcos, dsin;
    KC(dsrc.in(qkv, qkv_floats * 4)); KC(dctl.in(ctl, sizeof(BatchCtl))); KC(dst.in(st, (size_t)MAX_BATCH * sizeof(StepState)));
    KC(dtab.in(tables, (size_t)MAX_BATCH * table_stride * 4)); KC(dcos.in(cos_t, rope_floats * 4)); KC(dsin.in(sin_t, rope_floats * 4));
    for (int r = 0; r < reps; ++r) {
        Dev dqkv, dq, dkc, dvc, dout, dpo, dpml, dctr;
        KC(dqkv.fill(qkv_floats * 4, 0xFF)); KC(dq.fill(q_floats * 4, 0xFF));        // 0xFFFFFFFF: a NaN
        KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes)); KC(dout.in(out16, out_halves * 2));
        KC(dpo.fill(part * hd * 4, 0xFF)); KC(dpml.fill(part * 2 * 4, 0xFF)); KC(dctr.fill((size_t)bucket * n_kv * 4, 0));
        late_qkv_kernel<<<64, 256>>>(dsrc.p<float>(), dqkv.p<float>(), qkv_floats, delay_ns);
        KC(cudaGetLastError());
        const BatchCtl* c = dctl.p<BatchCtl>();
        const StepState* s = dst.p<StepState>();
        if (!fused)
            KC(batch_rope_kv_launch(dqkv.p<float>(), bucket, c, s, dtab.p<int>(), table_stride, n_head, n_kv, hd, dcos.p<float>(), dsin.p<float>(),
                                    dq.p<float>(), dkc.p<__half>(), dvc.p<__half>(), 0));
        BatchAttnParams a{};
        if (fused) { a.qkv = dqkv.p<float>(); a.ld_qkv = ld; a.cos_t = dcos.p<float>(); a.sin_t = dsin.p<float>(); }
        else a.q = dq.p<float>();
        a.k_cache = dkc.p<__half>(); a.v_cache = dvc.p<__half>(); a.tables = dtab.p<int>(); a.table_stride = table_stride; a.st = s; a.ctl = c;
        a.out16 = dout.p<__half>() + out_off; a.part_o = dpo.p<float>(); a.part_ml = dpml.p<float>(); a.counters = dctr.p<unsigned>();
        a.n_head = n_head; a.n_kv_heads = n_kv; a.head_dim = hd; a.n_splits = n_splits; a.scale = scale;
        KC(batch_attn_launch(a, bucket, 0));
        KC(cudaDeviceSynchronize());
        KC(cudaMemcpy(static_cast<uint16_t*>(out_all) + (size_t)r * out_halves, dout.d, out_halves * 2, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(static_cast<uint8_t*>(kc_all) + (size_t)r * cache_bytes, dkc.d, cache_bytes, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(static_cast<uint8_t*>(vc_all) + (size_t)r * cache_bytes, dvc.d, cache_bytes, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(ctr_all + (size_t)r * bucket * n_kv, dctr.d, (size_t)bucket * n_kv * 4, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(q_all + r * q_floats, dq.d, q_floats * 4, cudaMemcpyDeviceToHost));
    }
    return (int)cudaSuccess;
}

// batch_sample_greedy_launch then batch_collect_launch, reps times on fresh copies of the state, the outputs and the scratch.
// st [MAX_BATCH]; out_ids / out_lps [MAX_BATCH][max_out] plus anything the caller appends (sentinels); bout [MAX_BATCH] BatchOut
// (rows >= bucket: sentinels); scratch [MAX_BATCH][BATCH_SAMPLE_ROW_FLOATS].  Everything is written back in place after the last
// replay; *_all get each replay's state and BatchOut.
int bc_sample_greedy(int reps, const float* logits, int n_vocab, int bucket, const void* ctl, void* st, int* out_ids, float* out_lps,
                     size_t out_len, int max_out, void* bout, float* scratch, void* st_all, void* bout_all) {
    Dev dlg, dctl;
    KC(dlg.in(logits, (size_t)bucket * n_vocab * 4)); KC(dctl.in(ctl, sizeof(BatchCtl)));
    const size_t st_bytes = (size_t)MAX_BATCH * sizeof(StepState), bout_bytes = (size_t)MAX_BATCH * sizeof(BatchOut);
    const size_t sc_bytes = (size_t)MAX_BATCH * BATCH_SAMPLE_ROW_FLOATS * 4;
    for (int r = 0; r < reps; ++r) {
        Dev dst, did, dlp, dbo, dsc;
        KC(dst.in(st, st_bytes)); KC(did.in(out_ids, out_len * 4)); KC(dlp.in(out_lps, out_len * 4)); KC(dbo.in(bout, bout_bytes));
        KC(dsc.in(scratch, sc_bytes));
        KC(batch_sample_greedy_launch(dlg.p<float>(), n_vocab, bucket, dctl.p<BatchCtl>(), dst.p<StepState>(), did.p<int>(), dlp.p<float>(), max_out,
                                      dsc.p<float>(), 0));
        KC(batch_collect_launch(dctl.p<BatchCtl>(), dst.p<StepState>(), dlp.p<float>(), max_out, dbo.p<BatchOut>(), bucket, 0));
        KC(cudaDeviceSynchronize());
        KC(cudaMemcpy(static_cast<uint8_t*>(st_all) + r * st_bytes, dst.d, st_bytes, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(static_cast<uint8_t*>(bout_all) + r * bout_bytes, dbo.d, bout_bytes, cudaMemcpyDeviceToHost));
        if (r == reps - 1) { KC(dst.out(st)); KC(did.out(out_ids)); KC(dlp.out(out_lps)); KC(dbo.out(bout)); KC(dsc.out(scratch)); }
    }
    return (int)cudaSuccess;
}

// the single-sequence greedy sampler (sample_greedy_launch) on one row of logits: st is one StepState, out_ids / out_lps [max_out]
int bc_sample_single(const float* logits, int n_vocab, void* st, int* out_ids, float* out_lps, int max_out) {
    Dev dlg, dst, did, dlp, dsc;
    KC(dlg.in(logits, (size_t)n_vocab * 4)); KC(dst.in(st, sizeof(StepState))); KC(did.in(out_ids, (size_t)max_out * 4));
    KC(dlp.in(out_lps, (size_t)max_out * 4));
    KC(dsc.fill(SAMPLE_SCRATCH_FLOATS * 4, 0));
    SampleParams p{};
    p.logits = dlg.p<float>(); p.n_vocab = n_vocab; p.st = dst.p<StepState>(); p.out_ids = did.p<int>(); p.out_logprobs = dlp.p<float>();
    p.max_out = max_out; p.scratch = dsc.p<float>();
    KC(sample_greedy_launch(p, false, 0));
    KC(cudaDeviceSynchronize());
    KC(dst.out(st)); KC(did.out(out_ids)); KC(dlp.out(out_lps));
    return (int)cudaSuccess;
}

// batch_rmsnorm_launch of `rows` rows into y, a buffer of y_halves halves (the rows past `rows`: the caller's sentinels)
int bc_rmsnorm(const float* x, const float* w, int rows, int n, float eps, void* y, size_t y_halves) {
    Dev dx, dw, dy;
    KC(dx.in(x, (size_t)rows * n * 4)); KC(dw.in(w, (size_t)n * 4)); KC(dy.in(y, y_halves * 2));
    KC(batch_rmsnorm_launch(dx.p<float>(), dw.p<float>(), rows, n, eps, dy.p<__half>(), 0));
    KC(cudaDeviceSynchronize());
    KC(dy.out(y));
    return (int)cudaSuccess;
}

// batch_gather_tokens_launch then embed_rows_launch, as the batched step starts: x [x_floats] (rows past bucket: sentinels),
// ids [MAX_BATCH] (past bucket: sentinels)
int bc_embed_rows(const void* w, size_t w_bytes, int type, int cols, int row_bytes, const void* ctl, const void* st, int bucket, float* x,
                  size_t x_floats, int* ids) {
    Dev dw, dctl, dst, dx, did;
    KC(dw.in(w, w_bytes)); KC(dctl.in(ctl, sizeof(BatchCtl))); KC(dst.in(st, (size_t)MAX_BATCH * sizeof(StepState)));
    KC(dx.in(x, x_floats * 4)); KC(did.in(ids, (size_t)MAX_BATCH * 4));
    KC(batch_gather_tokens_launch(dctl.p<BatchCtl>(), dst.p<StepState>(), did.p<int>(), bucket, 0));
    KC(embed_rows_launch(dw.p<uint8_t>(), type, cols, row_bytes, did.p<int>(), bucket, dx.p<float>(), 0));
    KC(cudaDeviceSynchronize());
    KC(dx.out(x)); KC(did.out(ids));
    return (int)cudaSuccess;
}

}  // extern "C"
