// Test-only launcher shim: lets tests/test_gpu_decode_attn.py run the batch-1 decode attention (attn_decode_launch) alone on
// host buffers, behind an upstream kernel that appends the pending K / V rows late.  Not part of the C ABI of
// libgridllm_native.so.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"

using namespace gl;

namespace {

struct Dev {                         // device copy of one host buffer (null / zero bytes: no buffer)
    void* d = nullptr;
    void* h = nullptr;
    size_t bytes = 0;
    cudaError_t in(void* host, size_t n) {
        h = host; bytes = n;
        if (!host || !n) return cudaSuccess;
        cudaError_t e = cudaMalloc(&d, n);
        return e == cudaSuccess ? cudaMemcpy(d, host, n, cudaMemcpyHostToDevice) : e;
    }
    ~Dev() { if (d) cudaFree(d); }
    template <typename T> T* p(size_t byte_off = 0) const { return d ? reinterpret_cast<T*>(static_cast<uint8_t*>(d) + byte_off) : nullptr; }
};

#define KC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// The upstream kernel of a decode attention launch: lets its dependant start at once, waits ~delay_ns, then appends the K / V
// rows of positions [row0, pos] (rows: [n][n_kv][head_dim] each) and publishes the position, as the QKV epilogue and the
// sampler do.  The dependant's pre-wait phase therefore sees those rows missing and a position that may still be row0.
__global__ void append_rows_kernel(StepState* st, __half* kc, __half* vc, const int* table, const __half* krows, const __half* vrows, int row0,
                                   int pos, int n_kv, int hd, unsigned delay_ns) {
    pdl_launch_dependents();
    const unsigned long long t0 = globaltimer_ns();
    while (globaltimer_ns() - t0 < delay_ns) { }
    const int per = n_kv * hd;
    for (int i = threadIdx.x; i < (pos - row0 + 1) * per; i += blockDim.x) {
        const int r = row0 + i / per, h = (i % per) / hd, d = i % hd;
        const size_t off = (((size_t)table[r / KV_PAGE_TOKENS] * n_kv + h) * KV_PAGE_TOKENS + r % KV_PAGE_TOKENS) * hd + d;
        kc[off] = krows[i];
        vc[off] = vrows[i];
    }
    __syncthreads();
    if (threadIdx.x == 0) st->pos = pos;
}

}  // namespace

extern "C" {

// attn_decode_launch (with programmatic dependent launch) behind append_rows_kernel: the caches hold the rows below row0, the
// state's position starts at row0 (row0 = pos: only the newest row is pending; row0 < pos: a stale lower bound) and becomes pos.
// out starts out_off floats into `out` (the rest: caller's sentinels).  reps launches, each on fresh copies of the caches, the
// state and out: out_all = reps x out_floats.  Returns the cudaError_t.
int ac_attn_decode(void* q, size_t q_bytes, void* kc, void* vc, size_t cache_bytes, int* table, int n_table, void* krows, void* vrows,
                   size_t rows_bytes, int row0, int pos, int n_head, int n_kv, int hd, int n_splits, float scale, void* out, size_t out_floats,
                   size_t out_off, int reps, unsigned delay_ns, void* out_all) {
    static const cudaError_t conf = attn_decode_configure();
    KC(conf);
    Dev dq, dtab, dkr, dvr;
    KC(dq.in(q, q_bytes)); KC(dtab.in(table, (size_t)n_table * 4)); KC(dkr.in(krows, rows_bytes)); KC(dvr.in(vrows, rows_bytes));
    for (int r = 0; r < reps; ++r) {
        Dev dkc, dvc, dout, dst;
        StepState st{};
        st.pos = row0;
        KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes)); KC(dout.in(out, out_floats * 4)); KC(dst.in(&st, sizeof(st)));
        append_rows_kernel<<<1, 256>>>(dst.p<StepState>(), dkc.p<__half>(), dvc.p<__half>(), dtab.p<int>(), dkr.p<__half>(), dvr.p<__half>(),
                                       row0, pos, n_kv, hd, delay_ns);
        KC(cudaGetLastError());
        AttnParams a{};
        a.q = dq.p<float>(); a.k_cache = dkc.p<__half>(); a.v_cache = dvc.p<__half>(); a.page_table = dtab.p<int>(); a.n_table = n_table;
        a.st = dst.p<StepState>(); a.out = dout.p<float>(out_off * 4);
        a.n_head = n_head; a.n_kv_heads = n_kv; a.head_dim = hd; a.n_splits = n_splits; a.scale = scale;
        KC(attn_decode_launch(a, true, 0));
        KC(cudaDeviceSynchronize());
        KC(cudaMemcpy(static_cast<float*>(out_all) + (size_t)r * out_floats, dout.d, out_floats * 4, cudaMemcpyDeviceToHost));
    }
    return (int)cudaSuccess;
}

}  // extern "C"
