// Test-only launcher shim: lets tests/test_gpu_kv_shift.py run the context-shift kernel (kv_shift_launch) alone on host
// buffers.  Not part of the C ABI of libgridllm_native.so.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.h"

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
    cudaError_t out(void* host) const { return d ? cudaMemcpy(host, d, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    ~Dev() { if (d) cudaFree(d); }
    template <typename T> T* p(size_t byte_off = 0) const { return d ? reinterpret_cast<T*>(static_cast<uint8_t*>(d) + byte_off) : nullptr; }
};

#define KC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

}  // namespace

extern "C" {

int sc_state_bytes() { return (int)sizeof(StepState); }

// One kv_shift_launch (as many rounds as the engine would launch) over n_seq sequences.  kc / vc: whole host buffers of
// buf_bytes each (sentinels included); the cache starts cache_off bytes into them.  tables: [n_seq][table_stride] page tables.
// st_buf: int32 host buffer of st_bytes (sentinels included); sequence i's StepState starts st_off[i] bytes into it (-1: none).
// reps launches, each on fresh copies; kc_out / vc_out / st_out receive reps copies of the whole buffers.  Returns cudaError_t.
int sc_kv_shift(const void* kc, const void* vc, size_t buf_bytes, size_t cache_off, size_t layer_elems, int n_layer, int n_kv, int hd,
                const float* cos_t, const float* sin_t, size_t table_floats, const int* tables, int table_stride, const int* keep,
                const int* discard, const int* n_rows, int n_seq, const void* st_buf, size_t st_bytes, const long long* st_off, int reps,
                void* kc_out, void* vc_out, void* st_out) {
    Dev dcos, dsin, dtab;
    KC(dcos.in(cos_t, table_floats * 4)); KC(dsin.in(sin_t, table_floats * 4));
    KC(dtab.in(tables, (size_t)n_seq * table_stride * 4));
    for (int r = 0; r < reps; ++r) {
        Dev dk, dv, dst, dseq;
        KC(dk.in(kc, buf_bytes)); KC(dv.in(vc, buf_bytes)); KC(dst.in(st_buf, st_bytes));
        std::vector<KvShiftSeq> seqs(n_seq);
        int max_rows = 0, rounds = 1;
        for (int i = 0; i < n_seq; ++i) {
            seqs[i] = KvShiftSeq{dtab.p<int>((size_t)i * table_stride * 4), keep[i], discard[i], n_rows[i],
                                 st_off[i] < 0 ? nullptr : dst.p<StepState>((size_t)st_off[i])};
            max_rows = std::max(max_rows, std::min(n_rows[i], discard[i]));
            rounds = std::max(rounds, kv_shift_rounds(n_rows[i], discard[i]));
        }
        KC(dseq.in(seqs.data(), seqs.size() * sizeof(KvShiftSeq)));
        const KvShiftParams p{dk.p<__half>(cache_off), dv.p<__half>(cache_off), layer_elems, dseq.p<KvShiftSeq>(), n_seq, n_layer, n_kv, hd,
                              dcos.p<float>(), dsin.p<float>()};
        KC(kv_shift_launch(p, max_rows, rounds, 0));
        KC(cudaDeviceSynchronize());
        KC(dk.out(static_cast<uint8_t*>(kc_out) + (size_t)r * buf_bytes));
        KC(dv.out(static_cast<uint8_t*>(vc_out) + (size_t)r * buf_bytes));
        KC(dst.out(static_cast<uint8_t*>(st_out) + (size_t)r * st_bytes));
    }
    return (int)cudaSuccess;
}

// Device time of kv_shift_launch on a synthetic pool (values are whatever cudaMalloc left; the time does not depend on them):
// n_seq sequences of W positions each, keep k, the rule's discard, n_layer x n_kv x hd.  *ms = mean of iters launches (each
// restores nothing: the rows move again, which reads and writes the same bytes).  Used by tools/shift_probe.py.
int sc_time_kv_shift(int n_layer, int n_kv, int hd, int W, int keep, int n_seq, int iters, float* ms) {
    const int pages = W / KV_PAGE_TOKENS;
    const size_t layer_elems = (size_t)n_seq * pages * n_kv * KV_PAGE_TOKENS * hd;
    const int d = (W - keep + 1) / 2;
    std::vector<int> tables((size_t)n_seq * pages);
    for (size_t i = 0; i < tables.size(); ++i) tables[i] = (int)i;
    std::vector<float> tab((size_t)W * hd / 2, 0.5f);
    Dev dk, dv, dtab, dcos, dseq, dst;
    KC(cudaMalloc(&dk.d, layer_elems * n_layer * 2)); KC(cudaMalloc(&dv.d, layer_elems * n_layer * 2));
    KC(cudaMemset(dk.d, 0, layer_elems * n_layer * 2)); KC(cudaMemset(dv.d, 0, layer_elems * n_layer * 2));
    KC(dtab.in(tables.data(), tables.size() * 4)); KC(dcos.in(tab.data(), tab.size() * 4));
    std::vector<StepState> sts(n_seq);
    KC(dst.in(sts.data(), sts.size() * sizeof(StepState)));
    std::vector<KvShiftSeq> seqs(n_seq);
    for (int i = 0; i < n_seq; ++i) seqs[i] = KvShiftSeq{dtab.p<int>((size_t)i * pages * 4), keep, d, W - keep - d, dst.p<StepState>(i * sizeof(StepState))};
    KC(dseq.in(seqs.data(), seqs.size() * sizeof(KvShiftSeq)));
    const KvShiftParams p{dk.p<__half>(), dv.p<__half>(), layer_elems, dseq.p<KvShiftSeq>(), n_seq, n_layer, n_kv, hd, dcos.p<float>(), dcos.p<float>()};
    cudaEvent_t a, b;
    KC(cudaEventCreate(&a)); KC(cudaEventCreate(&b));
    for (int i = 0; i < 3; ++i) KC(kv_shift_launch(p, W - keep - d, 1, 0));
    KC(cudaEventRecord(a, 0));
    for (int i = 0; i < iters; ++i) KC(kv_shift_launch(p, W - keep - d, 1, 0));
    KC(cudaEventRecord(b, 0));
    KC(cudaEventSynchronize(b));
    float t = 0.f;
    KC(cudaEventElapsedTime(&t, a, b));
    *ms = t / iters;
    cudaEventDestroy(a); cudaEventDestroy(b);
    return (int)cudaSuccess;
}

}  // extern "C"
