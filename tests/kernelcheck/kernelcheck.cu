// Test-only launcher shim: lets tests/test_gpu_kernels.py call the tensor-core GEMMs, the quantised-weight GEMM and the prompt
// attention kernel one by one on host buffers.  Every kc_* entry point allocates device copies of its buffers, calls the
// library's launcher, synchronises, copies back every buffer the kernel may touch (whole, so the caller's sentinels come back
// too) and frees.  It returns the cudaError_t.  No arithmetic happens here.  Not part of the C ABI of libgridllm_native.so.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "prefill.h"
#include "qgemm.h"

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
    cudaError_t out() const { return d ? cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    ~Dev() { if (d) cudaFree(d); }
    template <typename T> T* p(size_t byte_off = 0) const { return d ? reinterpret_cast<T*>(static_cast<uint8_t*>(d) + byte_off) : nullptr; }
};

cudaError_t configure() {
    static cudaError_t e = []() {
        cudaError_t r = prefill_configure();
        if (r == cudaSuccess) r = gemm_tc5_configure();
        if (r == cudaSuccess) r = qgemm_configure();
        if (r == cudaSuccess) r = flash_prefill_configure();
        return r;
    }();
    return e;
}

#define KC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// segments of a pack; tab_off[i] = offset of segment i's page table in tab (-1: none)
cudaError_t make_segs(PrefillSegs& s, int nseg, const int* start, const int* len, const int* pos0, const int* tab_off, const Dev& tab) {
    if (nseg < 1 || nseg > PF_MAX_SEGS) return cudaErrorInvalidValue;
    memset(&s, 0, sizeof(s));
    s.n = nseg;
    for (int i = 0; i < nseg; ++i) {
        s.start[i] = start[i]; s.len[i] = len[i]; s.pos0[i] = pos0[i];
        s.table[i] = tab_off[i] >= 0 ? tab.p<int>() + tab_off[i] : nullptr;
    }
    return cudaSuccess;
}

}  // namespace

extern "C" {

int kc_device_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    return n;
}

// gemm_tc5_supported for a plain epilogue, with C at the given address (no launch, nothing dereferenced)
int kc_gemm_tc5_supported(int epi, int m, int n, int k, int lda, int ldb, int ldc, unsigned long long a_addr, unsigned long long b_addr,
                          unsigned long long c_addr) {
    GemmParams g{};
    g.a = reinterpret_cast<const void*>(a_addr); g.b = reinterpret_cast<const void*>(b_addr); g.c = reinterpret_cast<void*>(c_addr);
    g.m = m; g.n = n; g.k = k; g.lda = lda; g.ldb = ldb; g.ldc = ldc; g.batch = 1; g.b_batch_div = 1; g.epi = epi;
    return gemm_tc5_supported(g) ? 1 : 0;
}

// C (+)= A B^T.  which 0: gemm_tc5_launch (a_rows_alloc = rows of A in memory), 1: gemm_tn_launch.  C starts c_off bytes into c.
int kc_gemm(int which, int bf16, int epi, void* a, size_t a_bytes, void* b, size_t b_bytes, void* c, size_t c_bytes, size_t c_off,
            int m, int n, int k, int lda, int ldb, int ldc, int a_rows_alloc, int batch, long long a_bs, long long b_bs, long long c_bs, int b_div) {
    KC(configure());
    Dev da, db, dc;
    KC(da.in(a, a_bytes)); KC(db.in(b, b_bytes)); KC(dc.in(c, c_bytes));
    GemmParams g{};
    g.a = da.d; g.b = db.d; g.c = dc.p<void>(c_off);
    g.m = m; g.n = n; g.k = k; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
    g.batch = batch; g.a_batch_stride = a_bs; g.b_batch_stride = b_bs; g.c_batch_stride = c_bs; g.b_batch_div = b_div; g.epi = epi;
    KC(which == 0 ? gemm_tc5_launch(g, a_rows_alloc, bf16 != 0, 0) : gemm_tn_launch(g, bf16 != 0, 0));
    KC(cudaDeviceSynchronize());
    return (int)dc.out();
}

// gemm_tc5 with GEMM_EPI_ROPE_SPLIT: Q / K rows, V^T columns and the cache pages of every segment (k_cache null: no cache)
int kc_gemm_rope(int bf16, void* a, size_t a_bytes, void* b, size_t b_bytes, int m, int n, int k, int lda, int ldb, int a_rows_alloc,
                 void* cos_t, void* sin_t, size_t cs_bytes, void* q, size_t q_bytes, void* kk, size_t k_bytes, void* vt, size_t vt_bytes,
                 void* kc, void* vc, size_t cache_bytes, int n_head, int n_kv, int hd, int vt_ld,
                 int nseg, const int* start, const int* len, const int* pos0, const int* tab_off, int* tab, size_t tab_bytes) {
    KC(configure());
    Dev da, db, dcos, dsin, dq, dk, dvt, dkc, dvc, dtab;
    KC(da.in(a, a_bytes)); KC(db.in(b, b_bytes)); KC(dcos.in(cos_t, cs_bytes)); KC(dsin.in(sin_t, cs_bytes));
    KC(dq.in(q, q_bytes)); KC(dk.in(kk, k_bytes)); KC(dvt.in(vt, vt_bytes)); KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes));
    KC(dtab.in(tab, tab_bytes));
    RopeSplitArgs ra{dcos.p<float>(), dsin.p<float>(), dq.p<__half>(), dk.p<__half>(), dvt.p<__half>(), dkc.p<__half>(), dvc.p<__half>(),
                     n_head, n_kv, hd, vt_ld, {}};
    KC(make_segs(ra.segs, nseg, start, len, pos0, tab_off, dtab));
    GemmParams g{};
    g.a = da.d; g.b = db.d; g.c = nullptr;
    g.m = m; g.n = n; g.k = k; g.lda = lda; g.ldb = ldb; g.ldc = 0; g.batch = 1; g.b_batch_div = 1; g.epi = GEMM_EPI_ROPE_SPLIT; g.rope = &ra;
    KC(gemm_tc5_launch(g, a_rows_alloc, bf16 != 0, 0));
    KC(cudaDeviceSynchronize());
    KC(dq.out()); KC(dk.out()); KC(dvt.out()); KC(dkc.out());
    return (int)dvc.out();
}

// rope_split_segs_launch: the stand-alone RoPE / split / cache append of a pack
int kc_rope_split_segs(void* qkv, size_t qkv_bytes, int rows_pad, int n_head, int n_kv, int hd, void* cos_t, void* sin_t, size_t cs_bytes,
                       void* q, size_t q_bytes, void* kk, size_t k_bytes, void* vt, size_t vt_bytes, void* kc, void* vc, size_t cache_bytes,
                       int vt_ld, int nseg, const int* start, const int* len, const int* pos0, const int* tab_off, int* tab, size_t tab_bytes) {
    KC(configure());
    Dev dx, dcos, dsin, dq, dk, dvt, dkc, dvc, dtab;
    KC(dx.in(qkv, qkv_bytes)); KC(dcos.in(cos_t, cs_bytes)); KC(dsin.in(sin_t, cs_bytes));
    KC(dq.in(q, q_bytes)); KC(dk.in(kk, k_bytes)); KC(dvt.in(vt, vt_bytes)); KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes));
    KC(dtab.in(tab, tab_bytes));
    PrefillSegs segs;
    KC(make_segs(segs, nseg, start, len, pos0, tab_off, dtab));
    KC(rope_split_segs_launch(dx.p<float>(), rows_pad, n_head, n_kv, hd, dcos.p<float>(), dsin.p<float>(), dq.p<__half>(), dk.p<__half>(),
                              dvt.p<__half>(), dkc.p<__half>(), dvc.p<__half>(), vt_ld, segs, 0));
    KC(cudaDeviceSynchronize());
    KC(dq.out()); KC(dk.out()); KC(dvt.out()); KC(dkc.out());
    return (int)dvc.out();
}

// flash_prefill_launch (paged when some segment has pos0 > 0: keys and values from k_cache / v_cache through the page tables)
int kc_flash_prefill(void* q, size_t q_bytes, void* kk, size_t k_bytes, void* vt, size_t vt_bytes, void* out, size_t out_bytes,
                     void* kc, void* vc, size_t cache_bytes, int n_head, int n_kv, int hd, int vt_ld, float scale,
                     int nseg, const int* start, const int* len, const int* pos0, const int* tab_off, int* tab, size_t tab_bytes) {
    KC(configure());
    Dev dq, dk, dvt, dout, dkc, dvc, dtab;
    KC(dq.in(q, q_bytes)); KC(dk.in(kk, k_bytes)); KC(dvt.in(vt, vt_bytes)); KC(dout.in(out, out_bytes));
    KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes)); KC(dtab.in(tab, tab_bytes));
    PrefillSegs segs;
    KC(make_segs(segs, nseg, start, len, pos0, tab_off, dtab));
    KC(flash_prefill_launch(dq.p<__half>(), dk.p<__half>(), dvt.p<__half>(), dout.p<__half>(), segs, n_head, n_kv, hd, vt_ld, scale,
                            dkc.p<__half>(), dvc.p<__half>(), 0));
    KC(cudaDeviceSynchronize());
    return (int)dout.out();
}

// would qgemm_launch run a GEMM of n_tiles x nkb qtiles in cluster mode?
int kc_qgemm_uses_cluster(int n_tiles, int nkb, int nb, int epi, int n_sm) {
    if (configure() != cudaSuccess) return -1;
    QGemmWeights wt;
    wt.n_tiles = n_tiles; wt.nkb = nkb; wt.n = n_tiles * 128; wt.k = nkb * 256;
    return qgemm_uses_cluster(wt, nb, epi, n_sm) ? 1 : 0;
}

// qgemm_pack_launch of nsrc native GGUF matrices (src[i]: rows[i] x k, type[i]) + QGemmWeights::describe + `reps` launches of
// qgemm_launch, each on a fresh copy of C (c_out: reps x c_bytes) and, when given, of xg / ssq_out.  Outputs beside C:
// tile_off / tile_type (n_tiles each), info = {uses_cluster, two_segment, n_tiles, nkb}, counters after every launch (reps x n_tiles).
int kc_qgemm(int nsrc, int mode, int k, void** src, const size_t* src_bytes, const int* types, const int* rows,
             unsigned long long* tile_off, unsigned char* tile_type, int* info,
             void* act, size_t act_bytes, int act_rows_alloc, int nb, void* c, size_t c_bytes, int ldc, int epi, int n_sm, int reps, void* c_out,
             unsigned* counters_out,
             void* gamma, size_t gamma_bytes, void* xg, size_t xg_bytes, int ldxg, void* ssq_out, size_t ssq_out_bytes,
             void* ssq_in, size_t ssq_in_bytes, int ssq_parts, int n_norm, float eps, void* xg_out_all, void* ssq_out_all) {
    KC(configure());
    if (nsrc < 1 || nsrc > 3 || reps < 1) return (int)cudaErrorInvalidValue;
    Dev dsrc[3], dw, dact, dc, dg, dxg, dso, dsi, dtoff, dttype, dcnt, dpart;
    QGemmSource qs[3];
    size_t stream_bytes = 0;
    for (int i = 0; i < nsrc; ++i) {
        KC(dsrc[i].in(src[i], src_bytes[i]));
        qs[i] = QGemmSource{dsrc[i].p<uint8_t>(), types[i], rows[i]};
        stream_bytes += src_bytes[i];
    }
    int n_rows = 0;
    for (int i = 0; i < nsrc; ++i) n_rows += rows[i];
    const int n_tiles = n_rows / 128, nkb = k / 256;
    KC(cudaMalloc(&dw.d, stream_bytes));
    KC(qgemm_pack_launch(qs, nsrc, mode, k, dw.p<uint8_t>(), reinterpret_cast<uint64_t*>(tile_off), tile_type, 0));
    QGemmWeights wt;
    wt.w = dw.p<uint8_t>(); wt.n = n_rows; wt.k = k; wt.n_tiles = n_tiles; wt.nkb = nkb; wt.bytes = stream_bytes;
    KC(dtoff.in(tile_off, (size_t)n_tiles * 8)); KC(dttype.in(tile_type, (size_t)n_tiles));
    wt.tile_off = dtoff.p<uint64_t>(); wt.tile_type = dttype.p<uint8_t>();
    KC(cudaMalloc(&dcnt.d, (size_t)n_tiles * 4));
    KC(cudaMemset(dcnt.d, 0, (size_t)n_tiles * 4));
    wt.counters = dcnt.p<unsigned>();
    wt.describe(reinterpret_cast<const uint64_t*>(tile_off), tile_type);
    const size_t part_bytes = qgemm_partial_floats(nb) * 4;
    KC(cudaMalloc(&dpart.d, part_bytes));
    KC(cudaMemset(dpart.d, 0xFF, part_bytes));                  // NaN: a partial read before it is written shows up in C
    KC(dact.in(act, act_bytes));
    KC(dg.in(gamma, gamma_bytes)); KC(dsi.in(ssq_in, ssq_in_bytes));
    QGemmNorm norm;
    norm.gamma_next = dg.p<float>(); norm.ldxg = ldxg; norm.ssq_in = dsi.p<float>(); norm.ssq_parts = ssq_parts; norm.n_norm = n_norm; norm.eps = eps;
    info[0] = qgemm_uses_cluster(wt, nb, epi, n_sm) ? 1 : 0;
    info[1] = wt.two_segment ? 1 : 0;
    info[2] = n_tiles;
    info[3] = nkb;
    for (int r = 0; r < reps; ++r) {
        KC(dc.in(c, c_bytes));
        KC(dxg.in(xg, xg_bytes)); KC(dso.in(ssq_out, ssq_out_bytes));
        norm.xg_out = dxg.p<__half>(); norm.ssq_out = dso.p<float>();
        const bool use_norm = gamma || ssq_in;
        KC(qgemm_launch(wt, dact.p<__half>(), act_rows_alloc, nb, dc.d, ldc, epi, dpart.p<float>(), n_sm, 0, use_norm ? &norm : nullptr));
        KC(cudaDeviceSynchronize());
        KC(cudaMemcpy(static_cast<uint8_t*>(c_out) + (size_t)r * c_bytes, dc.d, c_bytes, cudaMemcpyDeviceToHost));
        KC(cudaMemcpy(counters_out + (size_t)r * n_tiles, dcnt.d, (size_t)n_tiles * 4, cudaMemcpyDeviceToHost));
        if (dxg.d) KC(cudaMemcpy(static_cast<uint8_t*>(xg_out_all) + (size_t)r * xg_bytes, dxg.d, xg_bytes, cudaMemcpyDeviceToHost));
        if (dso.d) KC(cudaMemcpy(static_cast<uint8_t*>(ssq_out_all) + (size_t)r * ssq_out_bytes, dso.d, ssq_out_bytes, cudaMemcpyDeviceToHost));
        if (dc.d) { cudaFree(dc.d); dc.d = nullptr; }
        if (dxg.d) { cudaFree(dxg.d); dxg.d = nullptr; }
        if (dso.d) { cudaFree(dso.d); dso.d = nullptr; }
    }
    return (int)cudaSuccess;
}

}  // extern "C"
