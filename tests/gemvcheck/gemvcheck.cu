// Test-only launcher shim: lets tests/test_gpu_decode_gemv.py run the batch-1 decode GEMV (gemv_launch) alone on host buffers,
// with the ring geometry the engine picks (gemv_geometry) or an override, behind an upstream kernel that writes x, the residual
// and the position late; and the pieces of the fp-weight decode route one at a time.  Not part of the C ABI of
// libgridllm_native.so.
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"
#include "gguf_file.h"
#include "kernels.h"
#include "rowdot.h"

using namespace gl;

namespace {

struct Dev {                         // device copy of one host buffer (null / zero bytes: no buffer)
    void* d = nullptr;
    size_t bytes = 0;
    cudaError_t in(const void* host, size_t n) {
        bytes = n;
        if (!n) return cudaSuccess;
        cudaError_t e = cudaMalloc(&d, n);
        if (e != cudaSuccess || !host) return e;
        return cudaMemcpy(d, host, n, cudaMemcpyHostToDevice);
    }
    cudaError_t out(void* host) const { return d ? cudaMemcpy(host, d, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    ~Dev() { if (d) cudaFree(d); }
    template <typename T> T* p(size_t byte_off = 0) const { return d ? reinterpret_cast<T*>(static_cast<uint8_t*>(d) + byte_off) : nullptr; }
};

#define KC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// The upstream kernel of a GEMV launch: lets its dependant start at once, waits ~delay_ns, then writes x and the residual
// and publishes the position, as the previous kernels of a decode step do.  Until then the dependant's pre-wait phase sees
// NaN in x and the residual and an in-bounds decoy position whose page is NaN.
__global__ void upstream_kernel(StepState* st, float* x, const float* x_src, int cols, float* resid, const float* resid_src, int n_resid,
                                int pos, unsigned delay_ns) {
    pdl_launch_dependents();
    const unsigned long long t0 = globaltimer_ns();
    while (globaltimer_ns() - t0 < delay_ns) { }
    for (int i = threadIdx.x; i < cols; i += blockDim.x) x[i] = x_src[i];
    if (resid)
        for (int i = threadIdx.x; i < n_resid; i += blockDim.x) resid[i] = resid_src[i];
    __syncthreads();
    if (threadIdx.x == 0) st->pos = pos;
}

// GGUF rows -> the engine layout the loader builds (tile rows: the item's rows, half of them for a gate / up pair)
std::vector<uint8_t> engine_matrix(const uint8_t* gguf, int type, int rows, int cols, int tile_rows) {
    std::vector<uint8_t> mat(engine_matrix_bytes(type, rows, cols, tile_rows), 0);
    const size_t rb = row_bytes((uint32_t)type, cols);
    for (int r = 0; r < rows; ++r) repack_row(type, gguf + (size_t)r * rb, mat.data(), cols, tile_rows, r);
    return mat;
}

}  // namespace

extern "C" {

int gc_state_bytes() { return (int)sizeof(StepState); }

// One decode GEMV launch, reps times on fresh device copies.
//   w0..w2 / types / rows: GGUF-layout blocks of nmat matrices (pair: gate, up), repacked here as the loader does.
//   epi: GemvEpilogue; norm_w (null: no RMSNorm) / eps; x [cols]; resid [rows0] (EPI_ADD; alias: out is the residual).
//   EPI_QKV: rope tables [n_ctx][head_dim / 2], page table, K / V caches; the state's position is decoy_pos until the upstream
//   kernel publishes pos.
//   geom_in: {n_tracks, depth, polite_tracks, prologue 0 / 1 / 2, lean rings 0 / 1}, -1 each = what the engine picks.
//   geom_out: {n_tracks, depth, slot_bytes, prologue, nks} of the launch.
//   out_init [out_floats + 2 pad]: the output with its sentinels (alias: the residual in the middle, which the upstream kernel
//   writes); out_all [reps][out_floats + 2 pad], kc_all / vc_all [reps][cache_bytes], resid_all [reps][rows0] (not aliased).
// Returns 0, a cudaError_t (> 0; a launch gemv_launch refuses comes back without running), -1 when gemv_geometry refuses the
// shape, -2 when the staging does not fit shared memory, -3 for an invalid override.
int gc_gemv(const uint8_t* w0, const uint8_t* w1, const uint8_t* w2, const int* types, const int* rows, int nmat, int pair, int cols,
            int epi, const float* norm_w, float eps, const float* x, const float* resid, int alias, const float* rope_cos,
            const float* rope_sin, size_t rope_floats, int head_dim, int n_kv, const int* table, int n_table, const void* kc,
            const void* vc, size_t cache_bytes, int pos, int decoy_pos, int abits, int nw, int n_ctas, int pdl, const int* geom_in,
            int reps, unsigned delay_ns, const float* out_init, size_t out_floats, size_t pad, float* out_all, void* kc_all,
            void* vc_all, float* resid_all, int* geom_out) {
    static const cudaError_t conf = gemv_configure();
    KC(conf);
    const uint8_t* ws[3] = {w0, w1, w2};
    GemvMat mats[3] = {};
    std::vector<uint8_t> host[3];
    Dev dw[3];
    for (int i = 0; i < nmat && i < 3; ++i) {
        const int tile = pair ? item_rows(types[i]) / 2 : item_rows(types[i]);
        if (!ksplit(cols).nks) return -1;
        host[i] = engine_matrix(ws[i], types[i], rows[i], cols, tile);
        KC(dw[i].in(host[i].data(), host[i].size()));
        mats[i] = GemvMat{dw[i].p<uint8_t>(), types[i], rows[i], tile};
    }
    GemvParams p{};
    GemvGeomOpts o;
    o.nw = nw;
    if (geom_in[3] == 0) { o.hb256 = false; o.xraw = false; }
    else if (geom_in[3] == 1) { o.hb256 = false; o.xraw = true; o.xraw_wide = true; }
    else if (geom_in[3] == 2) { o.hb256 = true; o.xraw = false; }
    if (geom_in[4] >= 0) o.lean_rings = geom_in[4] != 0;
    const int g = gemv_geometry(p, mats, nmat, pair != 0, cols, o, n_ctas);
    if (g == GEMV_GEOM_SHAPE) return -1;
    if (g != GEMV_GEOM_OK) return -2;
    if (geom_in[0] > 0) p.n_tracks = geom_in[0];
    if (geom_in[1] > 0) p.depth = geom_in[1];
    p.polite_tracks = geom_in[2] > 0 ? geom_in[2] : 0;
    if (p.n_tracks > nw || p.n_tracks * p.depth > RING_MAX_SLOTS ||
        gemv_smem_bytes(cols, p.n_tracks * p.depth, p.slot_bytes) + (size_t)p.xraw_bytes > 227 * 1024)
        return -3;
    geom_out[0] = p.n_tracks; geom_out[1] = p.depth; geom_out[2] = p.slot_bytes;
    geom_out[3] = p.hb256 ? 2 : (p.xraw_bytes > 0 ? 1 : 0); geom_out[4] = p.pd.nks;

    const size_t out_total = out_floats + 2 * pad;
    const int n_resid = rows[0];
    Dev dnorm, dxsrc, drsrc, dcos, dsin, dtab;
    KC(dnorm.in(norm_w, norm_w ? (size_t)cols * 4 : 0)); KC(dxsrc.in(x, (size_t)cols * 4));
    KC(drsrc.in(resid, resid ? (size_t)n_resid * 4 : 0));
    KC(dcos.in(rope_cos, rope_cos ? rope_floats * 4 : 0)); KC(dsin.in(rope_sin, rope_sin ? rope_floats * 4 : 0));
    KC(dtab.in(table, table ? (size_t)n_table * 4 : 0));
    const std::vector<float> nan_x((size_t)cols, __builtin_nanf("")), nan_r((size_t)n_resid, __builtin_nanf(""));
    for (int r = 0; r < reps; ++r) {
        Dev dx, dout, dres, dkc, dvc, dst;
        StepState st{};
        st.pos = decoy_pos;
        KC(dx.in(nan_x.data(), (size_t)cols * 4)); KC(dout.in(out_init, out_total * 4)); KC(dst.in(&st, sizeof(st)));
        KC(dkc.in(kc, kc ? cache_bytes : 0)); KC(dvc.in(vc, vc ? cache_bytes : 0));
        float* rdev = nullptr;
        if (resid && alias) rdev = dout.p<float>(pad * 4);
        else if (resid) { KC(dres.in(nan_r.data(), (size_t)n_resid * 4)); rdev = dres.p<float>(); }
        upstream_kernel<<<1, 256>>>(dst.p<StepState>(), dx.p<float>(), dxsrc.p<float>(), cols, rdev, drsrc.p<float>(), n_resid, pos, delay_ns);
        KC(cudaGetLastError());
        p.x = dx.p<float>(); p.norm_w = dnorm.p<float>(); p.eps = eps; p.epi = epi; p.out = dout.p<float>(pad * 4); p.resid = rdev;
        p.rope_cos = dcos.p<float>(); p.rope_sin = dsin.p<float>(); p.head_dim = head_dim; p.n_kv_heads = n_kv;
        p.k_cache = dkc.p<__half>(); p.v_cache = dvc.p<__half>(); p.page_table = dtab.p<int>(); p.st = dst.p<StepState>();
        p.trace = nullptr;
        KC(gemv_launch(p, abits, nw, n_ctas, pdl != 0, 0));
        KC(cudaDeviceSynchronize());
        KC(cudaMemcpy(out_all + (size_t)r * out_total, dout.d, out_total * 4, cudaMemcpyDeviceToHost));
        if (kc) { KC(dkc.out(static_cast<uint8_t*>(kc_all) + (size_t)r * cache_bytes)); KC(dvc.out(static_cast<uint8_t*>(vc_all) + (size_t)r * cache_bytes)); }
        if (resid && !alias) KC(dres.out(resid_all + (size_t)r * n_resid));
    }
    return 0;
}

// ---- the fp-weight decode route (fused_ = false), one launch at a time ---------------------------------------------------------
// y [rows] = W x with W [rows][cols] of type F32 / F16 / BF16 (GGUF layout)
int gc_fp_gemv(const void* w, int type, int rows, int cols, const float* x, float* y) {
    Dev dw, dx, dy;
    KC(dw.in(w, row_bytes((uint32_t)type, cols) * (size_t)rows)); KC(dx.in(x, (size_t)cols * 4)); KC(dy.in(nullptr, (size_t)rows * 4));
    KC(gemv_fp_launch(dw.d, type, rows, cols, dx.p<float>(), dy.p<float>(), 0));
    KC(cudaDeviceSynchronize());
    return (int)dy.out(y);
}

int gc_rmsnorm(const float* x, const float* w, int n, float eps, float* y) {
    Dev dx, dw, dy;
    KC(dx.in(x, (size_t)n * 4)); KC(dw.in(w, (size_t)n * 4)); KC(dy.in(nullptr, (size_t)n * 4));
    KC(rmsnorm_launch(dx.p<float>(), dw.p<float>(), n, eps, dy.p<float>(), 0));
    KC(cudaDeviceSynchronize());
    return (int)dy.out(y);
}

// q [n_head hd] rotated in place; K / V rows [n_kv hd] appended at pos through the page table
int gc_rope_kv(float* q, const float* k, const float* v, int n_head, int n_kv, int hd, const float* cos_t, const float* sin_t, size_t rope_floats,
               int pos, const int* table, int n_table, void* kc, void* vc, size_t cache_bytes) {
    Dev dq, dk, dv, dcos, dsin, dtab, dkc, dvc, dst;
    StepState st{};
    st.pos = pos;
    KC(dq.in(q, (size_t)n_head * hd * 4)); KC(dk.in(k, (size_t)n_kv * hd * 4)); KC(dv.in(v, (size_t)n_kv * hd * 4));
    KC(dcos.in(cos_t, rope_floats * 4)); KC(dsin.in(sin_t, rope_floats * 4)); KC(dtab.in(table, (size_t)n_table * 4));
    KC(dkc.in(kc, cache_bytes)); KC(dvc.in(vc, cache_bytes)); KC(dst.in(&st, sizeof(st)));
    KC(rope_kv_launch(dq.p<float>(), dk.p<float>(), dv.p<float>(), n_head, n_kv, hd, dcos.p<float>(), dsin.p<float>(), dst.p<StepState>(),
                      dkc.p<__half>(), dvc.p<__half>(), dtab.p<int>(), 0));
    KC(cudaDeviceSynchronize());
    KC(dq.out(q)); KC(dkc.out(kc));
    return (int)dvc.out(vc);
}

// op 0: out = silu(a) * b (silu_mul_launch); op 1: out = a + b (add_launch)
int gc_eltwise(int op, const float* a, const float* b, int n, float* out) {
    Dev da, db, dout;
    KC(da.in(a, (size_t)n * 4)); KC(db.in(b, (size_t)n * 4)); KC(dout.in(nullptr, (size_t)n * 4));
    KC(op == 0 ? silu_mul_launch(da.p<float>(), db.p<float>(), n, dout.p<float>(), 0) : add_launch(da.p<float>(), db.p<float>(), n, dout.p<float>(), 0));
    KC(cudaDeviceSynchronize());
    return (int)dout.out(out);
}

// embed_launch on a token_embd of n_vocab GGUF rows; st (a StepState, gc_state_bytes()) is updated in place (its token)
int gc_embed(const void* w, int type, int n_vocab, int cols, void* st, const int* prompt_ids, int n_ids, float* x) {
    Dev dw, dst, dids, dx;
    const size_t rb = row_bytes((uint32_t)type, cols);
    KC(dw.in(w, rb * (size_t)n_vocab)); KC(dst.in(st, sizeof(StepState))); KC(dids.in(prompt_ids, (size_t)n_ids * 4));
    KC(dx.in(nullptr, (size_t)cols * 4));
    EmbedParams ep{dw.p<uint8_t>(), type, cols, (int)rb, dst.p<StepState>(), dids.p<int>(), dx.p<float>()};
    KC(embed_launch(ep, false, 0));
    KC(cudaDeviceSynchronize());
    KC(dst.out(st));
    return (int)dx.out(x);
}

}  // extern "C"
