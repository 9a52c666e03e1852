// Context shift of the paged KV cache (kernels.h kv_shift_launch; rule in include/gridllm_native.h): llama.cpp's K-shift --
// RoPE by a delta position on the cached K -- applied to the rows a shift keeps, while they move down by `discard` positions.
//
// Grid: x = blocks of KS_ROWS moved rows, y = KV head, z = (sequence, layer).  A row of one KV head is head_dim fp16 values,
// taken as 16-byte vectors (8 values, 4 rotated pairs) by head_dim / 8 threads.  Every byte is read once and written once:
// the kernel is bound by HBM.
//
// No programmatic dependent launch in either direction: launched without the attribute (it waits for the step before it) and
// never executing griddepcontrol.launch_dependents (the next step's kernels, the decode attention among them, which reads the
// position before its own wait, start only after this grid has completed and lowered the position).
#include "common.cuh"
#include "kernels.h"

namespace gl {

namespace {

constexpr int KS_THREADS = 256;
constexpr int KS_ROWS = 32;            // moved rows per CTA

__device__ __forceinline__ size_t row_off(const int* table, int row, int kvh, int n_kv, int hd) {
    return (((size_t)table[row / KV_PAGE_TOKENS] * n_kv + kvh) * KV_PAGE_TOKENS + row % KV_PAGE_TOKENS) * hd;
}

__global__ void __launch_bounds__(KS_THREADS) kv_shift_kernel(const __grid_constant__ KvShiftParams p, int round, int last_round) {
    const int seq = blockIdx.z / p.n_layer, layer = blockIdx.z % p.n_layer, kvh = blockIdx.y;
    const KvShiftSeq q = p.seqs[seq];
    if (round == last_round && blockIdx.x == 0 && blockIdx.y == 0 && layer == 0 && threadIdx.x == 0 && q.st) q.st->pos -= q.discard;
    // this round's rows of the sequence: local rows [round * discard, min((round + 1) * discard, n_rows))
    const int lo = round * q.discard;
    const int hi = min(lo + q.discard, q.n_rows);
    const int hd = p.head_dim, vpr = hd / 8;                        // 16-byte vectors per row
    const int rows_per_pass = KS_THREADS / vpr;
    const int v = threadIdx.x % vpr;
    __half* k_cache = p.k_cache + (size_t)layer * p.layer_elems;
    __half* v_cache = p.v_cache + (size_t)layer * p.layer_elems;
    // pairs 4v .. 4v + 3 of the head: the rotation by -discard
    const float4 c = *reinterpret_cast<const float4*>(p.cos_t + (size_t)q.discard * (hd / 2) + 4 * v);
    const float4 s = *reinterpret_cast<const float4*>(p.sin_t + (size_t)q.discard * (hd / 2) + 4 * v);
    const float cc[4] = {c.x, c.y, c.z, c.w}, ss[4] = {s.x, s.y, s.z, s.w};
    for (int j = lo + blockIdx.x * KS_ROWS + threadIdx.x / vpr; j < min(hi, lo + (blockIdx.x + 1) * KS_ROWS); j += rows_per_pass) {
        const int src = q.keep + q.discard + j, dst = q.keep + j;
        const size_t so = row_off(q.table, src, kvh, p.n_kv, hd) + 8 * v, dof = row_off(q.table, dst, kvh, p.n_kv, hd) + 8 * v;
        const uint4 kr = __ldcs(reinterpret_cast<const uint4*>(k_cache + so));
        const uint4 vr = __ldcs(reinterpret_cast<const uint4*>(v_cache + so));
        const __half2* kh = reinterpret_cast<const __half2*>(&kr);
        uint4 ko;
        __half2* oh = reinterpret_cast<__half2*>(&ko);
        // in double: the products of an fp16 value and an fp32 table entry are exact, the sum is rounded once, and the one
        // rounding to fp16 gives the correctly rounded rotation (fp32 would lose bits to cancellation in a small result).
        // The kernel is bound by HBM, so the fp64 arithmetic costs nothing.
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 ab = __half22float2(kh[i]);
            const double a = ab.x, b = ab.y, c = cc[i], sn = ss[i];
            oh[i] = __halves2half2(__double2half(a * c + b * sn), __double2half(b * c - a * sn));
        }
        __stcs(reinterpret_cast<uint4*>(k_cache + dof), ko);
        __stcs(reinterpret_cast<uint4*>(v_cache + dof), vr);
    }
}

}  // namespace

int kv_shift_rounds(int n_rows, int discard) {
    if (n_rows <= 0 || discard <= 0) return 1;
    return (n_rows + discard - 1) / discard;
}

cudaError_t kv_shift_launch(const KvShiftParams& p, int max_rows, int n_rounds, cudaStream_t s) {
    if (p.n_seq <= 0) return cudaSuccess;
    if (p.head_dim % 32 || p.head_dim > 256 || (long long)p.n_seq * p.n_layer > 65535) return cudaErrorInvalidValue;
    n_rounds = n_rounds < 1 ? 1 : n_rounds;
    // rows of one round: at most min(discard, n_rows) per sequence, and never more than max_rows
    const int per_round = max_rows > 0 ? max_rows : 1;
    const dim3 grid((unsigned)((per_round + KS_ROWS - 1) / KS_ROWS), (unsigned)p.n_kv, (unsigned)(p.n_seq * p.n_layer));
    for (int r = 0; r < n_rounds; ++r) {
        kv_shift_kernel<<<grid, KS_THREADS, 0, s>>>(p, r, n_rounds - 1);      // plain stream order: no dependent launch
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace gl
