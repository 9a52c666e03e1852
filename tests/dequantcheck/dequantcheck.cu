// Test-only shim: the library's 16-bit operand dequantisation (dequant_launch, prefill.cu) against a reference kernel that
// dequantises one element per thread through the element accessors of rowdot.h -- the arithmetic every earlier resident copy
// was built with -- on one GGUF matrix.  Not part of the C ABI of libgridllm_native.so.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "prefill.h"
#include "rowdot.h"

using namespace gl;

namespace {

constexpr int F32 = 0, F16 = 1, Q8_0 = 8, Q4_K = 12, Q6_K = 14, BF16 = 30;

template <typename T> __device__ T to16(float v);
template <> __device__ __half to16<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __nv_bfloat16 to16<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void ref_kernel(const uint8_t* mat, int type, int rows, int cols, int row_stride, int tile_rows, T* dst, int dst_row0, int interleave) {
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
        int dr = r;
        if (interleave == 1) dr = (r >> 3) * 16 + (r & 7);
        else if (interleave == 2) dr = (r >> 3) * 16 + 8 + (r & 7);
        const uint8_t* row = mat + (size_t)r * row_stride;
        for (int c = threadIdx.x; c < cols; c += blockDim.x) {
            float v;
            if (type == F32) v = reinterpret_cast<const float*>(row)[c];
            else if (type == F16) v = __half2float(reinterpret_cast<const __half*>(row)[c]);
            else if (type == BF16) v = __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(row)[c] << 16);
            else v = dequant_engine_quant(mat, type, cols, tile_rows, r, c);
            dst[(size_t)(dst_row0 + dr) * cols + c] = to16<T>(v);
        }
    }
}

size_t gguf_row_bytes(int type, int cols) {
    switch (type) {
        case F32: return (size_t)cols * 4;
        case F16: case BF16: return (size_t)cols * 2;
        default: return (size_t)(cols / 256) * (type == Q8_0 ? 272 : quant_block_bytes(type));
    }
}

}  // namespace

extern "C" {

// One GGUF matrix [rows][cols] of `type` (host rows), stored in the engine layout with tile_rows (quantised types) or as plain
// 16-byte-aligned rows; both kernels write it to row dst_row0 on (interleave as in DequantSrc) of a [dst_rows][cols] 16-bit
// matrix whose untouched elements keep 0xFFFF.  out_new / out_ref: [dst_rows][cols] uint16.  Returns the cudaError_t.
int dq_check(int type, const uint8_t* gguf, int rows, int cols, int tile_rows, int dst_rows, int dst_row0, int interleave, int bf16,
             uint16_t* out_new, uint16_t* out_ref) {
    const bool quant = type == Q4_K || type == Q6_K || type == Q8_0;
    const size_t rb = gguf_row_bytes(type, cols);
    std::vector<uint8_t> mat;
    int row_stride = 0;
    if (quant) {
        mat.assign(engine_matrix_bytes(type, rows, cols, tile_rows), 0);
        for (int r = 0; r < rows; ++r) repack_row(type, gguf + (size_t)r * rb, mat.data(), cols, tile_rows, r);
    } else {
        row_stride = (int)align16(rb);
        tile_rows = 1;
        mat.assign((size_t)row_stride * rows, 0);
        for (int r = 0; r < rows; ++r) memcpy(mat.data() + (size_t)r * row_stride, gguf + (size_t)r * rb, rb);
    }
    uint8_t* dm = nullptr;
    uint16_t *dn = nullptr, *dr = nullptr;
    const size_t out_bytes = (size_t)dst_rows * cols * 2;
    cudaError_t e = cudaMalloc(&dm, mat.size());
    if (e == cudaSuccess) e = cudaMalloc(&dn, out_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dr, out_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(dm, mat.data(), mat.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(dn, 0xFF, out_bytes);
    if (e == cudaSuccess) e = cudaMemset(dr, 0xFF, out_bytes);
    if (e == cudaSuccess) {
        DequantOp op{};
        op.src[0] = DequantSrc{dm, type, rows, row_stride, tile_rows, dst_row0, interleave};
        op.n_src = 1; op.cols = cols; op.dst = dn;
        e = dequant_launch(op, bf16 != 0, 0);
    }
    if (e == cudaSuccess) {
        if (bf16) ref_kernel<__nv_bfloat16><<<256, 256>>>(dm, type, rows, cols, row_stride, tile_rows, (__nv_bfloat16*)dr, dst_row0, interleave);
        else ref_kernel<__half><<<256, 256>>>(dm, type, rows, cols, row_stride, tile_rows, (__half*)dr, dst_row0, interleave);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out_new, dn, out_bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(out_ref, dr, out_bytes, cudaMemcpyDeviceToHost);
    cudaFree(dm); cudaFree(dn); cudaFree(dr);
    return (int)e;
}

}
