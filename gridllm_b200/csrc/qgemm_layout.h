// Layout and dequantisation arithmetic of the batched decode GEMM on QUANTISED weights (qgemm.cu): the weights are read from
// HBM once per batched step in their GGUF bit budget (Q4_K 4.5, Q6_K 6.5625 bits / weight) and turned into fp16 tensor-core
// operands tile by tile inside the kernel.  Everything here is __host__ __device__ so that tests/hostcheck runs the exact
// per-thread program on the CPU (pack -> dequantise -> un-swizzle must reproduce the GGUF values), as rowdot.h does for the
// decode GEMV.  Reference side: the decode loop inside Ollama behind OllamaService.generate*Response
// (/root/reference/client/src/services/OllamaService.ts:142-145, 235-237) when several requests share a step.
//
// Vocabulary
//   qtile  : 128 weight rows x 256 columns (one K-quant super-block per row) -- the unit of work of the kernel, ONE contiguous
//            byte range in HBM (one 1-D TMA bulk copy): 18 432 B (Q4_K) / 26 880 B (Q6_K), exactly the GGUF bytes of those blocks
//   plane  : inside a qtile the fields of the 128 super-blocks are regrouped into planes of [128 rows][16 B], so that the 32
//            lanes of a warp (32 consecutive rows) read 512 contiguous bytes per 128-bit load -- no bank conflicts, no 2-byte
//            aligned 210-byte records
//   K-step : 64 columns = one wgmma A operand [128 rows x 64] fp16 in shared memory (128-byte swizzle), written by the unpack
//            warps; a qtile is 4 K-steps
//   chunk  : 8 consecutive columns of one row = four packed half2 words
//
// QG layouts (a lossless permutation of the GGUF bits; pack_block() below is the definition):
//   Q4_K qtile : [hdr  : 128 x 16 B]  d, dmin, scales[12] of each row's block, verbatim
//                [qs_j : 128 x 16 B, j = 0..7]  the 32 nibbles of sub-block j (columns 32j..32j+31): four 32-bit words, word t
//                                   = columns 32j+8t..+7, column i of the eight at nibble position NIB_POS[i]
//   Q6_K qtile : [lo_j : 128 x 16 B, j = 0..7]  low nibbles of columns 32j..32j+31, same word / nibble order
//                [hi_k : 128 x 16 B, k = 0..3]  the 2 high bits of columns 64k..64k+63: four 32-bit words, word u = columns
//                                   64k+16u..+15; of a pair of columns (2p, 2p+1) the first lives in the low 16-bit half, the
//                                   second in the high half, at bit qg_q6k_hi_pos(second eight?, p) -- see there
//                [sc   : 128 x 16 B]  int8 scales[16], verbatim       [d : 128 x 2 B]
//   NIB_POS = {0, 4, 1, 5, 2, 6, 3, 7}: columns (2p, 2p+1) are the same nibble of the word's two 16-bit halves -- one logic op
//   away from a half2 via the exponent trick (1024 + q, or 64 + q for a nibble at bits 4..7, is exact in fp16).
//
// Dequantised value (what the tensor core multiplies), in fp16 arithmetic with one rounding per step:
//   Q4_K : w = fma(q, s, -m),  s = fp16(d * sc), m = fp16(dmin * mn)         (GGUF: d*sc*q - dmin*mn)
//   Q6_K : w = (q - 32) * s,   s = fp16(d * sc)                             (GGUF: d*sc*(q-32))
#pragma once
#include <stdint.h>
#include <string.h>

#include "rowdot.h"
#if defined(__CUDACC__)
#include <cuda_fp16.h>
// the dequantisation program is device code under nvcc and plain host code under g++ (tests/hostcheck)
#define QG_FN __device__ __forceinline__
#else
#define QG_FN inline
#endif

namespace gl {

constexpr int QG_ROWS = 128;                 // weight rows of a qtile = M of the MMA
constexpr int QG_COLS = 256;                 // columns of a qtile = one super-block
constexpr int QG_KSTEP = 64;                 // columns of one operand tile
constexpr int QG_PLANE = QG_ROWS * 16;       // bytes of one plane
constexpr int QG_Q4K_BYTES = 9 * QG_PLANE;                       // 18 432
constexpr int QG_Q6K_BYTES = 13 * QG_PLANE + QG_ROWS * 2;        // 26 880

GL_HD int qg_qtile_bytes(int type) { return type == 12 ? QG_Q4K_BYTES : type == 14 ? QG_Q6K_BYTES : 0; }
GL_HD bool qg_type_ok(int type) { return type == 12 || type == 14; }

// nibble position of column i (0..7) inside a 32-bit word
GL_HD int qg_nib_pos(int i) { return (i >> 1) + 4 * (i & 1); }

// Q6_K high bits: bit position (inside its 16-bit half) of the 2-bit field of pair p of the FIRST (A) / SECOND (B) eight columns
// of a 16-column hi word.  A's fields sit where the exponent trick wants them ([4,5] under 1024, [8,9] under 64) or two bits
// above (pairs 2, 3: one shared >> 2); B's take the remaining bits and one shift each.
GL_HD int qg_q6k_hi_pos(int second_eight, int p) {
    return second_eight ? (p == 0 ? 12 : p == 1 ? 14 : p == 2 ? 0 : 2) : (p == 0 ? 4 : p == 1 ? 8 : p == 2 ? 6 : 10);
}

// ---- load time (device kernel in qgemm.cu; the host check runs the same code): one GGUF super-block of tile row r -> its
// 16-byte words in the planes of the qtile image.  Every (row, plane) word is written exactly once, by the thread that owns the row.
GL_HD void qg_store_word(uint8_t* dst, const uint32_t w[4]) {
    *reinterpret_cast<uint32_t*>(dst) = w[0];
    *reinterpret_cast<uint32_t*>(dst + 4) = w[1];
    *reinterpret_cast<uint32_t*>(dst + 8) = w[2];
    *reinterpret_cast<uint32_t*>(dst + 12) = w[3];
}

GL_HD void qg_pack_block(int type, const uint8_t* blk, uint8_t* qtile, int r) {
    if (type == 12) {                                                      // Q4_K: d dmin scales[12] qs[128]
        for (int i = 0; i < 16; ++i) qtile[r * 16 + i] = blk[i];
        for (int j = 0; j < 8; ++j) {                                      // sub-block j = columns 32j..32j+31
            uint32_t w[4] = {0, 0, 0, 0};
            for (int cc = 0; cc < 32; ++cc) {
                const int c = 32 * j + cc, g = c >> 6, in = c & 63;
                const uint8_t b = blk[16 + 32 * g + (in & 31)];
                const uint32_t q = in < 32 ? (uint32_t)(b & 0xF) : (uint32_t)(b >> 4);
                w[cc >> 3] |= q << (4 * qg_nib_pos(cc & 7));
            }
            qg_store_word(qtile + (1 + j) * QG_PLANE + r * 16, w);
        }
    } else {                                                               // Q6_K: ql[128] qh[64] scales[16] d
        for (int j = 0; j < 8; ++j) {
            uint32_t w[4] = {0, 0, 0, 0};
            for (int cc = 0; cc < 32; ++cc) {
                const int e = 32 * j + cc, h = e >> 7, rr = e & 127;
                const uint32_t ql = (uint32_t)(blk[h * 64 + (rr & 63)] >> (4 * (rr >> 6))) & 0xFu;
                w[cc >> 3] |= ql << (4 * qg_nib_pos(cc & 7));
            }
            qg_store_word(qtile + j * QG_PLANE + r * 16, w);
        }
        for (int k = 0; k < 4; ++k) {                                      // high bits of columns 64k..64k+63
            uint32_t w[4] = {0, 0, 0, 0};
            for (int cc = 0; cc < 64; ++cc) {
                const int e = 64 * k + cc, h = e >> 7, rr = e & 127;
                const uint32_t qh = (uint32_t)(blk[128 + h * 32 + (rr & 31)] >> (2 * (rr >> 5))) & 3u;
                // word cc/16; first / second eight columns of its sixteen; pair p = (cc%8)/2; the pair's first column in the low
                // 16-bit half, its second in the high half (like the nibbles)
                const int i = cc & 7;
                w[cc >> 4] |= qh << (16 * (i & 1) + qg_q6k_hi_pos((cc & 15) >> 3, i >> 1));
            }
            qg_store_word(qtile + (8 + k) * QG_PLANE + r * 16, w);
        }
        for (int i = 0; i < 16; ++i) qtile[12 * QG_PLANE + r * 16 + i] = blk[192 + i];
        qtile[13 * QG_PLANE + r * 2] = blk[208];
        qtile[13 * QG_PLANE + r * 2 + 1] = blk[209];
    }
}

// ---- fp16 pair arithmetic: device intrinsics, or an exact emulation on the host (one rounding per operation) -----------------
#if defined(__CUDACC__)
struct QH2 { __half2 v; };
QG_FN QH2 qh2_bits(uint32_t b) { QH2 r; r.v = *reinterpret_cast<__half2*>(&b); return r; }
QG_FN uint32_t qh2_to_bits(QH2 a) { return *reinterpret_cast<uint32_t*>(&a.v); }
QG_FN QH2 qh2_set(float x) { QH2 r; r.v = __float2half2_rn(x); return r; }
QG_FN QH2 qh2_sub(QH2 a, QH2 b) { QH2 r; r.v = __hsub2(a.v, b.v); return r; }
QG_FN QH2 qh2_mul(QH2 a, QH2 b) { QH2 r; r.v = __hmul2(a.v, b.v); return r; }
QG_FN QH2 qh2_fma(QH2 a, QH2 b, QH2 c) { QH2 r; r.v = __hfma2(a.v, b.v, c.v); return r; }
#else
struct QH2 { _Float16 lo, hi; };
inline QH2 qh2_bits(uint32_t b) { QH2 r; uint16_t l = (uint16_t)b, h = (uint16_t)(b >> 16); memcpy(&r.lo, &l, 2); memcpy(&r.hi, &h, 2); return r; }
inline uint32_t qh2_to_bits(QH2 a) { uint16_t l, h; memcpy(&l, &a.lo, 2); memcpy(&h, &a.hi, 2); return (uint32_t)l | ((uint32_t)h << 16); }
inline QH2 qh2_set(float x) { QH2 r; r.lo = r.hi = (_Float16)x; return r; }
inline QH2 qh2_sub(QH2 a, QH2 b) { QH2 r; r.lo = (_Float16)((float)a.lo - (float)b.lo); r.hi = (_Float16)((float)a.hi - (float)b.hi); return r; }
inline QH2 qh2_mul(QH2 a, QH2 b) { QH2 r; r.lo = (_Float16)((float)a.lo * (float)b.lo); r.hi = (_Float16)((float)a.hi * (float)b.hi); return r; }
// the exact product-sum of three fp16 values fits a double: one rounding, like the hardware fma
inline QH2 qh2_fma(QH2 a, QH2 b, QH2 c) {
    QH2 r;
    r.lo = (_Float16)((double)a.lo * (double)b.lo + (double)c.lo);
    r.hi = (_Float16)((double)a.hi * (double)b.hi + (double)c.hi);
    return r;
}
#endif

// The exponent trick: OR-ing a small integer into the mantissa of a suitable fp16 constant gives base + integer EXACTLY --
//   bits [0, 6) under 0x6400 (1024.0, one unit per mantissa step):  1024 + q
//   bits [4, 10) under 0x5400 (64.0, 1/16 per mantissa step):         64 + (bits >> 4)
// so the nibble at bits 4..7 of a word needs no shift, and a word of eight nibbles costs ONE shift (>> 8) and four logic ops.
constexpr uint32_t QG_MAGIC = 0x64006400u, QG_MAGIC_HI = 0x54005400u;
constexpr uint32_t QG_NIB_LO = 0x000F000Fu, QG_NIB_HI = 0x00F000F0u;

// (a & b) | c  and  a | (b & c): one LOP3 each on the device (written as separate & and | the compiler emits two when both
// constants are immediates; the unpack warps are bound by exactly this pipe)
#if defined(__CUDACC__)
QG_FN uint32_t qg_and_or(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
QG_FN uint32_t qg_or_and(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xF8;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
#else
inline uint32_t qg_and_or(uint32_t a, uint32_t b, uint32_t c) { return (a & b) | c; }
inline uint32_t qg_or_and(uint32_t a, uint32_t b, uint32_t c) { return a | (b & c); }
#endif

// Q4_K scale / min of sub-block j from the three scale words (bytes 0..3, 4..7, 8..11 of scales[12])
GL_HD void qg_q4k_scale_min(int j, uint32_t s0, uint32_t s1, uint32_t s2, int& sc, int& mn) {
    if (j < 4) {
        sc = (int)((s0 >> (8 * j)) & 63);
        mn = (int)((s1 >> (8 * j)) & 63);
    } else {
        const int k = j - 4;
        sc = (int)(((s2 >> (8 * k)) & 0xF) | (((s0 >> (8 * k + 6)) & 3) << 4));
        mn = (int)(((s2 >> (8 * k + 4)) & 0xF) | (((s1 >> (8 * k + 6)) & 3) << 4));
    }
}

// One 32-bit word of eight Q4_K nibbles -> four half2 (columns 0-1, 2-3, 4-5, 6-7): fma(q, s, -m).
// 1 shift + 4 logic ops (alu pipe), 4 subtractions + 4 fma (fma pipe) for eight weights.
QG_FN void qg_q4k_word(uint32_t w, QH2 s2, QH2 nm2, uint32_t out[4]) {
    const QH2 k1024 = qh2_bits(QG_MAGIC), k64 = qh2_bits(QG_MAGIC_HI);
    const uint32_t w8 = w >> 8;
    out[0] = qh2_to_bits(qh2_fma(qh2_sub(qh2_bits(qg_and_or(w, QG_NIB_LO, QG_MAGIC)), k1024), s2, nm2));
    out[1] = qh2_to_bits(qh2_fma(qh2_sub(qh2_bits(qg_and_or(w, QG_NIB_HI, QG_MAGIC_HI)), k64), s2, nm2));
    out[2] = qh2_to_bits(qh2_fma(qh2_sub(qh2_bits(qg_and_or(w8, QG_NIB_LO, QG_MAGIC)), k1024), s2, nm2));
    out[3] = qh2_to_bits(qh2_fma(qh2_sub(qh2_bits(qg_and_or(w8, QG_NIB_HI, QG_MAGIC_HI)), k64), s2, nm2));
}

// One 32-bit word of eight Q6_K low nibbles + the hi word of its 16-column group -> four half2: (q - 32) * s
// (the eight columns are one half of a 16-column sub-block: one scale)
template <int SECOND>
QG_FN void qg_q6k_word(uint32_t lo, uint32_t hw, QH2 s2, uint32_t out[4]) {
    const QH2 k1056 = qh2_bits(0x64206420u), k96 = qh2_bits(0x56005600u);      // 1024 + 32, 64 + 32
    const uint32_t lo8 = lo >> 8;
    uint32_t h0, h1, h2, h3;
    if (SECOND) { h0 = hw >> 8; h1 = hw >> 6; h2 = hw << 4; h3 = hw << 6; }
    else { h0 = hw; h1 = hw; h2 = hw >> 2; h3 = h2; }
    const uint32_t q0 = qg_or_and(qg_and_or(lo, QG_NIB_LO, QG_MAGIC), h0, 0x00300030u);
    const uint32_t q1 = qg_or_and(qg_and_or(lo, QG_NIB_HI, QG_MAGIC_HI), h1, 0x03000300u);
    const uint32_t q2 = qg_or_and(qg_and_or(lo8, QG_NIB_LO, QG_MAGIC), h2, 0x00300030u);
    const uint32_t q3 = qg_or_and(qg_and_or(lo8, QG_NIB_HI, QG_MAGIC_HI), h3, 0x03000300u);
    out[0] = qh2_to_bits(qh2_mul(qh2_sub(qh2_bits(q0), k1056), s2));
    out[1] = qh2_to_bits(qh2_mul(qh2_sub(qh2_bits(q1), k96), s2));
    out[2] = qh2_to_bits(qh2_mul(qh2_sub(qh2_bits(q2), k1056), s2));
    out[3] = qh2_to_bits(qh2_mul(qh2_sub(qh2_bits(q3), k96), s2));
}

struct QgU4 { uint32_t x, y, z, w; };

// 128-bit loads of the program: SHARED-memory instructions on the device (the kernel only ever passes shared-memory pointers; a
// generic-address load would cost an address-space lookup per access), plain memory on the host
#if defined(__CUDACC__)
QG_FN QgU4 qg_ld128(const uint8_t* p) {
    QgU4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"((uint32_t)__cvta_generic_to_shared(p)));
    return v;
}
QG_FN uint16_t qg_ld16(const uint8_t* p) {
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)));
    return v;
}
#else
QG_FN QgU4 qg_ld128(const uint8_t* p) { QgU4 v; memcpy(&v, p, 16); return v; }
QG_FN uint16_t qg_ld16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }
#endif

// ---- the per-thread program of the kernel's unpack warps -------------------------------------------------------------------
// Thread (row r, K-step kk) turns columns 64kk..64kk+63 of row r's super-block into 8 chunks of 8 fp16 (four packed half2 words
// each) and hands them to `store(c, words)`, c = 0..7 in column order.  The kernel collects the 32 words in registers and writes
// them to shared memory (the A operand of the MMA: row r, fp16 columns in order); the host check writes them to a plain array.
// `raw` is the qtile image (shared memory on the device).
template <typename StoreChunk>
QG_FN void qg_dequant_kstep(int type, const uint8_t* raw, int r, int kk, StoreChunk store) {
    if (type == 12) {
        const QgU4 hdr = qg_ld128(raw + r * 16);
        const float d = half_bits_to_float((uint16_t)(hdr.x & 0xFFFF)), dmin = half_bits_to_float((uint16_t)(hdr.x >> 16));
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int j = 2 * kk + jj;                                                  // sub-block of 32 columns
            int sc, mn;
            qg_q4k_scale_min(j, hdr.y, hdr.z, hdr.w, sc, mn);
            const QH2 s2 = qh2_set(d * (float)sc), nm2 = qh2_set(-(dmin * (float)mn));
            const QgU4 q = qg_ld128(raw + (1 + j) * QG_PLANE + r * 16);
            const uint32_t words[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                uint32_t o[4];
                qg_q4k_word(words[t], s2, nm2, o);
                store(jj * 4 + t, QgU4{o[0], o[1], o[2], o[3]});
            }
        }
    } else {
        const QgU4 scw = qg_ld128(raw + 12 * QG_PLANE + r * 16);
        // the four scales of this K-step (16-column sub-blocks 4kk..4kk+3) are ONE word of the row's sixteen: picked by kk with
        // selects, then indexed by compile-time constants only (an array indexed at run time would live in local memory)
        const uint32_t sc4 = kk == 0 ? scw.x : kk == 1 ? scw.y : kk == 2 ? scw.z : scw.w;
        const float d = half_bits_to_float(qg_ld16(raw + 13 * QG_PLANE + r * 2));
        const QgU4 hq = qg_ld128(raw + (8 + kk) * QG_PLANE + r * 16);                   // high bits of columns 64kk..64kk+63
        const uint32_t hwords[4] = {hq.x, hq.y, hq.z, hq.w};
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int j = 2 * kk + jj;                                                  // 32-column group
            const QgU4 q = qg_ld128(raw + j * QG_PLANE + r * 16);
            const uint32_t words[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                // columns 32j + 8t .. +7: 16-column sub-block 4kk + 2jj + t/2 (byte 2jj + t/2 of sc4), high bits in half-word t & 1
                // of word 2jj + t/2
                const int sc = (int)(int8_t)((sc4 >> (8 * (2 * jj + (t >> 1)))) & 0xFF);
                const QH2 s2 = qh2_set(d * (float)sc);
                const uint32_t hw = hwords[2 * jj + (t >> 1)];
                uint32_t o[4];
                if (t & 1) qg_q6k_word<1>(words[t], hw, s2, o);
                else qg_q6k_word<0>(words[t], hw, s2, o);
                store(jj * 4 + t, QgU4{o[0], o[1], o[2], o[3]});
            }
        }
    }
}

}  // namespace gl
