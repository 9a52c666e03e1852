// TEST INFRASTRUCTURE: runs the GEMV lane program (gridllm_b200/csrc/rowdot.h) on the CPU so the
// layout / bit-twiddling logic can be checked against the oracle without a GPU.  Never linked
// into libgridllm_native.so.
#include <cmath>
#include <cstdio>
#include <vector>
#include "../../gridllm_b200/csrc/rowdot.h"
#include "../../gridllm_b200/csrc/gguf_file.h"

using namespace gl;

// activation planes exactly as the GPU prologue lays them out: hi [cols], lo [cols] (16-B chunk j of unit u at
// physical chunk j ^ (u & 7)), sx / sm [cols/32], s16 [cols/16]
template <int AB>
struct Planes {
    std::vector<uint8_t> raw;
    std::vector<float> sxv, smv;
    std::vector<int> s16v;
    uint8_t *hi, *lo;
    float *sx, *sm;
    int* s16;
    Planes(const float* x, int cols) : raw(2 * (size_t)cols + 64), sxv(cols / 32 + 8), smv(cols / 32 + 8), s16v(cols / 16 + 8) {
        hi = raw.data() + ((16 - ((uintptr_t)raw.data() & 15)) & 15);
        lo = hi + cols;
        sx = sxv.data() + ((16 - ((uintptr_t)sxv.data() & 15)) & 15) / 4;
        sm = smv.data() + ((16 - ((uintptr_t)smv.data() & 15)) & 15) / 4;
        s16 = s16v.data() + ((16 - ((uintptr_t)s16v.data() & 15)) & 15) / 4;
        for (int u = 0; u < cols / UNIT_COLS; ++u) {
            for (int b = 0; b < 4; ++b) {
                const float* xb = x + u * 128 + b * 32;
                float amax = 0.f;
                for (int i = 0; i < 32; ++i) amax = std::fmax(amax, std::fabs(xb[i]));
                uint32_t h[8], l[8];
                int s0, s1;
                snap16<AB>(xb, amax, h, l, &s0);
                snap16<AB>(xb + 16, amax, h + 4, l + 4, &s1);
                for (int v = 0; v < 2; ++v) {
                    const int j = 2 * b + v;
                    memcpy(hi + (size_t)u * 128 + ((j ^ (u & 7)) << 4), h + 4 * v, 16);
                    memcpy(lo + (size_t)u * 128 + ((j ^ (u & 7)) << 4), l + 4 * v, 16);
                }
                sx[4 * u + b] = amax / (AB == 16 ? ACT16_RANGE : ACT8_RANGE);
                sm[4 * u + b] = sx[4 * u + b] * (float)(s0 + s1);
                s16[8 * u + 2 * b] = s0;
                s16[8 * u + 2 * b + 1] = s1;
            }
        }
    }
};

// The consumer loop of gemv_core.cuh on the host: the matrix is stored in the engine layout with R-row tiles, a "slot"
// is filled the way the producer lane does it (one contiguous range per (item, K-segment)), lane l = unit l of the segment.
template <int AB, int R>
static int run_items(int type, const uint8_t* w, int rows, int cols, const float* x, float* y) {
    const KSplit ks = ksplit(cols);
    if (!ks.nks) return -2;
    Planes<AB> pl(x, cols);
    const int n = 2 * ks.seg_nb, sb = kseg_bytes(type, ks.seg_nb);
    const size_t rb = row_bytes(type, cols);
    std::vector<uint8_t> matbuf(engine_matrix_bytes(type, rows, cols, R) + 16, 0), slotbuf((size_t)R * sb + 16);
    uint8_t* mat = matbuf.data() + ((16 - ((uintptr_t)matbuf.data() & 15)) & 15);
    uint8_t* slot = slotbuf.data() + ((16 - ((uintptr_t)slotbuf.data() & 15)) & 15);
    for (int r = 0; r < rows; ++r) repack_row(type, w + (size_t)r * rb, mat, cols, R, r);
    const size_t tile_bytes = (size_t)R * ks.nks * sb;
    for (int i = 0, it = 0; i < rows; i += R, ++it) {
        const int nv = rows - i < R ? rows - i : R;
        float acc[R];
        for (int r = 0; r < R; ++r) acc[r] = 0.f;
        for (int k = 0; k < ks.nks; ++k) {
            memset(slot, 0xA5, (size_t)R * sb);                           // rows beyond the ragged end hold garbage on the GPU too
            memcpy(slot, mat + (size_t)it * tile_bytes + (size_t)k * R * sb, (size_t)nv * sb);      // = the producer's one bulk copy
            for (int l = 0; l < n; ++l) {
                const int ug = k * n + l;
                XPlanes xp{pl.hi + (size_t)ug * 128, pl.lo + (size_t)ug * 128, pl.sx + 4 * ug, pl.sm + 4 * ug, pl.s16 + 8 * ug, ug & 7};
                float part[R];
                for (int r = 0; r < R; ++r) part[r] = 0.f;
                if (type == T_Q4_K) item_dot_q4k<AB, R>(slot, sb, l, xp, part);
                else if (type == T_Q6_K) item_dot_q6k<AB, R>(slot, sb, n, l, xp, part);
                else item_dot_q80<AB, R>(slot, sb, n, l, xp, part);
                for (int r = 0; r < R; ++r) acc[r] += part[r];
            }
        }
        for (int r = 0; r < nv; ++r) y[i + r] = acc[r];
    }
    return 0;
}

// rows per item: 0 = what gemv_plan picks for the type (Q4_K 4, Q6_K / Q8_0 2); else 1, 2 or 4
extern "C" int hc_gemv_r(int type, const uint8_t* w, int rows, int cols, const float* x, float* y, int abits, int rpi) {
    if (type != T_Q4_K && type != T_Q6_K && type != T_Q8_0) return -1;
    if (!rpi) rpi = type == T_Q4_K ? 4 : 2;
    if (abits == 16) {
        if (rpi == 4) return run_items<16, 4>(type, w, rows, cols, x, y);
        if (rpi == 2) return run_items<16, 2>(type, w, rows, cols, x, y);
        return run_items<16, 1>(type, w, rows, cols, x, y);
    }
    if (rpi == 4) return run_items<8, 4>(type, w, rows, cols, x, y);
    if (rpi == 2) return run_items<8, 2>(type, w, rows, cols, x, y);
    return run_items<8, 1>(type, w, rows, cols, x, y);
}
extern "C" int hc_gemv(int type, const uint8_t* w, int rows, int cols, const float* x, float* y, int abits) {
    return hc_gemv_r(type, w, rows, cols, x, y, abits, 0);
}

// engine row layout round trip: GGUF rows -> engine rows -> element-wise dequantisation (what the batched prefill's
// 16-bit copy is built from)
extern "C" int hc_dequant_engine(int type, const uint8_t* w, int rows, int cols, int tile_rows, float* out) {
    if (!ksplit(cols).nks) return -2;
    const size_t rb = row_bytes(type, cols);
    std::vector<uint8_t> mat(engine_matrix_bytes(type, rows, cols, tile_rows), 0);
    for (int i = 0; i < rows; ++i) repack_row(type, w + (size_t)i * rb, mat.data(), cols, tile_rows, i);
    for (int i = 0; i < rows; ++i)
        for (int c = 0; c < cols; ++c) out[(size_t)i * cols + c] = dequant_engine_quant(mat.data(), type, cols, tile_rows, i, c);
    return 0;
}
extern "C" int hc_ksplit(int cols, int* nks, int* seg_nb) {
    const KSplit k = ksplit(cols);
    *nks = k.nks; *seg_nb = k.seg_nb;
    return k.nks ? 0 : -1;
}

// GGUF reader check: returns number of tensors or -1; fills a few fields
extern "C" int hc_gguf_probe(const char* path, char* arch, int cap, uint64_t* n_kv, uint64_t* total_bytes) {
    GGUFFile f;
    std::string err = f.open(path);
    if (!err.empty()) { snprintf(arch, cap, "%s", err.c_str()); return -1; }
    snprintf(arch, cap, "%s", f.get_s("general.architecture", "").c_str());
    *n_kv = f.kv.size();
    uint64_t tot = 0;
    for (auto& t : f.tensors) tot += t.nbytes;
    *total_bytes = tot;
    return (int)f.tensors.size();
}

// tokenizer (product code, gridllm_b200/csrc/tokenizer.cpp) driven from the CPU tests
#include "../../gridllm_b200/csrc/tokenizer.h"
extern "C" int hc_tokenize(const char* gguf_path, const char* text, int add_bos, int parse_special, int32_t* ids, int cap) {
    GGUFFile f;
    if (!f.open(gguf_path).empty()) return -1;
    Tokenizer t;
    if (!t.load(f)) return -2;
    std::vector<int32_t> v = t.encode(text, add_bos != 0, parse_special != 0);
    if ((int)v.size() > cap) return -3;
    for (size_t i = 0; i < v.size(); ++i) ids[i] = v[i];
    return (int)v.size();
}
// the pre-tokeniser alone: byte offsets of the piece ENDS
extern "C" int hc_pretokenize(const char* text, int n_bytes, int32_t* ends, int cap) {
    std::vector<std::string> v = llama3_pretokenize(std::string(text, (size_t)n_bytes));
    if ((int)v.size() > cap) return -3;
    int off = 0;
    for (size_t i = 0; i < v.size(); ++i) { off += (int)v[i].size(); ends[i] = off; }
    return (int)v.size();
}
extern "C" int hc_detokenize(const char* gguf_path, const int32_t* ids, int n, char* buf, int cap) {
    GGUFFile f;
    if (!f.open(gguf_path).empty()) return -1;
    Tokenizer t;
    if (!t.load(f)) return -2;
    std::string s = t.decode(ids, n);
    if ((int)s.size() >= cap) return -3;
    memcpy(buf, s.data(), s.size());
    buf[s.size()] = 0;
    return (int)s.size();
}

// ---- batched decode GEMM on quantised weights (qgemm_layout.h): pack 128 GGUF super-blocks into a qtile, run the kernel's
// per-thread dequantisation program for every (row, K-step) of the qtile and hand back the fp16 bit patterns [128 rows][256 columns]
// in column order (the kernel stores the same chunks into 128-byte-swizzled shared-memory operand tiles) -------------------------
#include "../../gridllm_b200/csrc/qgemm_layout.h"
extern "C" int hc_qg_dequant(int type, const uint8_t* blocks /*[128][block bytes]*/, uint16_t* out /*[128][256]*/, int* qtile_bytes) {
    if (!qg_type_ok(type)) return -1;
    const int bb = type == 12 ? 144 : 210;
    std::vector<uint8_t> qt((size_t)qg_qtile_bytes(type) + 64, 0xAB);     // poison: every byte must be written by the packer
    for (int r = 0; r < QG_ROWS; ++r) qg_pack_block(type, blocks + (size_t)r * bb, qt.data(), r);
    *qtile_bytes = qg_qtile_bytes(type);
    std::vector<int> written((size_t)QG_ROWS * QG_COLS / 8, 0);
    for (int kk = 0; kk < 4; ++kk)                                           // the kernel's unpack threads: (row, half) run K-steps 2 half, 2 half + 1
        for (int r = 0; r < QG_ROWS; ++r)
            qg_dequant_kstep(type, qt.data(), r, kk, [&](int c, QgU4 v) {
                // chunk c of K-step kk = columns 64kk + 8c .. +7 of row r: words in column order, two fp16 per word (low half first) --
                // exactly the 16 bytes the kernel stores at chunk position c ^ (r % 8) of row r in K-step kk's operand tile
                memcpy(out + (size_t)r * QG_COLS + 64 * kk + 8 * c, &v, 16);
                ++written[((size_t)r * QG_COLS + 64 * kk + 8 * c) / 8];
            });
    for (int w : written)
        if (w != 1) return -2;                                               // every chunk exactly once
    return 0;
}
