// Context shift (gl_engine_opts context_shift; rule in include/gridllm_native.h): what a request keeps, what a shift discards
// and how an over-long prompt is cut.  Host only and self-contained, so that the CPU suite can compile and test it on its own
// (tests/hostcheck/shift_shim.cpp).
#pragma once
#include <stdint.h>

namespace gl {

// the keep count k of a request in a context of W positions: num_keep >= 0 clamped to W - 1, -1 the whole prompt (clamped
// likewise).  The caller has refused num_keep < -1.
inline int shift_keep(int num_keep, int n_prompt, int W) {
    const int k = num_keep < 0 ? n_prompt : num_keep;
    return k < W - 1 ? k : W - 1;
}

// positions dropped by one shift: d = ceil((W - k) / 2), >= 1 since k <= W - 1
inline int shift_discard(int W, int k) { return (W - k + 1) / 2; }

// rows a shift moves: [k + d, W) -> [k, W - d)
inline int shift_rows(int W, int k, int d) { return W - k - d; }

// a prompt of n_prompt >= W ids: its first k ids, then its newest W - d - k ids (the positions a shift would leave).  out holds
// W - d ids; returns that length.  A shorter prompt is copied as it is.
inline int cut_prompt(const int32_t* prompt, int n_prompt, int W, int k, int d, int32_t* out) {
    if (n_prompt < W) {
        for (int i = 0; i < n_prompt; ++i) out[i] = prompt[i];
        return n_prompt;
    }
    const int tail = W - d - k;
    for (int i = 0; i < k; ++i) out[i] = prompt[i];
    for (int i = 0; i < tail; ++i) out[k + i] = prompt[n_prompt - tail + i];
    return W - d;
}

// decode steps a chunk of gl_generate may run: each writes the row at the current position, so a chunk ends at the window
// (pos: the position the chunk's first step writes; one extra draw when the chunk starts with the head alone)
inline int shift_chunk(int chunk, int remaining, int pos, int W, bool head_only_first) {
    int n = chunk < remaining ? chunk : remaining;
    const int room = W - pos + (head_only_first ? 1 : 0);
    return n < room ? n : room;
}

}  // namespace gl
