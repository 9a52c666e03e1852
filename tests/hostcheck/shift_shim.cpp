// TEST INFRASTRUCTURE: the context-shift rule (gridllm_b200/csrc/context_shift.h) compiled for the host, so that
// tests/test_context_shift_cpu.py can check it.  Never linked into libgridllm_native.so.
#include "../../gridllm_b200/csrc/context_shift.h"

extern "C" {

int cs_keep(int num_keep, int n_prompt, int W) { return gl::shift_keep(num_keep, n_prompt, W); }
int cs_discard(int W, int k) { return gl::shift_discard(W, k); }
int cs_rows(int W, int k, int d) { return gl::shift_rows(W, k, d); }
int cs_cut(const int32_t* prompt, int n_prompt, int W, int k, int d, int32_t* out) { return gl::cut_prompt(prompt, n_prompt, W, k, d, out); }
int cs_chunk(int chunk, int remaining, int pos, int W, int head_only_first) { return gl::shift_chunk(chunk, remaining, pos, W, head_only_first != 0); }

}
