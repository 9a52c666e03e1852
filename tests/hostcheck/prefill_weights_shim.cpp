// TEST INFRASTRUCTURE: the prompt-pass weight rule (gridllm_b200/csrc/prefill_weights.h) compiled for the host, so that
// tests/test_prefill_weights_cpu.py can check it.  Never linked into libgridllm_native.so.
#include "../../gridllm_b200/csrc/prefill_weights.h"

extern "C" {

uint64_t pw_copy_bytes(int n_layer, int n_embd, int n_head, int n_kv, int hd, int n_ff) { return gl::prefill_copy_bytes(n_layer, n_embd, n_head, n_kv, hd, n_ff); }
uint64_t pw_stage_bytes(int n_embd, int n_head, int n_kv, int hd, int n_ff) { return gl::prefill_stage_bytes(n_embd, n_head, n_kv, hd, n_ff); }
int pw_source(int prefill_mode, int request, uint64_t copy_bytes, uint64_t free_bytes) { return gl::prefill_weights_source(prefill_mode, request, copy_bytes, free_bytes); }
uint64_t pw_margin() { return gl::PREFILL_COPY_MARGIN; }

}
