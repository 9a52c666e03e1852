// TEST INFRASTRUCTURE: gl_generate's prefix reuse rule (gridllm_b200/csrc/prefix_reuse.h) compiled for the host, so that
// tests/test_prefix_prefill_cpu.py can check it.  Never linked into libgridllm_native.so.
#include "../../gridllm_b200/csrc/prefix_reuse.h"

extern "C" {

int pr_reuse(const int32_t* prompt, int n_prompt, const int32_t* cached, int n_cached, int min_suffix) {
    return gl::prefix_reuse(prompt, n_prompt, cached, n_cached, min_suffix);
}

}
