// TEST INFRASTRUCTURE: the JSON automaton of the mask kernel (gridllm_b200/csrc/json_fsm.h) compiled for the host, so that
// tests/test_json_cpu.py can compare it with tests/json_oracle.py state for state.  Never linked into libgridllm_native.so.
#include <cstring>

#include "../../gridllm_b200/csrc/json_fsm.h"

using namespace gl;

extern "C" {

int jf_state_bytes() { return (int)sizeof(JsonState); }

// Runs p[0..n) from the initial state.  states[16 * i ..] = the state after byte i, for every accepted byte.  Returns the number of
// bytes accepted (n when all were); *done = json_done of the last accepted state.
int jf_trace(const unsigned char* p, int n, unsigned char* states, int* done) {
    JsonState s{};
    int i = 0;
    for (; i < n; ++i) {
        if (!json_step(s, p[i])) break;
        if (states) std::memcpy(states + 16 * (size_t)i, &s, 16);
    }
    if (done) *done = json_done(s) ? 1 : 0;
    return i;
}

}
