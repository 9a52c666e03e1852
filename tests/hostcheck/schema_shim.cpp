// TEST INFRASTRUCTURE: the schema compiler (gridllm_b200/csrc/schema_compile.cpp) and the automaton of the schema mask kernel
// (gridllm_b200/csrc/schema_fsm.h) compiled for the host, so that tests/test_schema_cpu.py can compare them with
// tests/schema_oracle.py.  Never linked into libgridllm_native.so.
#include <cstring>
#include <string>
#include <vector>

#include "../../gridllm_b200/csrc/schema_fsm.h"

using namespace gl;

namespace {
thread_local std::string g_err;
}

extern "C" {

int sf_state_bytes() { return (int)sizeof(SchemaState); }

const char* sf_error() { return g_err.c_str(); }

// compiles schema[0..n) into blob (cap bytes); returns GL_OK or the error code (message: sf_error), *blob_len = its size
int sf_compile(const char* schema, int n, unsigned char* blob, int cap, int* blob_len) {
    std::vector<uint8_t> b;
    const int rc = schema_compile(schema, (size_t)n, b, g_err);
    *blob_len = (int)b.size();
    if (rc == 0 && (int)b.size() <= cap) std::memcpy(blob, b.data(), b.size());
    return rc;
}

// runs p[0..n) from the initial state: returns the bytes accepted (n when all were), *done = the document is complete there
int sf_run(const unsigned char* blob, const unsigned char* p, int n, int* done) {
    const SchemaView v = schema_view(blob);
    SchemaState s;
    schema_init(s.js, s.cur, v);
    SchemaArrayFrames fr{s.fr};
    int i = 0;
    for (; i < n; ++i)
        if (!schema_step(v, s.js, s.cur, fr, p[i])) break;
    if (done) *done = schema_done(s.js) ? 1 : 0;
    return i;
}

// for each of the m pieces (offsets[0..m]): 1 when it is accepted whole after the prefix p[0..n) (which must be accepted);
// returns -1 when the prefix is not
int sf_allowed(const unsigned char* blob, const unsigned char* p, int n, const unsigned char* pieces, const int* offsets, int m,
               unsigned char* out) {
    const SchemaView v = schema_view(blob);
    SchemaState s;
    schema_init(s.js, s.cur, v);
    SchemaArrayFrames fr{s.fr};
    if (!schema_run(v, s.js, s.cur, fr, p, n)) return -1;
    for (int k = 0; k < m; ++k) {
        SchemaState t = s;
        SchemaArrayFrames tf{t.fr};
        out[k] = schema_run(v, t.js, t.cur, tf, pieces + offsets[k], offsets[k + 1] - offsets[k]) ? 1 : 0;
    }
    return schema_done(s.js) ? 1 : 0;
}

}
