// extern "C" surface of libgridllm_native.so -- see include/gridllm_native.h for the reference
// call site each entry point stands in for.
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <cstring>
#include <new>
#include <stdexcept>
#include <string>

#include "../../include/gridllm_native.h"
#include "engine.h"

using gl::Engine;
using gl::Status;

struct gl_engine {
    Engine* impl;
};

namespace {
int ret(const Status& s) {
    if (!s.ok()) gl::set_last_error(s.msg);
    return s.code;
}
int bad(const char* m) {
    gl::set_last_error(m);
    return GL_ERR_INVALID;
}

// The penalty fields took the place of six reserved words: the struct's size and the offsets of the older fields are what
// hosts built against ABI version 2 lay out (a caller that zeroes `reserved` gets no penalty and no min_p).
static_assert(sizeof(gl_sample_opts) == 72, "gl_sample_opts size is part of the ABI");
static_assert(offsetof(gl_sample_opts, seed) == 16 && offsetof(gl_sample_opts, stop_ids) == 32 &&
                  offsetof(gl_sample_opts, want_logits) == 40, "gl_sample_opts offsets are part of the ABI");
static_assert(offsetof(gl_sample_opts, repeat_penalty) == 44 && offsetof(gl_sample_opts, min_p) == 60 &&
                  offsetof(gl_sample_opts, reserved) == 64, "penalty fields sit where reserved[0..5] was");

// the penalty / min_p fields of a request (include/gridllm_native.h); nullptr when valid
const char* check_penalties(const gl_sample_opts& so) {
    if (!std::isfinite(so.repeat_penalty) || !std::isfinite(so.presence_penalty) || !std::isfinite(so.frequency_penalty) ||
        !std::isfinite(so.min_p))
        return "repeat_penalty, presence_penalty, frequency_penalty and min_p must be finite";
    if (so.repeat_penalty < 0.f) return "repeat_penalty must be >= 0";
    if (so.repeat_last_n < -1) return "repeat_last_n must be >= -1";
    if (so.min_p < 0.f || so.min_p > 1.f) return "min_p must lie in [0, 1]";
    return nullptr;
}

// format took the place of the last reserved word (an anonymous union keeps `reserved` addressable): a zeroed word is "off"
static_assert(offsetof(gl_sample_opts, format) == 64, "format sits where reserved[0] was");

// prefix_cache took the place of gl_engine_opts.reserved[0]: the size and the older offsets are unchanged, a zeroed word is "off"
static_assert(sizeof(gl_engine_opts) == 64, "gl_engine_opts size is part of the ABI");
static_assert(offsetof(gl_engine_opts, batch_weights) == 28 && offsetof(gl_engine_opts, prefix_cache) == 32 &&
                  offsetof(gl_engine_opts, reserved) == 36, "prefix_cache sits where reserved[0] was");
// batch_prefix_cache is the first of the remaining reserved words (gl_engine_opts.reserved[GL_OPT_BATCH_PREFIX_CACHE]), at offset 36
static_assert(GL_OPT_BATCH_PREFIX_CACHE == 0 && sizeof(gl_engine_opts) == 64, "batch_prefix_cache sits in reserved[0]");
// context_shift is reserved[GL_OPT_CONTEXT_SHIFT], at offset 40; num_keep took the tail padding of gl_sample_opts (offset 68, the
// size unchanged), which is why the engine reads it only when context_shift is on
static_assert(GL_OPT_CONTEXT_SHIFT == 1 && offsetof(gl_engine_opts, reserved) + 4 * GL_OPT_CONTEXT_SHIFT == 40, "context_shift sits in reserved[1]");
static_assert(offsetof(gl_sample_opts, num_keep) == 68 && sizeof(gl_sample_opts) == 72, "num_keep sits in the tail padding");

// the format field of a generating request; nullptr when valid
const char* check_format(const gl_sample_opts& so) {
    if (so.format != 0 && so.format != GL_FORMAT_JSON && so.format < GL_FORMAT_SCHEMA_BASE)
        return "format must be 0 (off), GL_FORMAT_JSON or a gl_format_schema code";
    if (so.format != 0 && so.ignore_eos) return "format json cannot be combined with ignore_eos: a JSON document ends on a stop token";
    return nullptr;
}
}  // namespace

extern "C" {

int gl_abi_version(void) { return GL_ABI_VERSION; }
const char* gl_last_error(void) { return gl::get_last_error(); }

int gl_device_count(int* n) {
    if (!n) return bad("gl_device_count: null");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) {
        *n = 0;
        gl::set_last_error(std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
        return GL_ERR_NO_DEVICE;
    }
    *n = c;
    return GL_OK;
}

int gl_engine_create(const char* gguf_path, int device, const gl_engine_opts* opts, gl_engine** out) {
    if (!gguf_path || !out) return bad("gl_engine_create: null argument");
    *out = nullptr;
    // nothing may unwind through the extern "C" boundary: a damaged file that makes the loader run out of memory or throw
    // is an error code, not std::terminate
    try {
        Engine* e = nullptr;
        Status s = Engine::create(gguf_path, device, opts, &e);
        if (!s.ok()) return ret(s);
        *out = new gl_engine{e};
        return GL_OK;
    } catch (const std::bad_alloc&) {
        gl::set_last_error("gl_engine_create: out of host memory while loading (damaged or oversized GGUF?)");
        return GL_ERR_NOMEM;
    } catch (const std::exception& ex) {
        gl::set_last_error(std::string("gl_engine_create: ") + ex.what());
        return GL_ERR_FORMAT;
    }
}

void gl_engine_destroy(gl_engine* e) {
    if (!e) return;
    delete e->impl;
    delete e;
}

int gl_engine_info(const gl_engine* e, gl_model_info* out) {
    if (!e || !out) return bad("gl_engine_info: null argument");
    return ret(e->impl->info(out));
}

int gl_tokenize(const gl_engine* e, const char* utf8, int32_t n_bytes, int add_bos, int parse_special, int32_t* ids, int32_t cap,
                int32_t* n_out) {
    if (!e || !utf8 || !n_out) return bad("gl_tokenize: null argument");
    const gl::Tokenizer& t = e->impl->tokenizer();
    if (!t.ok()) { gl::set_last_error("model carries no supported tokenizer (tokenizer.ggml.model != gpt2)"); return GL_ERR_UNSUPPORTED; }
    std::string text(utf8, n_bytes >= 0 ? (size_t)n_bytes : std::strlen(utf8));
    std::vector<int32_t> v = t.encode(text, add_bos != 0, parse_special != 0);
    *n_out = (int32_t)v.size();
    if ((int32_t)v.size() > cap || (!ids && !v.empty())) { gl::set_last_error("gl_tokenize: output buffer too small"); return ids ? GL_ERR_INVALID : GL_OK; }
    if (!v.empty()) std::memcpy(ids, v.data(), v.size() * sizeof(int32_t));
    return GL_OK;
}

int gl_detokenize(const gl_engine* e, const int32_t* ids, int32_t n, char* buf, int32_t cap, int32_t* len_out) {
    if (!e || (!ids && n > 0) || !len_out) return bad("gl_detokenize: null argument");
    const gl::Tokenizer& t = e->impl->tokenizer();
    if (!t.ok()) { gl::set_last_error("model carries no supported tokenizer"); return GL_ERR_UNSUPPORTED; }
    std::string s = t.decode(ids, n);
    *len_out = (int32_t)s.size();
    if ((int32_t)s.size() > cap || !buf) { gl::set_last_error("gl_detokenize: output buffer too small"); return buf ? GL_ERR_INVALID : GL_OK; }
    std::memcpy(buf, s.data(), s.size());
    return GL_OK;
}

int gl_chat_template(const gl_engine* e, char* buf, int32_t cap, int32_t* len_out) {
    if (!e || !len_out) return bad("gl_chat_template: null argument");
    const std::string& s = e->impl->tokenizer().chat_template;      // "" when the file carries none
    *len_out = (int32_t)s.size();
    if (!buf) return GL_OK;                                          // size query
    if ((int32_t)s.size() > cap) { gl::set_last_error("gl_chat_template: output buffer too small"); return GL_ERR_INVALID; }
    std::memcpy(buf, s.data(), s.size());
    return GL_OK;
}

int gl_generate(gl_engine* e, const int32_t* prompt, int32_t n_prompt, const gl_sample_opts* opts, gl_token_cb cb, void* user,
                int32_t* out_ids, float* out_logprobs, gl_gen_stats* stats) {
    if (!e || !prompt) return bad("gl_generate: null argument");
    gl_sample_opts so{};
    if (opts) so = *opts;
    else { so.num_predict = 128; so.top_p = 1.f; }
    if (const char* m = check_penalties(so)) return bad(m);
    if (const char* m = check_format(so)) return bad(m);
    return ret(e->impl->generate(prompt, n_prompt, so, cb, user, out_ids, out_logprobs, stats));
}

int gl_embed(gl_engine* e, const int32_t* ids, const int32_t* seq_offsets, int32_t n_seq, float* out, gl_gen_stats* stats) {
    if (!e || !ids || !seq_offsets || !out || n_seq <= 0) return bad("gl_embed: bad argument");
    return ret(e->impl->embed(ids, seq_offsets, n_seq, out, stats));
}

// ---- continuous batching -------------------------------------------------------------------------
int gl_seq_open(gl_engine* e, const int32_t* prompt, int32_t n_prompt, const gl_sample_opts* opts, int32_t* slot) {
    if (!e || !prompt || !slot) return bad("gl_seq_open: null argument");
    gl_sample_opts so{};
    if (opts) so = *opts;
    else { so.num_predict = 128; so.top_p = 1.f; }
    if (const char* m = check_penalties(so)) return bad(m);
    if (const char* m = check_format(so)) return bad(m);
    int s = -1;
    const int rc = ret(e->impl->seq_open(prompt, n_prompt, so, &s));
    if (rc == GL_OK) *slot = s;
    return rc;
}

int gl_seq_open_many(gl_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seq, const gl_sample_opts* opts, int32_t* slots,
                     int32_t* n_opened) {
    if (!e || !ids || !offsets || !opts || !slots || !n_opened) return bad("gl_seq_open_many: null argument");
    for (int32_t i = 0; i < n_seq; ++i) {
        if (const char* m = check_penalties(opts[i])) return bad(m);
        if (const char* m = check_format(opts[i])) return bad(m);
    }
    int k = 0;
    const int rc = ret(e->impl->seq_open_many(ids, offsets, n_seq, opts, slots, &k));
    *n_opened = k;
    return rc;
}

int gl_batch_step(gl_engine* e, int32_t* slots, int32_t* ids, float* logprobs, int32_t* done, int32_t cap, int32_t* n) {
    if (!e || !n) return bad("gl_batch_step: null argument");
    int k = 0;
    const int rc = ret(e->impl->batch_step(slots, ids, logprobs, done, cap, &k));
    *n = k;
    return rc;
}

int gl_seq_close(gl_engine* e, int32_t slot) {
    if (!e) return bad("gl_seq_close: null engine");
    return ret(e->impl->seq_close(slot));
}

int gl_seq_logits(gl_engine* e, int32_t slot, float* out, int32_t n_vocab) {
    if (!e || !out) return bad("gl_seq_logits: null argument");
    return ret(e->impl->seq_logits(slot, out, n_vocab));
}

int gl_seq_stats(gl_engine* e, int32_t slot, gl_gen_stats* stats) {
    if (!e || !stats) return bad("gl_seq_stats: null argument");
    return ret(e->impl->seq_stats(slot, stats));
}

int gl_token_piece(const gl_engine* e, int32_t id, char* buf, int32_t cap, int32_t* len_out) {
    if (!e || !len_out) return bad("gl_token_piece: null argument");
    const gl::Tokenizer& t = e->impl->tokenizer();
    if (!t.ok()) { *len_out = 0; return GL_OK; }                    // no tokenizer: no piece, like the gl_generate callback
    const std::string pc = t.piece(id);
    *len_out = (int32_t)pc.size();
    if (!buf) return GL_OK;
    if ((int32_t)pc.size() > cap) { gl::set_last_error("gl_token_piece: output buffer too small"); return GL_ERR_INVALID; }
    std::memcpy(buf, pc.data(), pc.size());
    return GL_OK;
}

int gl_token_text(const gl_engine* e, int32_t id, char* buf, int32_t cap, int32_t* len_out) {
    if (!e || !len_out) return bad("gl_token_text: null argument");
    const gl::Tokenizer& t = e->impl->tokenizer();
    if (!t.ok()) { *len_out = 0; return GL_OK; }
    const std::string tx = t.text(id);
    *len_out = (int32_t)tx.size();
    if (!buf) return GL_OK;
    if ((int32_t)tx.size() > cap) { gl::set_last_error("gl_token_text: output buffer too small"); return GL_ERR_INVALID; }
    std::memcpy(buf, tx.data(), tx.size());
    return GL_OK;
}

int gl_batch_counters(gl_engine* e, uint64_t out[8], int32_t reset) {
    if (!e || !out) return bad("gl_batch_counters: null argument");
    e->impl->batch_counters(out, reset != 0);
    return GL_OK;
}

int gl_time_batch_step(gl_engine* e, int32_t batch, int32_t ctx_len, int32_t iters, float* ms_per_step, int32_t* launches_per_step,
                       uint64_t* weight_bytes) {
    if (!e) return bad("gl_time_batch_step: null engine");
    return ret(e->impl->time_batch_step(batch, ctx_len, iters, ms_per_step, launches_per_step, weight_bytes));
}

int gl_last_logits(gl_engine* e, int32_t step, float* out, int32_t n_vocab) {
    if (!e || !out) return bad("gl_last_logits: null argument");
    return ret(e->impl->last_logits(step, out, n_vocab));
}

int gl_sample_logits(gl_engine* e, const float* logits, int32_t n_vocab, const gl_sample_opts* opts, int32_t out_index, int32_t* id,
                     float* logprob) {
    if (!e || !logits || !opts) return bad("gl_sample_logits: null argument");
    if (const char* m = check_penalties(*opts)) return bad(m);
    int tid = 0;
    const int rc = ret(e->impl->sample_logits(logits, n_vocab, *opts, out_index, &tid, logprob));
    if (rc == GL_OK && id) *id = tid;
    return rc;
}

int gl_penalize_logits(gl_engine* e, float* logits, int32_t n_vocab, const gl_sample_opts* opts, const int32_t* history, int32_t n_history) {
    if (!e || !logits || !opts) return bad("gl_penalize_logits: null argument");
    if (const char* m = check_penalties(*opts)) return bad(m);
    return ret(e->impl->penalize_logits(logits, n_vocab, *opts, history, n_history));
}

int gl_constrain_logits(gl_engine* e, float* logits, int32_t n_vocab, const gl_sample_opts* opts, const int32_t* generated,
                        int32_t n_generated) {
    if (!e || !logits || !opts) return bad("gl_constrain_logits: null argument");
    if (opts->format != 0 && opts->format != GL_FORMAT_JSON && opts->format < GL_FORMAT_SCHEMA_BASE)
        return bad("format must be 0 (off), GL_FORMAT_JSON or a gl_format_schema code");
    return ret(e->impl->constrain_logits(logits, n_vocab, *opts, generated, n_generated));
}

int gl_format_schema(gl_engine* e, const char* schema_utf8, int32_t n_bytes, int32_t* format_out) {
    if (!e || !schema_utf8 || n_bytes < 0 || !format_out) return bad("gl_format_schema: bad argument");
    int code = 0;
    const int rc = ret(e->impl->format_schema(schema_utf8, n_bytes, &code));
    if (rc == GL_OK) *format_out = code;
    return rc;
}

int gl_gemv(gl_engine* e, int ggml_type, const void* w_host, int32_t rows, int32_t cols, const float* x, float* y, int32_t iters,
            float* kernel_ms) {
    if (!e) return bad("gl_gemv: null engine");
    return ret(e->impl->gemv_host(ggml_type, w_host, rows, cols, x, y, iters, kernel_ms));
}

int gl_gemv_model_tensor(gl_engine* e, const char* tensor_name, const float* x, float* y, int32_t iters, int32_t flush_l2,
                         float* kernel_ms, uint64_t* weight_bytes) {
    if (!e || !tensor_name || !x || !y) return bad("gl_gemv_model_tensor: null argument");
    return ret(e->impl->gemv_tensor(tensor_name, x, y, iters, flush_l2, kernel_ms, weight_bytes));
}

int gl_rmsnorm(gl_engine* e, const float* x, const float* w, int32_t n, float eps, float* y) {
    if (!e || !x || !w || !y || n <= 0) return bad("gl_rmsnorm: bad argument");
    return ret(e->impl->rmsnorm(x, w, n, eps, y));
}

int gl_decode_step(gl_engine* e, int32_t token, float* logits, int32_t* argmax, float* logprob) {
    if (!e) return bad("gl_decode_step: null engine");
    return ret(e->impl->decode_step(token, logits, argmax, logprob));
}

int gl_kv_reset(gl_engine* e) {
    if (!e) return bad("gl_kv_reset: null engine");
    return ret(e->impl->kv_reset());
}

int gl_position(const gl_engine* e, int32_t* pos) {
    if (!e || !pos) return bad("gl_position: null argument");
    *pos = e->impl->position();
    return GL_OK;
}

int gl_prefill(gl_engine* e, const int32_t* ids, int32_t n, float* last_logits) {
    if (!e || !ids) return bad("gl_prefill: null argument");
    return ret(e->impl->prefill(ids, n, last_logits));
}

int gl_time_decode(gl_engine* e, int32_t ctx_len, int32_t iters, float* ms_per_step, int32_t* launches_per_step) {
    if (!e) return bad("gl_time_decode: null engine");
    return ret(e->impl->time_decode(ctx_len, iters, ms_per_step, launches_per_step));
}

// profiling aid (not part of the reference-facing ABI): per-phase globaltimer stamps of the persistent kernel
int gl_debug_mega_trace(gl_engine* e, unsigned long long* out, int32_t cap, int32_t* n_ctas, int32_t* n_phases) {
    if (!e || !out) return bad("gl_debug_mega_trace: null argument");
    return ret(e->impl->mega_trace(out, cap, n_ctas, n_phases));
}

// profiling aid: %globaltimer stamps of every GEMV / attention launch of the last decode step (GL_TRACE=1)
int gl_debug_perop_trace(gl_engine* e, unsigned long long* out, int32_t cap, int32_t* n_launches) {
    if (!e || !out || !n_launches) return bad("gl_debug_perop_trace: null argument");
    return ret(e->impl->perop_trace(out, cap, n_launches));
}

}  // extern "C"
