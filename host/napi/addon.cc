// N-API shim over the C ABI (include/gridllm_native.h).  Thin by design: every export forwards to exactly one
// gl_* call; blocking calls run on the libuv pool (napi_create_async_work) and per-token callbacks reach JS
// through a napi_threadsafe_function, so the worker's heartbeat timers (WorkerClientService.ts:316-323) keep
// firing during a long job.  node_api.h is not present in the build image, so this file is compiled only
// where it exists (see host/napi/binding.gyp); the same ABI is exercised from Python (gridllm_b200/native.py).
//
// JS surface (consumed by host/src/NativeInferenceService.ts):
//   deviceCount(): number
//   createEngine(path, device, {maxCtx, actBits}) -> external
//   engineInfo(engine) -> {name, quantization, nParams, fileBytes, nVocab, nCtx, hasTokenizer, ...}
//   tokenize(engine, text, addBos, parseSpecial) -> Int32Array ; detokenize(engine, Int32Array) -> string
//   generate(engine, Int32Array prompt, {numPredict, ignoreEos, stopIds}, onToken|null) -> Promise<{ids, logprobs, stats}>
//   embed(engine, Int32Array ids, Int32Array offsets) -> Promise<{embeddings: Float32Array, stats}>
//   chatTemplate(engine) -> string   (tokenizer.chat_template of the GGUF; the TS host picks the message framing from it)
//   tokenText(engine, id) -> string  (the vocabulary's spelling of a token, control tokens included: bos_token / eos_token of a template)
//   seqOpen(engine, Int32Array prompt, {numPredict, ...}) -> Promise<number>      \  continuous batching (SURVEY.md 8f.1):
//   batchStep(engine) -> Promise<Array<{slot, id, logprob, done, piece}>>          |  every job the worker holds is a sequence;
//   seqClose(engine, slot) ; seqStats(engine, slot) -> stats                      /  one batched step serves all of them
//   destroyEngine(engine)
#include <node_api.h>

#include <cstring>
#include <atomic>
#include <memory>
#include <string>
#include <vector>

#include "../../include/gridllm_native.h"

namespace {

#define NAPI_OK(call)                                                   \
    do {                                                                \
        if ((call) != napi_ok) {                                        \
            napi_throw_error(env, nullptr, "N-API call failed: " #call); \
            return nullptr;                                             \
        }                                                               \
    } while (0)

napi_value throw_gl(napi_env env, const char* what) {
    std::string m = std::string(what) + ": " + gl_last_error();
    napi_throw_error(env, nullptr, m.c_str());
    return nullptr;
}

gl_engine* unwrap(napi_env env, napi_value v) {
    void* p = nullptr;
    napi_get_value_external(env, v, &p);
    return static_cast<gl_engine*>(p);
}

napi_value DeviceCount(napi_env env, napi_callback_info) {
    int n = 0;
    gl_device_count(&n);
    napi_value out;
    NAPI_OK(napi_create_int32(env, n, &out));
    return out;
}

napi_value CreateEngine(napi_env env, napi_callback_info info) {
    size_t argc = 3;
    napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    char path[4096];
    size_t len = 0;
    NAPI_OK(napi_get_value_string_utf8(env, argv[0], path, sizeof path, &len));
    int32_t device = 0;
    NAPI_OK(napi_get_value_int32(env, argv[1], &device));
    gl_engine_opts o{};
    if (argc > 2) {
        napi_value v;
        if (napi_get_named_property(env, argv[2], "maxCtx", &v) == napi_ok) napi_get_value_int32(env, v, &o.max_ctx);
        if (napi_get_named_property(env, argv[2], "actBits", &v) == napi_ok) napi_get_value_int32(env, v, &o.act_bits);
        if (napi_get_named_property(env, argv[2], "maxBatch", &v) == napi_ok) napi_get_value_int32(env, v, &o.max_batch);
        if (napi_get_named_property(env, argv[2], "kvPoolTokens", &v) == napi_ok) napi_get_value_int32(env, v, &o.kv_pool_tokens);
        if (napi_get_named_property(env, argv[2], "prefixCache", &v) == napi_ok) {      // boolean (or 0 / 1)
            bool b = false;
            if (napi_get_value_bool(env, v, &b) == napi_ok) o.prefix_cache = b ? 1 : 0;
            else napi_get_value_int32(env, v, &o.prefix_cache);
        }
    }
    o.use_graph = 1;
    o.use_pdl = 1;
    gl_engine* e = nullptr;
    if (gl_engine_create(path, device, &o, &e) != GL_OK) return throw_gl(env, "gl_engine_create");
    napi_value ext;
    NAPI_OK(napi_create_external(env, e, [](napi_env, void* p, void*) { gl_engine_destroy(static_cast<gl_engine*>(p)); }, nullptr, &ext));
    return ext;
}

// repetition penalties and min_p (Ollama's options of the same names, camel-cased like the other sampling options); an absent
// property leaves the field at its zero, which means "off" (include/gridllm_native.h)
void read_penalty_opts(napi_env env, napi_value o, gl_sample_opts& so) {
    napi_value v;
    double d = 0.0;
    if (napi_get_named_property(env, o, "repeatPenalty", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.repeat_penalty = (float)d;
    if (napi_get_named_property(env, o, "repeatLastN", &v) == napi_ok) napi_get_value_int32(env, v, &so.repeat_last_n);
    if (napi_get_named_property(env, o, "presencePenalty", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.presence_penalty = (float)d;
    if (napi_get_named_property(env, o, "frequencyPenalty", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.frequency_penalty = (float)d;
    if (napi_get_named_property(env, o, "minP", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.min_p = (float)d;
    // output format: "json" (or GL_FORMAT_JSON) turns the JSON grammar mask on, a formatSchema code the schema mask; absent, ""
    // or 0 is free text; anything else reaches the library as it is and is refused there (GL_ERR_INVALID)
    napi_valuetype vt;
    if (napi_get_named_property(env, o, "format", &v) == napi_ok && napi_typeof(env, v, &vt) == napi_ok) {
        if (vt == napi_string) {
            char buf[16] = {0};
            size_t len = 0;
            if (napi_get_value_string_utf8(env, v, buf, sizeof buf, &len) == napi_ok)
                so.format = len == 0 ? 0 : (std::strcmp(buf, "json") == 0 ? GL_FORMAT_JSON : -1);
        } else if (vt == napi_number) {
            napi_get_value_int32(env, v, &so.format);
        }
    }
}

// ---- generate: async work + threadsafe token callback --------------------------------------------------
struct GenJob {
    gl_engine* e;
    std::vector<int32_t> prompt, stop_ids, ids;
    std::vector<float> lps;
    gl_sample_opts so{};
    gl_gen_stats st{};
    int rc = 0;
    std::string err;
    napi_threadsafe_function tsfn = nullptr;
    napi_deferred deferred = nullptr;
    napi_async_work work = nullptr;
    // set on the JS thread when the token callback returns a truthy value; shared with the queued tokens, which can outlive the job
    std::shared_ptr<std::atomic<int>> cancel = std::make_shared<std::atomic<int>>(0);
};
struct Tok { int32_t id; float lp; std::string piece; std::shared_ptr<std::atomic<int>> cancel; };

int on_token(void* user, int32_t id, float lp, const char* piece, int32_t n) {
    GenJob* j = static_cast<GenJob*>(user);
    if (!j->tsfn) return 0;
    // tokens reach JS asynchronously, so a cancel request (job_cancellation, a completed stop string) arrives a few tokens
    // late: the wrapper trims the text, gl_generate stops at the next callback
    if (j->cancel->load(std::memory_order_relaxed)) return 1;
    Tok* t = new Tok{id, lp, piece ? std::string(piece, n) : std::string(), j->cancel};
    return napi_call_threadsafe_function(j->tsfn, t, napi_tsfn_nonblocking) == napi_ok ? 0 : 1;
}

void call_js(napi_env env, napi_value cb, void*, void* data) {
    Tok* t = static_cast<Tok*>(data);
    if (env && cb) {
        napi_value argv[3], undef;
        napi_create_int32(env, t->id, &argv[0]);
        napi_create_double(env, t->lp, &argv[1]);
        napi_create_string_utf8(env, t->piece.data(), t->piece.size(), &argv[2]);
        napi_get_undefined(env, &undef);
        napi_value ret;
        bool stop = false;
        if (napi_call_function(env, undef, cb, 3, argv, &ret) == napi_ok && napi_coerce_to_bool(env, ret, &ret) == napi_ok &&
            napi_get_value_bool(env, ret, &stop) == napi_ok && stop)
            t->cancel->store(1, std::memory_order_relaxed);
    }
    delete t;
}

void gen_execute(napi_env, void* data) {
    GenJob* j = static_cast<GenJob*>(data);
    j->so.n_stop_ids = (int32_t)j->stop_ids.size();
    j->so.stop_ids = j->stop_ids.data();
    j->ids.resize(j->so.num_predict > 0 ? j->so.num_predict : 128);
    j->lps.resize(j->ids.size());
    j->rc = gl_generate(j->e, j->prompt.data(), (int32_t)j->prompt.size(), &j->so, on_token, j, j->ids.data(), j->lps.data(), &j->st);
    if (j->rc != GL_OK) j->err = gl_last_error();
}

void gen_complete(napi_env env, napi_status, void* data) {
    GenJob* j = static_cast<GenJob*>(data);
    if (j->tsfn) napi_release_threadsafe_function(j->tsfn, napi_tsfn_release);
    if (j->rc != GL_OK && j->rc != GL_ERR_CANCELLED) {
        napi_value msg, err;
        napi_create_string_utf8(env, j->err.c_str(), NAPI_AUTO_LENGTH, &msg);
        napi_create_error(env, nullptr, msg, &err);
        napi_reject_deferred(env, j->deferred, err);
    } else {
        napi_value out, v, ab;
        napi_create_object(env, &out);
        void* p;
        napi_create_arraybuffer(env, j->st.eval_count * 4, &p, &ab);
        memcpy(p, j->ids.data(), j->st.eval_count * 4);
        napi_create_typedarray(env, napi_int32_array, j->st.eval_count, ab, 0, &v);
        napi_set_named_property(env, out, "ids", v);
        napi_create_arraybuffer(env, j->st.eval_count * 4, &p, &ab);
        memcpy(p, j->lps.data(), j->st.eval_count * 4);
        napi_create_typedarray(env, napi_float32_array, j->st.eval_count, ab, 0, &v);
        napi_set_named_property(env, out, "logprobs", v);
        napi_value st;
        napi_create_object(env, &st);
        auto seti = [&](const char* k, double d) { napi_value x; napi_create_double(env, d, &x); napi_set_named_property(env, st, k, x); };
        seti("promptEvalCount", j->st.prompt_eval_count); seti("evalCount", j->st.eval_count);
        seti("promptEvalDurationNs", (double)j->st.prompt_eval_duration_ns); seti("evalDurationNs", (double)j->st.eval_duration_ns);
        seti("totalDurationNs", (double)j->st.total_duration_ns); seti("loadDurationNs", (double)j->st.load_duration_ns);
        seti("doneReason", j->st.done_reason);
        napi_set_named_property(env, out, "stats", st);
        napi_resolve_deferred(env, j->deferred, out);
    }
    napi_delete_async_work(env, j->work);
    delete j;
}

napi_value Generate(napi_env env, napi_callback_info info) {
    size_t argc = 4;
    napi_value argv[4];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    GenJob* j = new GenJob();
    j->e = unwrap(env, argv[0]);
    void* data; size_t n; napi_typedarray_type ty; napi_value ab; size_t off;
    NAPI_OK(napi_get_typedarray_info(env, argv[1], &ty, &n, &data, &ab, &off));
    j->prompt.assign(static_cast<int32_t*>(data), static_cast<int32_t*>(data) + n);
    napi_value v;
    j->so.top_p = 1.f;
    if (napi_get_named_property(env, argv[2], "numPredict", &v) == napi_ok) napi_get_value_int32(env, v, &j->so.num_predict);
    bool b = false;
    if (napi_get_named_property(env, argv[2], "ignoreEos", &v) == napi_ok && napi_get_value_bool(env, v, &b) == napi_ok) j->so.ignore_eos = b;
    // sampling options (InferenceRequest.options: client/src/types/index.ts:1-27); absent = greedy
    double d = 0.0;
    if (napi_get_named_property(env, argv[2], "temperature", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) j->so.temperature = (float)d;
    if (napi_get_named_property(env, argv[2], "topK", &v) == napi_ok) napi_get_value_int32(env, v, &j->so.top_k);
    if (napi_get_named_property(env, argv[2], "topP", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) j->so.top_p = (float)d;
    bool lossless = false;
    if (napi_get_named_property(env, argv[2], "seed", &v) == napi_ok) napi_get_value_bigint_uint64(env, v, &j->so.seed, &lossless);
    read_penalty_opts(env, argv[2], j->so);
    napi_valuetype vt;
    if (argc > 3 && napi_typeof(env, argv[3], &vt) == napi_ok && vt == napi_function) {
        napi_value name;
        napi_create_string_utf8(env, "gl_token", NAPI_AUTO_LENGTH, &name);
        NAPI_OK(napi_create_threadsafe_function(env, argv[3], nullptr, name, 0, 1, nullptr, nullptr, nullptr, call_js, &j->tsfn));
    }
    napi_value promise, rname;
    NAPI_OK(napi_create_promise(env, &j->deferred, &promise));
    napi_create_string_utf8(env, "gl_generate", NAPI_AUTO_LENGTH, &rname);
    NAPI_OK(napi_create_async_work(env, nullptr, rname, gen_execute, gen_complete, j, &j->work));
    NAPI_OK(napi_queue_async_work(env, j->work));
    return promise;
}

napi_value EngineInfo(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    gl_model_info mi{};
    if (gl_engine_info(unwrap(env, argv[0]), &mi) != GL_OK) return throw_gl(env, "gl_engine_info");
    napi_value out, v;
    NAPI_OK(napi_create_object(env, &out));
    auto sets = [&](const char* k, const char* s) { napi_create_string_utf8(env, s, NAPI_AUTO_LENGTH, &v); napi_set_named_property(env, out, k, v); };
    auto setd = [&](const char* k, double d) { napi_create_double(env, d, &v); napi_set_named_property(env, out, k, v); };
    sets("arch", mi.arch); sets("name", mi.name); sets("quantization", mi.quantization);
    setd("nParams", (double)mi.n_params); setd("fileBytes", (double)mi.file_bytes); setd("nVocab", mi.n_vocab); setd("nCtx", mi.n_ctx);
    setd("nLayer", mi.n_layer); setd("nEmbd", mi.n_embd); setd("hasTokenizer", mi.has_tokenizer); setd("device", mi.device);
    return out;
}

napi_value Tokenize(napi_env env, napi_callback_info info) {
    size_t argc = 4;
    napi_value argv[4];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    size_t len = 0;
    NAPI_OK(napi_get_value_string_utf8(env, argv[1], nullptr, 0, &len));
    std::string text(len, '\0');
    NAPI_OK(napi_get_value_string_utf8(env, argv[1], &text[0], len + 1, &len));
    bool add_bos = true, special = false;
    if (argc > 2) napi_get_value_bool(env, argv[2], &add_bos);
    if (argc > 3) napi_get_value_bool(env, argv[3], &special);
    std::vector<int32_t> ids(len + 8);
    int32_t n = 0;
    if (gl_tokenize(unwrap(env, argv[0]), text.data(), (int32_t)len, add_bos, special, ids.data(), (int32_t)ids.size(), &n) != GL_OK)
        return throw_gl(env, "gl_tokenize");
    napi_value ab, out;
    void* p;
    NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 4, &p, &ab));
    memcpy(p, ids.data(), (size_t)n * 4);
    NAPI_OK(napi_create_typedarray(env, napi_int32_array, n, ab, 0, &out));
    return out;
}

napi_value Detokenize(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* data; size_t n; napi_typedarray_type ty; napi_value ab; size_t off;
    NAPI_OK(napi_get_typedarray_info(env, argv[1], &ty, &n, &data, &ab, &off));
    std::string buf(16 * (n + 1), '\0');
    int32_t len = 0;
    if (gl_detokenize(unwrap(env, argv[0]), static_cast<int32_t*>(data), (int32_t)n, &buf[0], (int32_t)buf.size(), &len) != GL_OK)
        return throw_gl(env, "gl_detokenize");
    napi_value out;
    NAPI_OK(napi_create_string_utf8(env, buf.data(), len, &out));
    return out;
}

// embed: same async-work pattern as generate, without a token callback
struct EmbJob {
    gl_engine* e;
    std::vector<int32_t> ids, offs;
    std::vector<float> out;
    gl_gen_stats st{};
    int rc = 0, n_embd = 0;
    std::string err;
    napi_deferred deferred = nullptr;
    napi_async_work work = nullptr;
};

void emb_execute(napi_env, void* data) {
    EmbJob* j = static_cast<EmbJob*>(data);
    gl_model_info mi{};
    gl_engine_info(j->e, &mi);
    j->n_embd = mi.n_embd;
    const int n_seq = (int)j->offs.size() - 1;
    j->out.resize((size_t)n_seq * mi.n_embd);
    j->rc = gl_embed(j->e, j->ids.data(), j->offs.data(), n_seq, j->out.data(), &j->st);
    if (j->rc != GL_OK) j->err = gl_last_error();
}

void emb_complete(napi_env env, napi_status, void* data) {
    EmbJob* j = static_cast<EmbJob*>(data);
    if (j->rc != GL_OK) {
        napi_value msg, err;
        napi_create_string_utf8(env, j->err.c_str(), NAPI_AUTO_LENGTH, &msg);
        napi_create_error(env, nullptr, msg, &err);
        napi_reject_deferred(env, j->deferred, err);
    } else {
        napi_value out, ab, v, st;
        void* p;
        napi_create_object(env, &out);
        napi_create_arraybuffer(env, j->out.size() * 4, &p, &ab);
        memcpy(p, j->out.data(), j->out.size() * 4);
        napi_create_typedarray(env, napi_float32_array, j->out.size(), ab, 0, &v);
        napi_set_named_property(env, out, "embeddings", v);
        napi_create_object(env, &st);
        auto seti = [&](const char* k, double d) { napi_value x; napi_create_double(env, d, &x); napi_set_named_property(env, st, k, x); };
        seti("promptEvalCount", j->st.prompt_eval_count); seti("totalDurationNs", (double)j->st.total_duration_ns);
        seti("loadDurationNs", (double)j->st.load_duration_ns);
        napi_set_named_property(env, out, "stats", st);
        napi_resolve_deferred(env, j->deferred, out);
    }
    napi_delete_async_work(env, j->work);
    delete j;
}

napi_value Embed(napi_env env, napi_callback_info info) {
    size_t argc = 3;
    napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    EmbJob* j = new EmbJob();
    j->e = unwrap(env, argv[0]);
    void* data; size_t n; napi_typedarray_type ty; napi_value ab; size_t off;
    NAPI_OK(napi_get_typedarray_info(env, argv[1], &ty, &n, &data, &ab, &off));
    j->ids.assign(static_cast<int32_t*>(data), static_cast<int32_t*>(data) + n);
    NAPI_OK(napi_get_typedarray_info(env, argv[2], &ty, &n, &data, &ab, &off));
    j->offs.assign(static_cast<int32_t*>(data), static_cast<int32_t*>(data) + n);
    napi_value promise, rname;
    NAPI_OK(napi_create_promise(env, &j->deferred, &promise));
    napi_create_string_utf8(env, "gl_embed", NAPI_AUTO_LENGTH, &rname);
    NAPI_OK(napi_create_async_work(env, nullptr, rname, emb_execute, emb_complete, j, &j->work));
    NAPI_OK(napi_queue_async_work(env, j->work));
    return promise;
}

napi_value DestroyEngine(napi_env env, napi_callback_info) {
    // engines are released by the external's finalizer (CreateEngine); kept for API symmetry
    napi_value u;
    napi_get_undefined(env, &u);
    return u;
}

// tokenizer.chat_template of the GGUF ("" when the file carries none)
napi_value ChatTemplate(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    gl_engine* e = unwrap(env, argv[0]);
    int32_t len = 0;
    if (gl_chat_template(e, nullptr, 0, &len) != GL_OK) return throw_gl(env, "gl_chat_template");
    std::string buf((size_t)len, '\0');
    if (len > 0 && gl_chat_template(e, &buf[0], len, &len) != GL_OK) return throw_gl(env, "gl_chat_template");
    napi_value out;
    NAPI_OK(napi_create_string_utf8(env, buf.data(), (size_t)len, &out));
    return out;
}

// the vocabulary's spelling of a token, control tokens included: bos_token / eos_token of a chat template (gl_token_text)
napi_value TokenText(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    gl_engine* e = unwrap(env, argv[0]);
    int32_t id = -1, len = 0;
    NAPI_OK(napi_get_value_int32(env, argv[1], &id));
    char buf[512];
    if (gl_token_text(e, id, buf, (int32_t)sizeof buf, &len) != GL_OK) return throw_gl(env, "gl_token_text");
    napi_value out;
    NAPI_OK(napi_create_string_utf8(env, buf, (size_t)len, &out));
    return out;
}

// formatSchema(engine, schemaText) -> the gl_format_schema code for a request's `format` (throws with the library's message,
// e.g. "format schema: 'pattern' is not supported at /properties/zip")
napi_value FormatSchema(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    gl_engine* e = unwrap(env, argv[0]);
    size_t len = 0;
    NAPI_OK(napi_get_value_string_utf8(env, argv[1], nullptr, 0, &len));
    std::string text(len + 1, '\0');
    NAPI_OK(napi_get_value_string_utf8(env, argv[1], &text[0], len + 1, &len));
    int32_t code = 0;
    if (gl_format_schema(e, text.data(), (int32_t)len, &code) != GL_OK) return throw_gl(env, "gl_format_schema");
    napi_value out;
    NAPI_OK(napi_create_int32(env, code, &out));
    return out;
}

void read_sample_opts(napi_env env, napi_value o, gl_sample_opts& so, std::vector<int32_t>& stop_ids) {
    napi_value v;
    so.num_predict = 128;
    so.top_p = 1.f;
    double d = 0;
    bool b = false;
    if (napi_get_named_property(env, o, "numPredict", &v) == napi_ok && napi_get_value_int32(env, v, &so.num_predict) != napi_ok) so.num_predict = 128;
    if (so.num_predict <= 0) so.num_predict = 128;
    if (napi_get_named_property(env, o, "ignoreEos", &v) == napi_ok && napi_get_value_bool(env, v, &b) == napi_ok) so.ignore_eos = b ? 1 : 0;
    if (napi_get_named_property(env, o, "temperature", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.temperature = (float)d;
    if (napi_get_named_property(env, o, "topK", &v) == napi_ok) napi_get_value_int32(env, v, &so.top_k);
    if (napi_get_named_property(env, o, "topP", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.top_p = (float)d;
    if (napi_get_named_property(env, o, "seed", &v) == napi_ok && napi_get_value_double(env, v, &d) == napi_ok) so.seed = (uint64_t)d;
    read_penalty_opts(env, o, so);
    if (napi_get_named_property(env, o, "stopIds", &v) == napi_ok) {
        void* data; size_t n; napi_typedarray_type ty; napi_value ab; size_t off;
        if (napi_get_typedarray_info(env, v, &ty, &n, &data, &ab, &off) == napi_ok && ty == napi_int32_array)
            stop_ids.assign(static_cast<int32_t*>(data), static_cast<int32_t*>(data) + n);
    }
}

// ---- continuous batching: gl_seq_open (a prefill: async work) / gl_batch_step (one token for every open sequence: async work) ----
struct SeqJob {
    gl_engine* e;
    std::vector<int32_t> prompt, stop_ids;
    gl_sample_opts so{};
    int32_t slot = -1;
    // batch step
    std::vector<int32_t> slots, ids, done;
    std::vector<float> lps;
    std::vector<std::string> pieces;
    int32_t n = 0;
    bool is_step = false;
    int rc = 0;
    std::string err;
    napi_deferred deferred = nullptr;
    napi_async_work work = nullptr;
};
void seq_execute(napi_env, void* data) {
    SeqJob* j = static_cast<SeqJob*>(data);
    if (!j->is_step) {
        j->so.n_stop_ids = (int32_t)j->stop_ids.size();
        j->so.stop_ids = j->stop_ids.data();
        j->rc = gl_seq_open(j->e, j->prompt.data(), (int32_t)j->prompt.size(), &j->so, &j->slot);
    } else {
        j->slots.resize(128); j->ids.resize(128); j->done.resize(128); j->lps.resize(128);
        j->rc = gl_batch_step(j->e, j->slots.data(), j->ids.data(), j->lps.data(), j->done.data(), 128, &j->n);
        for (int i = 0; j->rc == GL_OK && i < j->n; ++i) {
            char buf[256];
            int32_t len = 0;
            if (j->ids[i] >= 0 && gl_token_piece(j->e, j->ids[i], buf, (int32_t)sizeof buf, &len) == GL_OK) j->pieces.emplace_back(buf, (size_t)len);
            else j->pieces.emplace_back();
        }
    }
    if (j->rc != GL_OK) j->err = gl_last_error();
}
void seq_complete(napi_env env, napi_status, void* data) {
    SeqJob* j = static_cast<SeqJob*>(data);
    if (j->rc != GL_OK) {
        napi_value msg, err;
        napi_create_string_utf8(env, j->err.c_str(), NAPI_AUTO_LENGTH, &msg);
        napi_create_error(env, nullptr, msg, &err);
        napi_reject_deferred(env, j->deferred, err);
    } else if (!j->is_step) {
        napi_value v;
        napi_create_int32(env, j->slot, &v);
        napi_resolve_deferred(env, j->deferred, v);
    } else {
        // an object {n, slots, ids, logprobs, done, pieces: {0: ..., 1: ...}} -- typed arrays, one entry per open sequence
        napi_value out, v, ab;
        napi_create_object(env, &out);
        napi_create_int32(env, j->n, &v);
        napi_set_named_property(env, out, "n", v);
        auto put_i32 = [&](const char* k, const std::vector<int32_t>& a) {
            void* p;
            napi_create_arraybuffer(env, (size_t)j->n * 4, &p, &ab);
            memcpy(p, a.data(), (size_t)j->n * 4);
            napi_create_typedarray(env, napi_int32_array, (size_t)j->n, ab, 0, &v);
            napi_set_named_property(env, out, k, v);
        };
        put_i32("slots", j->slots); put_i32("ids", j->ids); put_i32("done", j->done);
        void* p;
        napi_create_arraybuffer(env, (size_t)j->n * 4, &p, &ab);
        memcpy(p, j->lps.data(), (size_t)j->n * 4);
        napi_create_typedarray(env, napi_float32_array, (size_t)j->n, ab, 0, &v);
        napi_set_named_property(env, out, "logprobs", v);
        napi_value pieces;
        napi_create_object(env, &pieces);
        for (int i = 0; i < j->n; ++i) {
            napi_create_string_utf8(env, j->pieces[i].data(), j->pieces[i].size(), &v);
            napi_set_named_property(env, pieces, std::to_string(i).c_str(), v);
        }
        napi_set_named_property(env, out, "pieces", pieces);
        napi_resolve_deferred(env, j->deferred, out);
    }
    napi_delete_async_work(env, j->work);
    delete j;
}
napi_value queue_seq(napi_env env, SeqJob* j, const char* name) {
    napi_value promise, rname;
    if (napi_create_promise(env, &j->deferred, &promise) != napi_ok) { delete j; return nullptr; }
    napi_create_string_utf8(env, name, NAPI_AUTO_LENGTH, &rname);
    if (napi_create_async_work(env, nullptr, rname, seq_execute, seq_complete, j, &j->work) != napi_ok || napi_queue_async_work(env, j->work) != napi_ok) {
        delete j;
        napi_throw_error(env, nullptr, "could not queue engine work");
        return nullptr;
    }
    return promise;
}
napi_value SeqOpen(napi_env env, napi_callback_info info) {
    size_t argc = 3;
    napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    SeqJob* j = new SeqJob();
    j->e = unwrap(env, argv[0]);
    void* data; size_t n; napi_typedarray_type ty; napi_value ab; size_t off;
    if (napi_get_typedarray_info(env, argv[1], &ty, &n, &data, &ab, &off) != napi_ok || ty != napi_int32_array) {
        delete j;
        napi_throw_error(env, nullptr, "seqOpen: prompt must be an Int32Array");
        return nullptr;
    }
    j->prompt.assign(static_cast<int32_t*>(data), static_cast<int32_t*>(data) + n);
    if (argc > 2) read_sample_opts(env, argv[2], j->so, j->stop_ids);
    else { j->so.num_predict = 128; j->so.top_p = 1.f; }
    return queue_seq(env, j, "gl_seq_open");
}
napi_value BatchStep(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    SeqJob* j = new SeqJob();
    j->e = unwrap(env, argv[0]);
    j->is_step = true;
    return queue_seq(env, j, "gl_batch_step");
}
napi_value SeqClose(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    int32_t slot = -1;
    NAPI_OK(napi_get_value_int32(env, argv[1], &slot));
    if (gl_seq_close(unwrap(env, argv[0]), slot) != GL_OK) return throw_gl(env, "gl_seq_close");
    napi_value u;
    NAPI_OK(napi_get_undefined(env, &u));
    return u;
}
napi_value SeqStats(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    int32_t slot = -1;
    NAPI_OK(napi_get_value_int32(env, argv[1], &slot));
    gl_gen_stats st{};
    if (gl_seq_stats(unwrap(env, argv[0]), slot, &st) != GL_OK) return throw_gl(env, "gl_seq_stats");
    napi_value out;
    NAPI_OK(napi_create_object(env, &out));
    auto seti = [&](const char* k, double d) { napi_value x; napi_create_double(env, d, &x); napi_set_named_property(env, out, k, x); };
    seti("promptEvalCount", st.prompt_eval_count); seti("evalCount", st.eval_count);
    seti("promptEvalDurationNs", (double)st.prompt_eval_duration_ns); seti("evalDurationNs", (double)st.eval_duration_ns);
    seti("totalDurationNs", (double)st.total_duration_ns); seti("loadDurationNs", (double)st.load_duration_ns); seti("doneReason", st.done_reason);
    return out;
}

napi_value Init(napi_env env, napi_value exports) {
    napi_property_descriptor d[] = {
        {"deviceCount", nullptr, DeviceCount, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"createEngine", nullptr, CreateEngine, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"generate", nullptr, Generate, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"engineInfo", nullptr, EngineInfo, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"tokenize", nullptr, Tokenize, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"detokenize", nullptr, Detokenize, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"embed", nullptr, Embed, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"chatTemplate", nullptr, ChatTemplate, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"tokenText", nullptr, TokenText, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"formatSchema", nullptr, FormatSchema, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"seqOpen", nullptr, SeqOpen, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"batchStep", nullptr, BatchStep, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"seqClose", nullptr, SeqClose, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"seqStats", nullptr, SeqStats, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"destroyEngine", nullptr, DestroyEngine, nullptr, nullptr, nullptr, napi_default, nullptr},
    };
    napi_define_properties(env, exports, sizeof d / sizeof d[0], d);
    return exports;
}

}  // namespace

NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
