/*
 * gridllm_native.h -- C ABI of libgridllm_native.so, the H100-native inference engine that
 * replaces the GridLLM worker's Ollama HTTP call-out.
 *
 * The reference has no FFI today: the seam is the TypeScript class OllamaService
 * (/root/reference/client/src/services/OllamaService.ts) as consumed by WorkerClientService
 * (client/src/services/WorkerClientService.ts:32,43,133,520,548,554,596,602,645).  Each entry
 * point below names the reference call it stands in for.  Host bindings that sit on this ABI:
 *   - gridllm_b200/native.py          (ctypes; what the tests and bench run)
 *   - host/napi/addon.cc              (N-API shim, compiled where node_api.h exists)
 *   - host/src/NativeInferenceService.ts (the drop-in for OllamaService; see INTEGRATION.md)
 *
 * Conventions: every function returns 0 (GL_OK) or a negative gl_status; gl_last_error()
 * returns a thread-local message owned by the library.  All buffers are caller-owned plain
 * pointers + sizes; no torch / CUDA types cross the boundary.  One gl_engine = one GPU = one
 * CUDA stream; calls on the same engine must be serialised by the caller, different engines are
 * independent (8 engines <-> 8 worker ids in one process; SURVEY.md section 8e).
 * There is NO CPU fallback: without a usable CUDA device gl_engine_create fails with
 * GL_ERR_NO_DEVICE.
 */
#ifndef GRIDLLM_NATIVE_H
#define GRIDLLM_NATIVE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GL_ABI_VERSION 2

typedef enum gl_status {
    GL_OK = 0,
    GL_ERR_INVALID = -1,      /* bad argument */
    GL_ERR_IO = -2,           /* file missing / unreadable */
    GL_ERR_FORMAT = -3,       /* not a GGUF v2/v3 file, or missing tensor / key */
    GL_ERR_UNSUPPORTED = -4,  /* architecture / tensor type / shape outside the hot path */
    GL_ERR_CUDA = -5,         /* CUDA runtime error (message has the cudaError string) */
    GL_ERR_NOMEM = -6,
    GL_ERR_CANCELLED = -7,    /* token callback asked to stop */
    GL_ERR_NO_DEVICE = -8,    /* no CUDA device: the product path never falls back to CPU */
    GL_ERR_CONTEXT = -9       /* prompt + num_predict exceeds the engine's context */
} gl_status;

/* ggml tensor type ids the engine understands (public ggml enum values). */
enum { GL_TYPE_F32 = 0, GL_TYPE_F16 = 1, GL_TYPE_Q8_0 = 8, GL_TYPE_Q4_K = 12, GL_TYPE_Q6_K = 14, GL_TYPE_BF16 = 30 };

typedef struct gl_engine gl_engine;

typedef struct gl_engine_opts {
    int32_t max_ctx;          /* tokens of KV cache to provision; 0 = min(model ctx, 8192) */
    int32_t act_bits;         /* GEMV activation fixed point: 16 (default, 2x int8 planes) or 8 (ggml-like) */
    int32_t use_graph;        /* 1 (default): decode step replayed as a CUDA graph; 0: plain launches */
    int32_t use_pdl;          /* 1 (default): programmatic dependent launch between step kernels */
    int32_t prefill_mode;     /* 0 auto, 1 sequential decode steps, 2 batched tensor-core prefill.
                                 The prompt pass's 16-bit layer matrices: resident (a copy of every layer matrix built at load, 2 bytes
                                 per weight) when copy + 4 GB fits in the HBM free after the weights and the KV pool, else streamed
                                 (each layer's four GEMM operands dequantised into one staging buffer, the size of the largest
                                 operand, just before their GEMMs: 4 more launches per layer per pass; a 70B q4 model on one
                                 80 GB H100).  Environment GL_PREFILL_WEIGHTS: 0 auto (default), 1 resident (the load fails with
                                 GL_ERR_NOMEM when it does not fit), 2 streamed.  Under prefill_mode 1 neither is built.
                                 Continuous batching (gl_seq_open*) needs the resident copy. */
    int32_t max_batch;        /* continuous batching: sequences that may be open at once (gl_seq_open); 0 / 1 = none, <= 128.
                                 The KV pool is provisioned for max_batch sequences of max_ctx tokens unless kv_pool_tokens says otherwise */
    int32_t kv_pool_tokens;   /* tokens of KV cache shared by all open sequences; 0 = max_ctx * max(1, max_batch) */
    int32_t batch_weights;    /* batched step reads: 0 auto (the quantised weights, dequantised tile by tile inside the GEMM, when the
                                 model's types allow it; else the resident 16-bit copy), 1 the 16-bit copy, 2 the quantised weights */
    /* Prefix reuse across gl_generate calls (Ollama keeps the longest cached common prefix); 0 = off (every call prefills its whole
     * prompt).  The engine records, on the host, the ids at positions [0, n_cached) whose K / V in its single-sequence pages are
     * final after a gl_generate: the prompt, then the generated ids the device has fed (the last draw and a stop token never
     * are).  The next gl_generate keeps the pages of r = max(0, min(L, n_prompt - 8)) positions, L = the longest common prefix
     * of its prompt and the record, and evaluates positions [r, n_prompt) only: at least 8 prompt tokens (the minimum of the
     * tensor-core prompt pass) always run, so the suffix takes the same kind of pass a cold call would.  A reused prefix that
     * came from a prompt pass gives the bits of a cold call; one that reaches into generated tokens holds K / V the decode
     * kernels wrote, and the output is then within the decode-vs-prefill tolerance of a cold call, not bit-identical.
     * The record is cleared by gl_kv_reset and by every other call that writes the single-sequence pages or step state:
     * gl_prefill, gl_decode_step, gl_embed of a sequence longer than 2 048 tokens, gl_sample_logits / gl_penalize_logits /
     * gl_constrain_logits, gl_time_decode.  No reuse under the persistent decode kernel (GL_MEGA=1); gl_seq_open sequences
     * share prefixes through batch_prefix_cache instead.  With prefix_cache on, gl_gen_stats.prompt_eval_count of gl_generate
     * counts the tokens this call evaluated (n_prompt - r) and prompt_eval_duration their device time. */
    int32_t prefix_cache;
    /* reserved[GL_OPT_BATCH_PREFIX_CACHE] is batch_prefix_cache: prompt-prefix KV pages shared between gl_seq_open /
     * gl_seq_open_many sequences; 0 = off (every slot owns all its pages and prefills its whole prompt).  Pages are
     * reference-counted.  After a slot's prompt pass, its full prompt pages [0, floor(n_prompt / 16)) are indexed by their ids
     * (a trie of 16-token pages, ids compared exactly); the last partial page, rows written by decode steps, prompts that
     * stepped through the decode kernels (shorter than the prompt pass's minimum of 8 tokens, prefill_mode 1) and
     * gl_time_batch_step's sequences never are.  A new sequence whose prompt starts with a chain of L indexed pages reads
     * r = 16 floor(min(16 L, n_prompt - 8) / 16) positions from those pages and evaluates only [r, n_prompt): the K / V of a
     * prompt prefix depend on its ids alone, so it gets the bits of a cold open.  Prompts of one gl_seq_open_many call that
     * share a prefix nothing has indexed yet share the first one's pages within the same pass.  It reserves only its own
     * pages, ceil((n_prompt + num_predict) / 16) - r / 16; every position it writes is >= r, so shared pages are never written.
     * When its last reference closes, an indexed page is retained, and allocation (batch slots and gl_generate alike) takes
     * free pages first, then evicts retained pages, least recently released leaves first: GL_ERR_NOMEM comes only when open
     * sequences hold the pool.  gl_gen_stats.prompt_eval_count of gl_seq_stats counts the evaluated tokens and
     * prompt_eval_duration their share of the pass; gl_batch_counters out[7] counts the prompt tokens taken from shared pages.
     * No sharing under GL_PREFILL_FLASH=0 or the persistent decode kernel (GL_MEGA=1).
     * reserved[GL_OPT_CONTEXT_SHIFT] is context_shift (Ollama's context shift): 0 = off, nothing below applies and a sequence
     * longer than the context is GL_ERR_CONTEXT.  With it on, gl_generate, gl_seq_open and gl_seq_open_many keep generating
     * when a sequence fills the context W = gl_model_info.n_ctx, and cut prompts of W tokens or more.  Let k be the request's
     * keep count (gl_sample_opts.num_keep, read only when this option is on: >= 0 clamped to min(num_keep, W - 1), -1 the whole
     * prompt clamped to W - 1, < -1 GL_ERR_INVALID) and d = ceil((W - k) / 2) >= 1 the discard:
     *   - shift: when the next step of a sequence must write the row at position W, positions [k, k + d) are dropped and the
     *     rows [k + d, W) move to [k, W - d), each K row rotated by -d positions (the pair rotation with the engine's fp32
     *     cos / sin table row d, rounded to fp16), V rows copied bit for bit; rows [0, k) are untouched and the step runs at
     *     position W - d.  Moved rows keep the context they were computed in.  The penalty history (prompt, then every
     *     generated id), the grammar-mask state, the output index and the seeded draw (seed, i) are unchanged by a shift.
     *   - prompt cut: a prompt of n_prompt >= W ids is cut to its first k ids plus its newest W - d - k ids (the positions a
     *     shift would leave) and evaluated by one cold prompt pass; prompt_eval_count counts the evaluated ids and the penalty
     *     history starts with the cut prompt.
     *   - num_predict <= W (the output buffers hold W ids); more is GL_ERR_CONTEXT.  Pages are reserved for
     *     min(n_prompt + num_predict, W) positions.
     *   - a sequence with n_prompt + num_predict > W (one that may shift or was cut) neither reads nor indexes shared prompt
     *     pages (batch_prefix_cache), and after gl_generate of such a sequence the prefix_cache record keeps positions [0, k)
     *     only.  Sequences that fit behave exactly as with the option off.
     *   - under the persistent decode kernel (GL_MEGA=1) a gl_generate that would cut or shift is GL_ERR_UNSUPPORTED.
     * The other reserved words must be 0. */
    int32_t reserved[7];
} gl_engine_opts;

#define GL_OPT_BATCH_PREFIX_CACHE 0       /* index of batch_prefix_cache in gl_engine_opts.reserved */
#define GL_OPT_CONTEXT_SHIFT 1            /* index of context_shift in gl_engine_opts.reserved */

typedef struct gl_model_info {
    char     arch[32];
    char     name[96];
    char     quantization[24];   /* "Q4_K_M", "Q8_0", "BF16", ... from general.file_type */
    int32_t  n_layer, n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_ctx_train, n_ctx;
    float    rope_base, rms_eps;
    int32_t  bos_id, eos_id, eot_id, has_tokenizer;
    uint64_t n_params;
    uint64_t file_bytes;
    uint64_t weight_bytes;       /* matrix payload resident in HBM */
    uint64_t decode_bytes_per_token; /* algorithmic weight bytes one decode token must read */
    int32_t  device;
    int32_t  sm_count;
} gl_model_info;

typedef struct gl_sample_opts {
    int32_t  num_predict;     /* OllamaService.ts:105  max_tokens = options.num_predict || 128 */
    float    temperature;     /* 0 = greedy (the parity configuration); > 0: draw from softmax(logits / temperature) */
    int32_t  top_k;           /* candidates = the top_k best logits; <= 0 or > 1024: the 1024 best (not the whole vocabulary) */
    float    top_p;           /* shortest prefix of the candidates whose mass reaches top_p; <= 0 or >= 1: off */
    uint64_t seed;            /* the draw for output i depends on (seed, i) only: a request is reproducible */
    int32_t  ignore_eos;      /* 1: fixed-length generation (bench workloads) */
    int32_t  n_stop_ids;
    const int32_t* stop_ids;  /* extra stop token ids (host resolves stop strings) */
    int32_t  want_logits;     /* 1: keep per-step logits for gl_last_logits (parity tests) */
    /* Repetition penalties (Ollama's options of the same names; arithmetic of llama.cpp's penalties sampler, which Ollama's
     * runner uses -- parity with a real Ollama is unpinned, like the sampler's).  A caller that zeroes these fields gets no
     * penalty and no min_p: every field's zero means "off".
     * History H of a sequence = the prompt ids of the call (BOS and any prepended context included), then every token generated
     * so far (a drawn stop token ends the sequence and is never added).  Window W = the last N entries of H: N = repeat_last_n
     * when > 0, the whole of H when -1; 0 turns every penalty off.  Before EVERY draw (the first token after the prompt
     * included; greedy and sampled alike), for each distinct id t in W occurring c times, in single fp32 operations:
     *   a = logit[t];  if repeat_penalty is active (> 0 and != 1): a = a <= 0 ? a * repeat_penalty : a / repeat_penalty;
     *   logit[t] = a - (c * frequency_penalty + presence_penalty).
     * Reported logprobs and the logits of gl_last_logits / gl_seq_logits are those of the PENALISED logits (what the token was
     * drawn from).  Invalid (GL_ERR_INVALID): non-finite values, repeat_penalty < 0, repeat_last_n < -1, min_p outside [0, 1]. */
    float    repeat_penalty;    /* 0 or 1: off */
    int32_t  repeat_last_n;     /* window: > 0 last N ids, -1 the whole history, 0 no penalty of any kind */
    float    presence_penalty;  /* subtracted once from every id in the window */
    float    frequency_penalty; /* subtracted once per occurrence in the window */
    float    min_p;             /* temperature > 0 only: after top-p keep the prefix of candidates with exp((l - l0) / T) >= min_p; 0 = off */
    /* Output format (Ollama's `format`; 0 = off, GL_FORMAT_JSON = 1; anything else GL_ERR_INVALID).  With GL_FORMAT_JSON the
     * bytes a sequence generates -- the concatenation of the gl_token_piece bytes of its tokens -- are held to the language
     *   root    ::= object
     *   value   ::= object | array | string | number | ("true" | "false" | "null") ws
     *   object  ::= "{" ws ( string ":" ws value ( "," ws string ":" ws value )* )? "}" ws
     *   array   ::= "[" ws ( value ( "," ws value )* )? "]" ws
     *   string  ::= "\"" ( char | "\\" ( ["\\/bfnrt] | "u" hex hex hex hex ) )* "\"" ws
     *   char    ::= any Unicode scalar value >= U+0020 other than " and \, as well-formed UTF-8 (a piece may end inside one)
     *   number  ::= "-"? ( "0" | [1-9] [0-9]* ) ( "." [0-9]+ )? ( [eE] [-+]? [0-9]+ )? ws
     *   ws      ::= "" | " " | "\n" [ \t]{0,20}
     * with nesting depth <= 64 (root included; an opening bracket at depth 64 is masked), starting from the initial state (the
     * prompt does not count).  Before EVERY draw (the first token after the prompt included), after the repetition penalties
     * and before temperature / top-k / top-p / min-p / the greedy argmax, every token whose piece would take the bytes outside
     * the language gets logit -inf; a masked token is never drawn.  Stop tokens (eos, eot when the model has one, stop_ids)
     * are allowed only once the root object has closed, anywhere in its trailing ws, and masked everywhere else; other control
     * tokens (empty piece) are always masked.  After the root closes only ws and stop tokens remain, so a document ends within
     * 22 further draws (done_reason "stop"); a generation cut by num_predict is a valid prefix (done_reason "length").
     * Reported logprobs and the logits of gl_last_logits / gl_seq_logits are those of the masked distribution.
     * Refused: with ignore_eos (GL_ERR_INVALID); stop_ids that are not control tokens (GL_ERR_INVALID); a model without a
     * tokenizer, or whose vocabulary lacks a single-byte token for each of \t, \n, 0x20-0x7E (and 0x80-0xBF when some piece
     * is not whole well-formed UTF-8), or has no eos (GL_ERR_UNSUPPORTED, checked once, at the first JSON request); gl_generate
     * on the persistent decode kernel (GL_MEGA=1, GL_ERR_UNSUPPORTED).  A code >= GL_FORMAT_SCHEMA_BASE from gl_format_schema
     * holds the bytes to the documents of that JSON schema instead (see there); everything else above applies to it as well. */
    union {
        int32_t  format;
        int32_t  reserved[1];
    };
    /* Ollama's num_keep: the prompt positions a context shift keeps (see gl_engine_opts context_shift): >= 0 that many, -1 the
     * whole prompt.  Read only when the engine's context_shift option is on (a caller built against an older header may leave
     * this word, then tail padding, uninitialised). */
    int32_t  num_keep;
} gl_sample_opts;

#define GL_FORMAT_JSON 1
#define GL_FORMAT_SCHEMA_BASE 256

typedef struct gl_gen_stats {
    int32_t prompt_eval_count;     /* InferenceResponse.prompt_eval_count (client/src/types/index.ts:61) */
    int32_t eval_count;            /* InferenceResponse.eval_count */
    int64_t prompt_eval_duration_ns; /* device time (cudaEvent) */
    int64_t eval_duration_ns;      /* device time (cudaEvent) */
    int64_t total_duration_ns;     /* host wall time of the call */
    int64_t load_duration_ns;
    int32_t done_reason;           /* 0 "stop" (eos / stop id), 1 "length", 2 cancelled */
    int32_t kernel_launches;       /* kernels of this library launched by the call */
} gl_gen_stats;

/* Return non-zero to cancel (job_cancellation, JobScheduler.ts:530-536). piece may be NULL when the
 * model carries no tokenizer. */
typedef int (*gl_token_cb)(void* user, int32_t id, float logprob, const char* piece, int32_t piece_len);

/* ---- library / device ---------------------------------------------------------------- */
int         gl_abi_version(void);
const char* gl_last_error(void);
int         gl_device_count(int* n);                       /* checkHealth(): OllamaService.ts:65-83 */

/* ---- engine lifetime (constructor / model load: OllamaService.ts:17-25, Ollama model load) */
int  gl_engine_create(const char* gguf_path, int device, const gl_engine_opts* opts, gl_engine** out);
void gl_engine_destroy(gl_engine* e);
int  gl_engine_info(const gl_engine* e, gl_model_info* out); /* getAvailableModels(): OllamaService.ts:85-95 */

/* ---- tokenizer (inside Ollama for the reference; needed by every generate*/
int  gl_tokenize(const gl_engine* e, const char* utf8, int32_t n_bytes, int add_bos, int parse_special,
                 int32_t* ids, int32_t cap, int32_t* n_out);
int  gl_detokenize(const gl_engine* e, const int32_t* ids, int32_t n, char* buf, int32_t cap, int32_t* len_out);
/* tokenizer.chat_template of the GGUF (UTF-8, not NUL-terminated; *len_out = its length, 0 when absent; buf may be NULL to
 * query the size).  The host picks the message framing from it (generateChat*Response, OllamaService.ts:353-599). */
int  gl_chat_template(const gl_engine* e, char* buf, int32_t cap, int32_t* len_out);

/* ---- the hot path ---------------------------------------------------------------------
 * gl_generate: generateResponse / generateStreamResponse / generateChat*Response
 *   (OllamaService.ts:97-184, 186-284, 353-449, 451-599): prefill the prompt, then decode up to
 *   num_predict tokens; cb (may be NULL) is invoked once per generated token in order.
 *   out_ids / out_logprobs (may be NULL) receive up to num_predict entries.  With gl_engine_opts context_shift on, a prompt of
 *   the context's length or more is cut and generation goes on past the context by shifting the KV cache (rule, bounds and
 *   interactions: gl_engine_opts context_shift). */
int  gl_generate(gl_engine* e, const int32_t* prompt, int32_t n_prompt, const gl_sample_opts* opts,
                 gl_token_cb cb, void* user, int32_t* out_ids, float* out_logprobs, gl_gen_stats* stats);
/* gl_embed: generateEmbedding (OllamaService.ts:601-665): prefill only, output_norm, mean-pool,
 *   L2-normalise. seq_offsets has n_seq+1 entries into ids. out is [n_seq][n_embd].  Sequences are packed into tensor-core prompt
 *   passes whichever source the pass reads its weights from (resident or streamed, gl_engine_opts prefill_mode); a sequence longer
 *   than 2 048 tokens takes passes of its own.  Under prefill_mode 1 every sequence steps through the decode kernels. */
int  gl_embed(gl_engine* e, const int32_t* ids, const int32_t* seq_offsets, int32_t n_seq,
              float* out, gl_gen_stats* stats);
/* ---- continuous batching inside one engine (SURVEY.md section 8f.1) ----------------------------------------------------
 * The reference worker holds one job at a time (WorkerClientService.ts:500-505; MAX_CONCURRENT_JOBS_PER_WORKER,
 * server/src/config/index.ts:31).  With that limit raised the worker opens one sequence per job and steps them TOGETHER:
 * one batched decode step reads the weights once for every open sequence.
 *   gl_seq_open   prefill `prompt` into a free slot's own KV pages and draw its first token (reported by the next
 *                 gl_batch_step); pages for n_prompt + num_predict tokens are reserved up front, so a step cannot run out
 *                 (with batch_prefix_cache, less the prompt prefix it shares).
 *                 GL_ERR_NOMEM when no slot / not enough pages are free -- the caller may retry after a gl_seq_close.
 *                 With context_shift on (gl_engine_opts), a prompt of the context's length or more is cut, pages for
 *                 min(n_prompt + num_predict, W) positions are reserved, and gl_batch_step shifts the KV rows of every
 *                 sequence that reaches the context in one launch before the step.
 *   gl_batch_step one token for every open, unfinished sequence.  Entry i: slots[i], ids[i], logprobs[i], done[i].
 *                 done = 1 with id >= 0: that token was the sequence's last (num_predict reached);  done = 1 with id = -1:
 *                 the token drawn was a stop token (not part of the output).  Finished sequences stay open, holding
 *                 their pages, until gl_seq_close.  *n = entries written (<= cap).
 *   gl_seq_close  return the slot and its pages.
 *   gl_seq_logits logits [n_vocab] the sequence's LAST token was drawn from, penalties and the JSON mask applied (parity
 *                 tests; valid until the next step).
 * Sequences join and leave between steps; a sequence's tokens do not depend on who shares its batch. */
int  gl_seq_open(gl_engine* e, const int32_t* prompt, int32_t n_prompt, const gl_sample_opts* opts, int32_t* slot);
/* Several prompts in one call: they share one packed prompt pass (block-diagonal causal attention, every weight matrix read
 * once per <= 2048 prompt tokens instead of once per prompt) and one lm_head pass for their first tokens.  ids / offsets as for
 * gl_embed (offsets has n_seq + 1 entries), opts has n_seq entries.  Prompts are opened in order until slots or KV pages run
 * out: slots[i] = -1 for those that did not fit (the caller retries them after a gl_seq_close); *n_opened = how many did.
 * GL_ERR_NOMEM only when none could be opened. */
int  gl_seq_open_many(gl_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seq, const gl_sample_opts* opts, int32_t* slots,
                      int32_t* n_opened);
int  gl_batch_step(gl_engine* e, int32_t* slots, int32_t* ids, float* logprobs, int32_t* done, int32_t cap, int32_t* n);
int  gl_seq_close(gl_engine* e, int32_t slot);
int  gl_seq_logits(gl_engine* e, int32_t slot, float* out, int32_t n_vocab);
/* counts and DEVICE durations of one open sequence (InferenceResponse fields, client/src/types/index.ts:39-68):
 * prompt_eval_duration = the prefill of gl_seq_open, eval_duration = the sum of the batched steps it took part in (a step's
 * device time is shared by everyone in it: B sequences each see the whole step), done_reason as for gl_generate. */
int  gl_seq_stats(gl_engine* e, int32_t slot, gl_gen_stats* stats);
/* the bytes of one token as gl_generate's callback would hand them over (may be an incomplete UTF-8 sequence) */
int  gl_token_piece(const gl_engine* e, int32_t id, char* buf, int32_t cap, int32_t* len_out);
/* the vocabulary's own spelling of a token, control tokens included ("<|begin_of_text|>", "</s>", ...; *len_out = 0 without a
 * tokenizer): what a chat template's bos_token / eos_token must be rendered with (generateChat*Response, OllamaService.ts:353-599).
 * gl_token_piece renders control tokens as nothing, which is what a stream wants and a template cannot use. */
int  gl_token_text(const gl_engine* e, int32_t id, char* buf, int32_t cap, int32_t* len_out);
/* engine-wide batching counters since creation (or the last reset): out[0] batched steps, [1] sum over steps of sequences in
 * the step, [2] device ns of those steps, [3] device ns of the prefills of gl_seq_open, [4] prompt tokens prefilled,
 * [5] sequences opened, [6] kernel launches, [7] prompt tokens taken from shared pages (batch_prefix_cache; [4] counts the
 * evaluated ones).  reset != 0 zeroes them after reading. */
int  gl_batch_counters(gl_engine* e, uint64_t out[8], int32_t reset);
/* mean device time (ms) of one batched decode step with `batch` synthetic sequences at context length ctx_len (roofline line
 * of the batched workload); weight_bytes = bytes of weights one such step reads */
int  gl_time_batch_step(gl_engine* e, int32_t batch, int32_t ctx_len, int32_t iters, float* ms_per_step, int32_t* launches_per_step,
                        uint64_t* weight_bytes);

/* logits of generation step i of the last gl_generate that ran with want_logits=1 (after the repetition penalties and the
 * JSON mask, if the request had them: the logits the token was drawn from) */
int  gl_last_logits(gl_engine* e, int32_t step, float* out, int32_t n_vocab);

/* the sampler alone on caller-supplied logits [n_vocab]: the token gl_generate would emit as output number out_index
 * of a request with these options (temperature 0: argmax; else the seeded top-k / top-p / min-p draw), and its log-softmax.
 * No repetition penalty is applied (see gl_penalize_logits).  Parity tests of the draw against oracle/sampler.py (min-p: tests/penalty_oracle.py).  Rewinds
 * the sequence like gl_kv_reset(). */
int  gl_sample_logits(gl_engine* e, const float* logits, int32_t n_vocab, const gl_sample_opts* opts, int32_t out_index,
                      int32_t* id, float* logprob);
/* the repetition-penalty kernel alone, in place on caller-supplied logits [n_vocab], with history[0..n_history) as the
 * sequence's history H (the penalty fields of opts; everything else in opts is ignored).  Parity tests against
 * tests/penalty_oracle.py; hosts may probe for this symbol to learn that the penalty fields are honoured.  Rewinds the sequence
 * like gl_kv_reset(). */
int  gl_penalize_logits(gl_engine* e, float* logits, int32_t n_vocab, const gl_sample_opts* opts, const int32_t* history,
                        int32_t n_history);
/* the JSON grammar mask alone, in place on caller-supplied logits [n_vocab]: the state the device automaton reaches from the
 * initial state through generated[0..n_generated) (the output so far), then the mask kernel (opts->format; format 0 leaves the
 * logits as they are; the stop tokens are eos / eot / opts->stop_ids).  GL_ERR_INVALID when generated is not a prefix the mask
 * allows.  Parity tests against tests/json_oracle.py; hosts may probe for this symbol to learn that format is honoured.
 * Rewinds the sequence like gl_kv_reset(). */
int  gl_constrain_logits(gl_engine* e, float* logits, int32_t n_vocab, const gl_sample_opts* opts, const int32_t* generated,
                         int32_t n_generated);

/* gl_format_schema: compile a JSON schema (Ollama's `format` as an object) and register it with the engine; *format_out gets
 * a code >= GL_FORMAT_SCHEMA_BASE for gl_sample_opts.format.  Identical bytes give the same code.  The engine keeps at most
 * 64 compiled schemas: when full, it evicts the least recently used one that no open sequence uses (GL_ERR_NOMEM when every
 * one is in use).  Codes are never reused; an unknown or evicted code is GL_ERR_INVALID wherever a format is taken.
 * Malformed JSON is GL_ERR_INVALID; a schema outside the subset below is GL_ERR_UNSUPPORTED, with a message that names the
 * keyword and its JSON pointer ("'pattern' is not supported at /properties/zip").
 * A registered schema S restricts the generated bytes to the documents of S, written with the ws rule, the nesting bound (64,
 * root included) and the string / number syntax of the GL_FORMAT_JSON language, and:
 *   - root: an object schema (type "object", properties, or a $ref to one); any other root is refused.
 *   - objects with properties are closed (additionalProperties absent or false).  Keys come in this order: the required
 *     properties in `properties` order, then any subset of the optional ones, in `properties` order (llama.cpp's
 *     json-schema-to-grammar order; unpinned against a real Ollama).  {"type": "object"} without properties is any object.
 *     Refused: additionalProperties true or a schema, a `required` name that is not in `properties`.
 *   - arrays: items (absent: any value), minItems, maxItems.  strings: minLength, maxLength, in code points, an escape counting
 *     as one (so a surrogate pair written as two \u escapes counts as two).  integer: -? (0 | [1-9][0-9]*), no fraction or
 *     exponent.  number, boolean, null; type lists.
 *   - enum / const: strings, integers, booleans, null, spelled canonically: compact, UTF-8 as is, only ", \ and U+0000-U+001F
 *     escaped (\b \f \n \r \t, else \u00xx in lowercase hex) -- Python's json.dumps(ensure_ascii=False).  Keys likewise.
 *   - anyOf / oneOf: only alternatives whose sets of first value bytes are disjoint (X | null, string | integer, ...).  allOf
 *     with one member is that member.  $ref: "#", "#/$defs/..", "#/definitions/..", recursion allowed.
 *   - ignored: title, description, $schema, $id, $comment, examples, default, deprecated, readOnly, writeOnly, discriminator.
 *     Every other keyword is refused (pattern, format, minimum / maximum / exclusive*, multipleOf, uniqueItems, prefixItems,
 *     patternProperties, not, if / then / else, ...).
 *   - no dead ends: a schema whose smallest document nests deeper than 64, an empty enum and min > max are refused; the mask
 *     never opens a container, picks an optional key or starts an array item from which no document closes within the bound.
 *   - limits: <= 4 096 nodes, <= 255 properties per object, counts <= 65 534.
 *   - the vocabulary must have a single-byte token for every byte of the keys and enum members (beside the GL_FORMAT_JSON
 *     requirements), else GL_ERR_UNSUPPORTED.
 * Stop tokens, control tokens, penalties before the mask, the first draw after the prompt, logprobs and gl_*_logits are as for
 * GL_FORMAT_JSON; gl_constrain_logits takes schema codes.  Refused under GL_MEGA=1. */
int  gl_format_schema(gl_engine* e, const char* schema_utf8, int32_t n_bytes, int32_t* format_out);

/* ---- kernel-level entry points (parity tests and roofline measurement) ------------------ */
/* y[rows] = W[rows x cols] (GGUF-layout blocks of ggml_type, host memory) * x[cols].
 * iters>=1 timed launches after 2 warm-ups; kernel_ms = mean device time of one launch. */
int  gl_gemv(gl_engine* e, int ggml_type, const void* w_host, int32_t rows, int32_t cols,
             const float* x, float* y, int32_t iters, float* kernel_ms);
/* device-resident GEMV bandwidth probe on matrix `tensor_name` of the loaded model (no H2D in the
 * timed region); flush_l2!=0 writes a >L2 buffer between iterations. */
int  gl_gemv_model_tensor(gl_engine* e, const char* tensor_name, const float* x, float* y,
                          int32_t iters, int32_t flush_l2, float* kernel_ms, uint64_t* weight_bytes);
/* y = rmsnorm(x) * w (the fused-prologue arithmetic, exposed stand-alone) */
int  gl_rmsnorm(gl_engine* e, const float* x, const float* w, int32_t n, float eps, float* y);
/* one decode step at the engine's current position: feeds `token`, returns logits (may be NULL),
 * greedy id and its logprob.  gl_kv_reset() rewinds the sequence. */
int  gl_decode_step(gl_engine* e, int32_t token, float* logits, int32_t* argmax, float* logprob);
int  gl_kv_reset(gl_engine* e);
int  gl_position(const gl_engine* e, int32_t* pos);
/* batched prefill of n tokens from the current position; logits of the LAST token (may be NULL).  Like gl_generate, gl_seq_open
 * and gl_embed, it takes the tensor-core prompt pass at any length up to the engine's context (passes of 4 096 rows; a pass that
 * does not start at position 0 attends to the earlier positions through the KV pages), and a prompt prefilled in pieces gives
 * the bits of the same prompt in one call.  The pass reads the resident 16-bit copy or streams the layer matrices (gl_engine_opts
 * prefill_mode); both give the same bits.  Under prefill_mode 1, or fewer than 8 tokens, the tokens step through the decode kernels. */
int  gl_prefill(gl_engine* e, const int32_t* ids, int32_t n, float* last_logits);
/* mean device time (ms) of one decode step replayed `iters` times at context length ctx_len
 * (KV content is whatever is resident; used for the roofline line) */
int  gl_time_decode(gl_engine* e, int32_t ctx_len, int32_t iters, float* ms_per_step, int32_t* launches_per_step);

#ifdef __cplusplus
}
#endif
#endif /* GRIDLLM_NATIVE_H */
