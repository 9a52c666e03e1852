"""ctypes binding of ``libgridllm_native.so`` (include/gridllm_native.h).

This is the Python twin of the N-API shim (host/napi/addon.cc): both call exactly the C ABI.
There is no CPU fallback -- if the shared library is missing or no CUDA device is visible,
every entry point raises ``NativeError``.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgridllm_native.so")

GL_OK = 0
GL_ERR_CANCELLED = -7
GL_ERR_NO_DEVICE = -8
STATUS_NAMES = {0: "GL_OK", -1: "GL_ERR_INVALID", -2: "GL_ERR_IO", -3: "GL_ERR_FORMAT", -4: "GL_ERR_UNSUPPORTED",
                -5: "GL_ERR_CUDA", -6: "GL_ERR_NOMEM", -7: "GL_ERR_CANCELLED", -8: "GL_ERR_NO_DEVICE",
                -9: "GL_ERR_CONTEXT"}

# every symbol include/gridllm_native.h declares (tests/test_abi.py checks the library exports all)
ABI_SYMBOLS = [
    "gl_abi_version", "gl_last_error", "gl_device_count", "gl_engine_create", "gl_engine_destroy",
    "gl_engine_info", "gl_tokenize", "gl_detokenize", "gl_chat_template", "gl_generate", "gl_embed", "gl_last_logits", "gl_sample_logits",
    "gl_penalize_logits", "gl_constrain_logits", "gl_format_schema",
    "gl_seq_open", "gl_seq_open_many", "gl_batch_step", "gl_seq_close", "gl_seq_logits", "gl_seq_stats", "gl_token_piece", "gl_token_text", "gl_batch_counters", "gl_time_batch_step",
    "gl_gemv", "gl_gemv_model_tensor", "gl_rmsnorm", "gl_decode_step", "gl_kv_reset", "gl_position",
    "gl_prefill", "gl_time_decode",
]


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{STATUS_NAMES.get(code, code)}: {msg}")
        self.code = code
        self.detail = msg


class EngineOpts(C.Structure):
    _fields_ = [("max_ctx", C.c_int32), ("act_bits", C.c_int32), ("use_graph", C.c_int32), ("use_pdl", C.c_int32),
                ("prefill_mode", C.c_int32), ("max_batch", C.c_int32), ("kv_pool_tokens", C.c_int32), ("batch_weights", C.c_int32),
                ("prefix_cache", C.c_int32), ("reserved", C.c_int32 * 7)]

    GL_OPT_BATCH_PREFIX_CACHE = 0          # include/gridllm_native.h: the reserved word that holds batch_prefix_cache

    @property
    def batch_prefix_cache(self) -> int:
        return self.reserved[self.GL_OPT_BATCH_PREFIX_CACHE]

    @batch_prefix_cache.setter
    def batch_prefix_cache(self, v: int) -> None:
        self.reserved[self.GL_OPT_BATCH_PREFIX_CACHE] = int(v)

    GL_OPT_CONTEXT_SHIFT = 1               # include/gridllm_native.h: the reserved word that holds context_shift

    @property
    def context_shift(self) -> int:
        return self.reserved[self.GL_OPT_CONTEXT_SHIFT]

    @context_shift.setter
    def context_shift(self, v: int) -> None:
        self.reserved[self.GL_OPT_CONTEXT_SHIFT] = int(v)


class ModelInfo(C.Structure):
    _fields_ = [("arch", C.c_char * 32), ("name", C.c_char * 96), ("quantization", C.c_char * 24),
                ("n_layer", C.c_int32), ("n_embd", C.c_int32), ("n_head", C.c_int32), ("n_head_kv", C.c_int32),
                ("head_dim", C.c_int32), ("n_ff", C.c_int32), ("n_vocab", C.c_int32), ("n_ctx_train", C.c_int32),
                ("n_ctx", C.c_int32), ("rope_base", C.c_float), ("rms_eps", C.c_float),
                ("bos_id", C.c_int32), ("eos_id", C.c_int32), ("eot_id", C.c_int32), ("has_tokenizer", C.c_int32),
                ("n_params", C.c_uint64), ("file_bytes", C.c_uint64), ("weight_bytes", C.c_uint64),
                ("decode_bytes_per_token", C.c_uint64), ("device", C.c_int32), ("sm_count", C.c_int32)]


class _FormatWord(C.Union):
    _fields_ = [("format", C.c_int32), ("reserved", C.c_int32 * 1)]


class SampleOpts(C.Structure):
    _anonymous_ = ("_fmt",)
    _fields_ = [("num_predict", C.c_int32), ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("seed", C.c_uint64), ("ignore_eos", C.c_int32), ("n_stop_ids", C.c_int32),
                ("stop_ids", C.POINTER(C.c_int32)), ("want_logits", C.c_int32),
                # repetition penalties and min_p (include/gridllm_native.h); zero = off
                ("repeat_penalty", C.c_float), ("repeat_last_n", C.c_int32), ("presence_penalty", C.c_float),
                ("frequency_penalty", C.c_float), ("min_p", C.c_float),
                # output format (0 off, GL_FORMAT_JSON), in the union with the last reserved word
                ("_fmt", _FormatWord),
                # context shift: prompt positions a shift keeps (-1 the whole prompt); read only with Engine(context_shift=True)
                ("num_keep", C.c_int32)]


GL_FORMAT_JSON = 1
GL_FORMAT_SCHEMA_BASE = 256     # gl_format_schema codes start here


def _format_code(fmt) -> int:
    """the `format` keyword -> gl_sample_opts.format: None / "" / 0 off, "json" (or GL_FORMAT_JSON) the JSON grammar mask"""
    if fmt is None or fmt == "" or fmt == 0:
        return 0
    if fmt == "json" or fmt == GL_FORMAT_JSON:
        return GL_FORMAT_JSON
    raise ValueError(f"format must be None or 'json', not {fmt!r}")

# the keywords of generate / seq_open / seq_open_many / sample_logits that fill the fields above, with values that mean "off"
# (repeat_last_n 64 is Ollama's default window: setting only repeat_penalty penalises the last 64 ids, as Ollama does)
PENALTY_DEFAULTS = {"repeat_penalty": 1.0, "repeat_last_n": 64, "presence_penalty": 0.0, "frequency_penalty": 0.0, "min_p": 0.0}


def _set_penalties(so: SampleOpts, kw: dict) -> None:
    v = dict(PENALTY_DEFAULTS, **{k: x for k, x in kw.items() if x is not None})
    so.repeat_penalty, so.repeat_last_n = float(v["repeat_penalty"]), int(v["repeat_last_n"])
    so.presence_penalty, so.frequency_penalty, so.min_p = float(v["presence_penalty"]), float(v["frequency_penalty"]), float(v["min_p"])


class GenStats(C.Structure):
    _fields_ = [("prompt_eval_count", C.c_int32), ("eval_count", C.c_int32),
                ("prompt_eval_duration_ns", C.c_int64), ("eval_duration_ns", C.c_int64),
                ("total_duration_ns", C.c_int64), ("load_duration_ns", C.c_int64),
                ("done_reason", C.c_int32), ("kernel_launches", C.c_int32)]


TOKEN_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int32, C.c_float, C.POINTER(C.c_char), C.c_int32)

_lib = None


def load_library() -> C.CDLL:
    """Load the in-tree shared library; raise loudly if it was never built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(GL_ERR_NO_DEVICE, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(the native worker has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.gl_last_error.restype = C.c_char_p
    lib.gl_abi_version.restype = C.c_int
    vp, i32, f32p, i32p = C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32)
    lib.gl_device_count.argtypes = [C.POINTER(C.c_int)]
    lib.gl_engine_create.argtypes = [C.c_char_p, C.c_int, C.POINTER(EngineOpts), C.POINTER(vp)]
    lib.gl_engine_destroy.argtypes = [vp]
    lib.gl_engine_destroy.restype = None
    lib.gl_engine_info.argtypes = [vp, C.POINTER(ModelInfo)]
    lib.gl_tokenize.argtypes = [vp, C.c_char_p, i32, C.c_int, C.c_int, i32p, i32, i32p]
    lib.gl_detokenize.argtypes = [vp, i32p, i32, C.c_char_p, i32, i32p]
    lib.gl_chat_template.argtypes = [vp, C.c_char_p, i32, i32p]
    lib.gl_generate.argtypes = [vp, i32p, i32, C.POINTER(SampleOpts), TOKEN_CB, vp, i32p, f32p, C.POINTER(GenStats)]
    lib.gl_embed.argtypes = [vp, i32p, i32p, i32, f32p, C.POINTER(GenStats)]
    lib.gl_last_logits.argtypes = [vp, i32, f32p, i32]
    lib.gl_sample_logits.argtypes = [vp, f32p, i32, C.POINTER(SampleOpts), i32, i32p, f32p]
    lib.gl_penalize_logits.argtypes = [vp, f32p, i32, C.POINTER(SampleOpts), i32p, i32]
    lib.gl_constrain_logits.argtypes = [vp, f32p, i32, C.POINTER(SampleOpts), i32p, i32]
    lib.gl_format_schema.argtypes = [vp, C.c_char_p, i32, i32p]
    lib.gl_seq_open.argtypes = [vp, i32p, i32, C.POINTER(SampleOpts), i32p]
    lib.gl_seq_open_many.argtypes = [vp, i32p, i32p, i32, C.POINTER(SampleOpts), i32p, i32p]
    lib.gl_batch_step.argtypes = [vp, i32p, i32p, f32p, i32p, i32, i32p]
    lib.gl_seq_close.argtypes = [vp, i32]
    lib.gl_seq_logits.argtypes = [vp, i32, f32p, i32]
    lib.gl_seq_stats.argtypes = [vp, i32, C.POINTER(GenStats)]
    lib.gl_token_piece.argtypes = [vp, i32, C.c_char_p, i32, i32p]
    lib.gl_token_text.argtypes = [vp, i32, C.c_char_p, i32, i32p]
    lib.gl_batch_counters.argtypes = [vp, C.POINTER(C.c_uint64), i32]
    lib.gl_time_batch_step.argtypes = [vp, i32, i32, i32, f32p, i32p, C.POINTER(C.c_uint64)]
    lib.gl_gemv.argtypes = [vp, C.c_int, vp, i32, i32, f32p, f32p, i32, f32p]
    lib.gl_gemv_model_tensor.argtypes = [vp, C.c_char_p, f32p, f32p, i32, i32, f32p, C.POINTER(C.c_uint64)]
    lib.gl_rmsnorm.argtypes = [vp, f32p, f32p, i32, C.c_float, f32p]
    lib.gl_decode_step.argtypes = [vp, i32, f32p, i32p, f32p]
    lib.gl_kv_reset.argtypes = [vp]
    lib.gl_position.argtypes = [vp, i32p]
    lib.gl_prefill.argtypes = [vp, i32p, i32, f32p]
    lib.gl_time_decode.argtypes = [vp, i32, i32, f32p, i32p]
    _lib = lib
    return lib


def _check(rc: int):
    if rc != GL_OK:
        raise NativeError(rc, (load_library().gl_last_error() or b"").decode("utf-8", "replace"))


def device_count() -> int:
    n = C.c_int(0)
    rc = load_library().gl_device_count(C.byref(n))
    return n.value if rc == GL_OK else 0


def _f32p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _i32p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


@dataclass
class Generation:
    ids: np.ndarray
    logprobs: np.ndarray
    stats: GenStats


class Engine:
    """One GGUF model resident on one GPU (gl_engine)."""

    def __init__(self, gguf_path: str, device: int = 0, max_ctx: int = 0, act_bits: int = 16, use_graph: bool = True,
                 use_pdl: bool = True, prefill_mode: int = 0, max_batch: int = 0, kv_pool_tokens: int = 0, batch_weights: int = 0,
                 prefix_cache: bool = False, batch_prefix_cache: bool = False, context_shift: bool = False):
        self._lib = load_library()
        self._h = C.c_void_p()
        o = EngineOpts()
        o.max_ctx, o.act_bits, o.use_graph, o.use_pdl = max_ctx, act_bits, int(use_graph), int(use_pdl)
        o.prefill_mode = prefill_mode   # 0 auto (batched tensor-core prefill), 1 sequential decode steps
        # continuous batching: sequences open at once (gl_seq_open), the KV pool they share, and which weights the batched step reads
        o.max_batch, o.kv_pool_tokens, o.batch_weights = int(max_batch), int(kv_pool_tokens), int(batch_weights)
        # generate() keeps the KV pages of the longest prefix it shares with the previous generate() (include/gridllm_native.h)
        o.prefix_cache = int(bool(prefix_cache))
        # seq_open / seq_open_many sequences share the KV pages of prompt prefixes, also with closed ones (include/gridllm_native.h)
        o.batch_prefix_cache = int(bool(batch_prefix_cache))
        # a sequence that fills the context keeps generating: over-long prompts are cut and the KV cache shifts (include/gridllm_native.h)
        o.context_shift = int(bool(context_shift))
        _check(self._lib.gl_engine_create(gguf_path.encode(), device, C.byref(o), C.byref(self._h)))
        self.info = ModelInfo()
        _check(self._lib.gl_engine_info(self._h, C.byref(self.info)))
        self.path = gguf_path

    def close(self):
        if self._h:
            self._lib.gl_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- tokenizer -------------------------------------------------------------------------
    def tokenize(self, text: str, add_bos: bool = True, parse_special: bool = True) -> np.ndarray:
        raw = text.encode("utf-8")
        cap = len(raw) + 8
        ids = np.empty(cap, dtype=np.int32)
        n = C.c_int32(0)
        _check(self._lib.gl_tokenize(self._h, raw, len(raw), int(add_bos), int(parse_special), _i32p(ids), cap, C.byref(n)))
        return ids[: n.value].copy()

    def detokenize(self, ids: Sequence[int]) -> str:
        a = np.ascontiguousarray(ids, dtype=np.int32)
        cap = 16 * max(1, len(a)) + 16
        buf = C.create_string_buffer(cap)
        n = C.c_int32(0)
        _check(self._lib.gl_detokenize(self._h, _i32p(a), len(a), buf, cap, C.byref(n)))
        return buf.raw[: n.value].decode("utf-8", "replace")

    @property
    def chat_template(self) -> str:
        """tokenizer.chat_template of the GGUF ('' when absent)"""
        n = C.c_int32(0)
        _check(self._lib.gl_chat_template(self._h, None, 0, C.byref(n)))
        if n.value <= 0:
            return ""
        buf = C.create_string_buffer(n.value)
        _check(self._lib.gl_chat_template(self._h, buf, n.value, C.byref(n)))
        return buf.raw[: n.value].decode("utf-8", "replace")

    # ---- hot path ---------------------------------------------------------------------------
    def generate(self, prompt: Sequence[int], num_predict: int = 128, ignore_eos: bool = False,
                 on_token: Optional[Callable[[int, float, bytes], bool]] = None, want_logits: bool = False,
                 stop_ids: Sequence[int] = (), temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0,
                 seed: int = 0, repeat_penalty: float = 1.0, repeat_last_n: int = 64, presence_penalty: float = 0.0,
                 frequency_penalty: float = 0.0, min_p: float = 0.0, format: Optional[str] = None, num_keep: int = 0) -> Generation:
        p = np.ascontiguousarray(prompt, dtype=np.int32)
        so = SampleOpts()
        so.num_predict, so.ignore_eos, so.want_logits = num_predict, int(ignore_eos), int(want_logits)
        so.num_keep = int(num_keep)
        so.format = self._format(format)
        so.temperature, so.top_k, so.top_p, so.seed = float(temperature), int(top_k), float(top_p), int(seed) & (2**64 - 1)
        _set_penalties(so, dict(repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n, presence_penalty=presence_penalty,
                                frequency_penalty=frequency_penalty, min_p=min_p))
        stops = np.ascontiguousarray(stop_ids, dtype=np.int32)
        so.n_stop_ids = len(stops)
        so.stop_ids = _i32p(stops) if len(stops) else None
        # the library maps num_predict <= 0 to 128 (OllamaService.ts:105): size the output buffers from the same rule, never
        # from the raw argument (a 0-length buffer would be written past its end)
        n_out = num_predict if num_predict > 0 else 128
        so.num_predict = n_out
        ids = np.zeros(n_out, dtype=np.int32)
        lps = np.zeros(n_out, dtype=np.float32)
        st = GenStats()

        def _cb(_user, tid, lp, piece, plen):
            data = C.string_at(piece, plen) if piece and plen > 0 else b""
            return 1 if on_token(int(tid), float(lp), data) else 0

        cb = TOKEN_CB(_cb) if on_token is not None else TOKEN_CB()
        rc = self._lib.gl_generate(self._h, _i32p(p), len(p), C.byref(so), cb, None, _i32p(ids), _f32p(lps), C.byref(st))
        if rc != GL_OK and rc != GL_ERR_CANCELLED:
            _check(rc)
        return Generation(ids[: st.eval_count].copy(), lps[: st.eval_count].copy(), st)

    # ---- continuous batching (gl_seq_open / gl_batch_step / gl_seq_close) ---------------------------------
    def seq_open(self, prompt: Sequence[int], num_predict: int = 128, ignore_eos: bool = False, temperature: float = 0.0, top_k: int = 0,
                 top_p: float = 1.0, seed: int = 0, stop_ids: Sequence[int] = (), repeat_penalty: float = 1.0, repeat_last_n: int = 64,
                 presence_penalty: float = 0.0, frequency_penalty: float = 0.0, min_p: float = 0.0, format: Optional[str] = None,
                 num_keep: int = 0) -> int:
        p = np.ascontiguousarray(prompt, dtype=np.int32)
        so = SampleOpts()
        so.num_predict, so.ignore_eos = (num_predict if num_predict > 0 else 128), int(ignore_eos)
        so.num_keep = int(num_keep)
        so.format = self._format(format)
        so.temperature, so.top_k, so.top_p, so.seed = float(temperature), int(top_k), float(top_p), int(seed) & (2**64 - 1)
        _set_penalties(so, dict(repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n, presence_penalty=presence_penalty,
                                frequency_penalty=frequency_penalty, min_p=min_p))
        stops = np.ascontiguousarray(stop_ids, dtype=np.int32)
        so.n_stop_ids = len(stops)
        so.stop_ids = _i32p(stops) if len(stops) else None
        slot = C.c_int32(-1)
        _check(self._lib.gl_seq_open(self._h, _i32p(p), len(p), C.byref(so), C.byref(slot)))
        return int(slot.value)

    def seq_open_many(self, prompts: Sequence[Sequence[int]], options: Sequence[dict]) -> List[int]:
        """Open several sequences with ONE packed prompt pass (gl_seq_open_many).  options[i]: the keyword arguments of seq_open
        for prompt i.  Returns one slot per prompt, -1 for those that did not fit (no free slot / KV pages) -- retry them later."""
        n = len(prompts)
        offs = np.zeros(n + 1, dtype=np.int32)
        for i, p in enumerate(prompts):
            offs[i + 1] = offs[i] + len(p)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.int32) for p in prompts]), dtype=np.int32)
        so = (SampleOpts * n)()
        keep = []                                      # stop-id arrays must outlive the call
        for i, o in enumerate(options):
            np_ = int(o.get("num_predict", 128))
            so[i].num_predict, so[i].ignore_eos = (np_ if np_ > 0 else 128), int(bool(o.get("ignore_eos", False)))
            so[i].temperature, so[i].top_k, so[i].top_p = float(o.get("temperature", 0.0)), int(o.get("top_k", 0)), float(o.get("top_p", 1.0))
            so[i].seed = int(o.get("seed", 0)) & (2**64 - 1)
            _set_penalties(so[i], {k: o.get(k) for k in PENALTY_DEFAULTS})
            so[i].format = self._format(o.get("format"))
            so[i].num_keep = int(o.get("num_keep", 0))
            stops = np.ascontiguousarray(o.get("stop_ids", ()), dtype=np.int32)
            keep.append(stops)
            so[i].n_stop_ids = len(stops)
            so[i].stop_ids = _i32p(stops) if len(stops) else None
        slots = np.full(n, -1, dtype=np.int32)
        k = C.c_int32(0)
        _check(self._lib.gl_seq_open_many(self._h, _i32p(ids), _i32p(offs), n, so, _i32p(slots), C.byref(k)))
        return [int(x) for x in slots]

    def batch_step(self, cap: int = 128):
        """-> [(slot, token id, logprob, done)]: one entry per open, unfinished sequence.  id -1 with done: a stop token was drawn."""
        slots, ids, done = (np.zeros(cap, np.int32) for _ in range(3))
        lps = np.zeros(cap, np.float32)
        n = C.c_int32(0)
        _check(self._lib.gl_batch_step(self._h, _i32p(slots), _i32p(ids), _f32p(lps), _i32p(done), cap, C.byref(n)))
        return [(int(slots[i]), int(ids[i]), float(lps[i]), bool(done[i])) for i in range(n.value)]

    def seq_close(self, slot: int) -> None:
        _check(self._lib.gl_seq_close(self._h, int(slot)))

    def seq_logits(self, slot: int) -> np.ndarray:
        out = np.empty(self.info.n_vocab, dtype=np.float32)
        _check(self._lib.gl_seq_logits(self._h, int(slot), _f32p(out), self.info.n_vocab))
        return out

    def seq_stats(self, slot: int) -> GenStats:
        st = GenStats()
        _check(self._lib.gl_seq_stats(self._h, int(slot), C.byref(st)))
        return st

    def token_piece(self, tid: int) -> bytes:
        """the bytes of one token, as gl_generate's callback hands them over (b'' when the model has no tokenizer)"""
        buf = C.create_string_buffer(256)
        n = C.c_int32(0)
        _check(self._lib.gl_token_piece(self._h, int(tid), buf, 256, C.byref(n)))
        return buf.raw[: n.value]

    def token_text(self, tid: int) -> str:
        """the vocabulary's spelling of a token, control tokens included ('' when the model has no tokenizer): bos_token / eos_token
        of a chat template"""
        buf = C.create_string_buffer(512)
        n = C.c_int32(0)
        _check(self._lib.gl_token_text(self._h, int(tid), buf, 512, C.byref(n)))
        return buf.raw[: n.value].decode("utf-8", "replace")

    def batch_counters(self, reset: bool = False) -> dict:
        out = (C.c_uint64 * 8)()
        _check(self._lib.gl_batch_counters(self._h, out, int(reset)))
        return {"steps": out[0], "rows": out[1], "step_ns": out[2], "prefill_ns": out[3], "prefill_tokens": out[4], "sequences": out[5],
                "launches": out[6], "shared_tokens": out[7]}

    def time_batch_step(self, batch: int, ctx_len: int, iters: int = 16):
        """-> (ms per batched step, kernel launches per step, weight bytes one step reads)"""
        ms, nl, wb = C.c_float(0), C.c_int32(0), C.c_uint64(0)
        _check(self._lib.gl_time_batch_step(self._h, batch, ctx_len, iters, C.byref(ms), C.byref(nl), C.byref(wb)))
        return ms.value, nl.value, wb.value

    def sample_logits(self, logits: np.ndarray, temperature: float, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
                      out_index: int = 0, min_p: float = 0.0):
        """The sampler alone (gl_sample_logits): (token id, logprob) for output number out_index of such a request."""
        a = np.ascontiguousarray(logits, dtype=np.float32)
        so = SampleOpts()
        so.num_predict, so.ignore_eos = 1, 1
        so.temperature, so.top_k, so.top_p, so.seed = float(temperature), int(top_k), float(top_p), int(seed) & (2**64 - 1)
        _set_penalties(so, dict(min_p=min_p))
        tid, lp = C.c_int32(0), C.c_float(0.0)
        _check(self._lib.gl_sample_logits(self._h, _f32p(a), len(a), C.byref(so), out_index, C.byref(tid), C.byref(lp)))
        return int(tid.value), float(lp.value)

    def penalize_logits(self, logits: np.ndarray, history: Sequence[int], repeat_penalty: float = 1.0, repeat_last_n: int = 64,
                        presence_penalty: float = 0.0, frequency_penalty: float = 0.0) -> np.ndarray:
        """The repetition-penalty kernel alone (gl_penalize_logits): a penalised copy of `logits` for a sequence whose history
        (prompt ids, then generated ids) is `history`."""
        out = np.array(logits, dtype=np.float32, copy=True)
        h = np.ascontiguousarray(history, dtype=np.int32)
        so = SampleOpts()
        so.num_predict, so.ignore_eos = 1, 1
        _set_penalties(so, dict(repeat_penalty=repeat_penalty, repeat_last_n=repeat_last_n, presence_penalty=presence_penalty,
                                frequency_penalty=frequency_penalty))
        _check(self._lib.gl_penalize_logits(self._h, _f32p(out), len(out), C.byref(so), _i32p(h) if len(h) else None, len(h)))
        return out

    def constrain_logits(self, logits: np.ndarray, generated: Sequence[int], format: Optional[str] = "json",
                         stop_ids: Sequence[int] = ()) -> np.ndarray:
        """The JSON grammar mask alone (gl_constrain_logits): a masked copy of `logits` for the draw that follows the output
        `generated` (token ids after the prompt).  NativeError GL_ERR_INVALID when `generated` is not a prefix the mask allows."""
        out = np.array(logits, dtype=np.float32, copy=True)
        g = np.ascontiguousarray(generated, dtype=np.int32)
        so = SampleOpts()
        so.num_predict = 1
        so.format = self._format(format)
        stops = np.ascontiguousarray(stop_ids, dtype=np.int32)
        so.n_stop_ids = len(stops)
        so.stop_ids = _i32p(stops) if len(stops) else None
        _check(self._lib.gl_constrain_logits(self._h, _f32p(out), len(out), C.byref(so), _i32p(g) if len(g) else None, len(g)))
        return out

    def format_schema(self, schema) -> int:
        """Compile and register a JSON schema (gl_format_schema): its code for `format=`.  A dict is serialised compactly with
        its key order kept; a str / bytes is taken as it is.  Identical text gives the same code.  NativeError GL_ERR_INVALID
        for malformed JSON, GL_ERR_UNSUPPORTED for a schema outside the subset (the message names the keyword and its
        JSON pointer)."""
        if isinstance(schema, dict):
            schema = json.dumps(schema, ensure_ascii=False, separators=(",", ":"))
        raw = schema.encode("utf-8") if isinstance(schema, str) else bytes(schema)
        code = C.c_int32(0)
        _check(self._lib.gl_format_schema(self._h, raw, len(raw), C.byref(code)))
        return int(code.value)

    def _format(self, fmt) -> int:
        """the `format` keyword: None / "" / 0 off, "json" the JSON grammar mask, a dict a JSON schema (compiled through the
        engine's cache), or a code from format_schema"""
        if isinstance(fmt, dict):
            return self.format_schema(fmt)
        if isinstance(fmt, int) and not isinstance(fmt, bool) and fmt >= GL_FORMAT_SCHEMA_BASE:
            return fmt
        return _format_code(fmt)

    def last_logits(self, step: int) -> np.ndarray:
        out = np.empty(self.info.n_vocab, dtype=np.float32)
        _check(self._lib.gl_last_logits(self._h, step, _f32p(out), self.info.n_vocab))
        return out

    def embed(self, seqs: Sequence[Sequence[int]]):
        offs = np.zeros(len(seqs) + 1, dtype=np.int32)
        for i, s in enumerate(seqs):
            offs[i + 1] = offs[i] + len(s)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int32) for s in seqs]), dtype=np.int32)
        out = np.empty((len(seqs), self.info.n_embd), dtype=np.float32)
        st = GenStats()
        _check(self._lib.gl_embed(self._h, _i32p(ids), _i32p(offs), len(seqs), _f32p(out), C.byref(st)))
        return out, st

    # ---- kernel-level -----------------------------------------------------------------------
    def gemv(self, ggml_type: int, w_blocks: np.ndarray, rows: int, cols: int, x: np.ndarray, iters: int = 1):
        w = np.ascontiguousarray(w_blocks).view(np.uint8)
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty(rows, dtype=np.float32)
        ms = C.c_float(0)
        _check(self._lib.gl_gemv(self._h, ggml_type, w.ctypes.data_as(C.c_void_p), rows, cols, _f32p(x), _f32p(y), iters, C.byref(ms)))
        return y, ms.value

    def gemv_tensor(self, name: str, x: np.ndarray, iters: int = 10, flush_l2: bool = True):
        x = np.ascontiguousarray(x, dtype=np.float32)
        rows = {"output.weight": self.info.n_vocab}.get(name)
        y = np.empty(max(self.info.n_vocab, self.info.n_ff, self.info.n_embd), dtype=np.float32)
        ms = C.c_float(0)
        wb = C.c_uint64(0)
        _check(self._lib.gl_gemv_model_tensor(self._h, name.encode(), _f32p(x), _f32p(y), iters, int(flush_l2), C.byref(ms), C.byref(wb)))
        return y, ms.value, wb.value

    def rmsnorm(self, x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        w = np.ascontiguousarray(w, dtype=np.float32)
        y = np.empty_like(x)
        _check(self._lib.gl_rmsnorm(self._h, _f32p(x), _f32p(w), len(x), eps, _f32p(y)))
        return y

    def decode_step(self, token: int, want_logits: bool = True):
        logits = np.empty(self.info.n_vocab, dtype=np.float32) if want_logits else None
        am = C.c_int32(0)
        lp = C.c_float(0)
        _check(self._lib.gl_decode_step(self._h, int(token), _f32p(logits) if want_logits else None, C.byref(am), C.byref(lp)))
        return logits, am.value, lp.value

    def kv_reset(self):
        _check(self._lib.gl_kv_reset(self._h))

    def position(self) -> int:
        p = C.c_int32(0)
        _check(self._lib.gl_position(self._h, C.byref(p)))
        return p.value

    def prefill(self, ids: Sequence[int], want_logits: bool = True):
        a = np.ascontiguousarray(ids, dtype=np.int32)
        logits = np.empty(self.info.n_vocab, dtype=np.float32) if want_logits else None
        _check(self._lib.gl_prefill(self._h, _i32p(a), len(a), _f32p(logits) if want_logits else None))
        return logits

    def time_decode(self, ctx_len: int, iters: int = 32):
        ms = C.c_float(0)
        nl = C.c_int32(0)
        _check(self._lib.gl_time_decode(self._h, ctx_len, iters, C.byref(ms), C.byref(nl)))
        return ms.value, nl.value
