"""NativeInferenceService -- the drop-in for the reference's ``OllamaService``.

Mirrors /root/reference/client/src/services/OllamaService.ts method for method (same names,
same request / response dictionaries as client/src/types/index.ts:1-27,39-74, same
"<Kind> failed: <message>" error convention the worker turns into job:failed), but instead of an
HTTP call to an Ollama daemon every method calls the in-process native engine through the C ABI
(gridllm_b200/native.py -> libgridllm_native.so).  The TypeScript twin that a GridLLM
maintainer would actually ship is host/src/NativeInferenceService.ts over host/napi/addon.cc;
node is not present in this image, so this Python class is the executable host side.

All generate* calls run the blocking native call on a worker thread (``asyncio.to_thread``) so the
event loop keeps servicing heartbeats, exactly like napi_create_async_work in the N-API shim.
"""
from __future__ import annotations

import asyncio
import hashlib
import os
import secrets
import threading
import time
from datetime import datetime, timezone
from typing import Any, AsyncGenerator, Dict, List, Optional

import numpy as np

from . import native as N

InferenceRequest = Dict[str, Any]
InferenceResponse = Dict[str, Any]
StreamResponse = Dict[str, Any]


def _now_iso() -> str:
    return datetime.now(timezone.utc).isoformat(timespec="milliseconds").replace("+00:00", "Z")


class StopFilter:
    """options.stop (forwarded by the reference: OllamaService.ts:101-134): generation ends at the first occurrence of a stop
    string in the GENERATED TEXT; the stop string is not part of the response.  A stop string can span tokens, so text that
    could still turn into one is held back (what Ollama's runner does for streamed responses [external])."""

    def __init__(self, stops: List[str]):
        self.stops = [s for s in stops if s]
        self.text = ""        # released text (the response so far)
        self.held = ""        # decoded but not yet released: a prefix of some stop string
        self._bytes = b""     # bytes of an incomplete UTF-8 character
        self.hit = False

    def feed(self, piece: bytes) -> str:
        """-> the text this token releases ('' while a possible stop string is pending); sets .hit when a stop string completed"""
        if self.hit:
            return ""
        self._bytes += piece or b""
        try:
            new = self._bytes.decode("utf-8")
            self._bytes = b""
        except UnicodeDecodeError:
            return ""
        buf = self.held + new
        cut = min((i for i in (buf.find(s) for s in self.stops) if i >= 0), default=-1)
        if cut >= 0:
            self.hit = True
            out, self.held = buf[:cut], ""
        else:
            keep = 0          # longest suffix of buf that is a proper prefix of a stop string
            for s in self.stops:
                for n in range(min(len(s) - 1, len(buf)), 0, -1):
                    if buf.endswith(s[:n]):
                        keep = max(keep, n)
                        break
            out, self.held = buf[:len(buf) - keep], buf[len(buf) - keep:]
        self.text += out
        return out

    def flush(self) -> str:
        """generation ended without a stop string: release what was held back"""
        out = "" if self.hit else self.held + self._bytes.decode("utf-8", "replace")
        self.held, self._bytes = "", b""
        self.text += out
        return out


class NativeInferenceService:
    """One engine = one GPU = one loaded model (SURVEY.md section 8e: one service per worker id)."""

    # what Ollama applies when a request leaves the sampling options out [external: Ollama's documented parameter defaults]
    OLLAMA_SAMPLING_DEFAULTS = {"temperature": 0.8, "top_k": 40, "top_p": 0.9}
    # Ollama's defaults for the repetition penalty [external: Ollama's documented parameter defaults]; opt-in, like the dict above
    OLLAMA_PENALTY_DEFAULTS = {"repeat_penalty": 1.1, "repeat_last_n": 64}
    PENALTY_OPTIONS = ("repeat_penalty", "repeat_last_n", "presence_penalty", "frequency_penalty", "min_p")

    def __init__(self, models: Dict[str, str], device: int = 0, max_ctx: int = 0,
                 sampling_defaults: Optional[Dict[str, Any]] = None, apply_template: bool = False, max_batch: int = 0,
                 jinja_templates: bool = True, penalty_defaults: Optional[Dict[str, Any]] = None, json_schema: bool = False,
                 context_shift: bool = False, **engine_kw):
        """models: Ollama-style model name -> GGUF path.
        sampling_defaults: options a request inherits when it does not carry them.  None = greedy (temperature 0, the
        BASELINE.json configuration); pass OLLAMA_SAMPLING_DEFAULTS to behave like an Ollama worker for such requests.
        apply_template: frame generate / completion prompts as one user turn of the model's chat template (with
        metadata.system as the system turn) unless metadata.raw, as Ollama does; default False = raw prompts.
        max_batch: > 1 turns on continuous batching (SURVEY.md section 8f.1): concurrent generate* calls become sequences of
        one engine and are decoded together, one batched step per token (gridllm_b200/batching.py); 0 / 1 = one request at a time.
        jinja_templates: render tokenizer.chat_template as Jinja for chat requests (default); False = family framing only.
        penalty_defaults: repetition-penalty options a request inherits when it does not carry them.  None = no penalty; pass
        OLLAMA_PENALTY_DEFAULTS to penalise like an Ollama worker.
        json_schema: enforce a JSON-schema `format` (metadata.format or options.format) on the GPU: the response is a document
        of the schema, and a schema outside the supported subset fails the request before it runs.  False (default): a schema
        object only asks for valid JSON of any shape.
        context_shift: keep answering when a conversation outgrows the engine's context, as Ollama does: a prompt of the
        context's length or more is cut to its first options.num_keep tokens (default 4, -1 the whole prompt) plus its newest
        ones, and a generation that reaches the context shifts the KV cache instead of stopping.  num_predict is then bounded
        by the context itself (<= 0 means the context's length), not by what is left of it.  The returned context is still
        the whole conversation as sent plus the reply.  Off by default: a generation ends at the context and a prompt that
        does not fit fails.
        engine_kw: further Engine options, e.g. prefix_cache=True: a request keeps the KV pages of the longest prefix it shares
        with the previous request on the same engine (a multi-turn client that sends metadata.context back then pays for its
        new tokens only, as with Ollama's cached prefix), and its prompt_eval_count counts the tokens it evaluated.  Off by
        default, like the other Ollama-behaviour switches.  prefix_cache covers one request at a time; with max_batch > 1 pass
        batch_prefix_cache=True instead: the batch runner's sequences share the KV pages of prompt prefixes, with each other
        and with sequences that have closed (a common system prompt, or a chat's earlier turns, is evaluated once), and
        prompt_eval_count counts the tokens each one evaluated."""
        self._sampling_defaults = dict(sampling_defaults or {})
        self._penalty_defaults = dict(penalty_defaults or {})
        self._json_schema = bool(json_schema)
        self._context_shift = bool(context_shift)
        # Ollama wraps the prompt of /api/generate and /v1/completions in the model's template (system + prompt as one user
        # turn) unless the request says raw [external]; off by default: the prompt text is tokenised as it is
        self._apply_template = bool(apply_template)
        # chat messages are framed by RENDERING the GGUF's tokenizer.chat_template (Jinja); False = by template family only
        self._jinja = bool(jinja_templates)
        self._paths = dict(models)
        self._device = device
        self._max_ctx = max_ctx
        self._engine_kw = dict(engine_kw, context_shift=True) if self._context_shift else engine_kw
        self._max_batch = int(max_batch) if int(max_batch) > 1 else 0
        if self._max_batch:
            self._engine_kw = dict(self._engine_kw, max_batch=self._max_batch)
        self._runners: Dict[str, Any] = {}
        self._engines: Dict[str, N.Engine] = {}
        self._lock = threading.Lock()          # one engine call at a time (one CUDA stream per engine)
        self._load_lock = threading.Lock()     # model load: once, and never on the event-loop thread (see _engine_async)
        self.isConnected = False
        self.lastHealthCheck = datetime.now(timezone.utc)

    # ---- engine management -------------------------------------------------------------------
    def _engine(self, name: str) -> N.Engine:
        if name not in self._paths:
            raise RuntimeError(f"model '{name}' not found")
        with self._load_lock:
            if name not in self._engines:
                self._engines[name] = N.Engine(self._paths[name], device=self._device, max_ctx=self._max_ctx, **self._engine_kw)
            return self._engines[name]

    async def _engine_async(self, name: str) -> N.Engine:
        """The first request for a model loads it (mmap, host repack, H2D of several GB, graph capture): seconds during which
        the event loop must keep firing heartbeats (the server drops a worker after WORKER_HEARTBEAT_TIMEOUT = 15 s,
        server/src/config/index.ts:24) -- so the load runs on a worker thread, like every other engine call."""
        if name in self._engines:
            return self._engines[name]
        return await asyncio.to_thread(self._engine, name)

    def preload(self) -> None:
        """load every configured model now (NativeWorker.start() calls this before registering)"""
        for name in self._paths:
            self._engine(name)

    @staticmethod
    def _num_predict(options: Dict[str, Any]) -> int:
        """options.num_predict (OllamaService.ts:105: `options.num_predict || 128`).  The gateway also lets -1 / -2 through
        (ollama.ts:47, Ollama's "until EOS / fill the context"): those become "as many as the context holds" in _run."""
        v = options.get("num_predict")
        if v is None or v == 0:
            return 128
        return int(v)

    NUM_KEEP_DEFAULT = 4        # this project's choice (Ollama's own default is not pinned here)

    @classmethod
    def _num_keep(cls, options: Dict[str, Any]) -> int:
        """options.num_keep: the prompt tokens a context shift keeps; absent -> 4, -1 the whole prompt"""
        v = options.get("num_keep")
        if v is None:
            return cls.NUM_KEEP_DEFAULT
        v = int(v)
        if v < -1:
            raise RuntimeError("num_keep must be >= -1")
        return v

    def close(self):
        for r in self._runners.values():
            r.close()
        self._runners.clear()
        for e in self._engines.values():
            e.close()
        self._engines.clear()

    def _runner(self, name: str):
        """the batch runner of a model's engine (continuous batching; one thread per engine)"""
        with self._load_lock:
            r = self._runners.get(name)
        if r is None:
            eng = self._engine(name)
            from .batching import BatchRunner
            with self._load_lock:
                r = self._runners.get(name)
                if r is None:
                    r = self._runners[name] = BatchRunner(eng, self._lock, self._max_batch, N.Generation)
        return r

    # ---- OllamaService.checkHealth (OllamaService.ts:65-83) ------------------------------------
    async def checkHealth(self) -> bool:
        try:
            self.isConnected = N.device_count() > self._device
        except Exception:
            self.isConnected = False
        self.lastHealthCheck = datetime.now(timezone.utc)
        return self.isConnected

    # ---- OllamaService.getAvailableModels (:85-95); OllamaModel shape client/src/types/index.ts:76-88
    async def getAvailableModels(self) -> List[Dict[str, Any]]:
        try:
            out = []
            for name, path in self._paths.items():
                st = os.stat(path)
                info = self._engines[name].info if name in self._engines else None
                details = {"format": "gguf", "family": "llama", "families": ["llama"],
                           "parameter_size": f"{info.n_params / 1e9:.1f}B" if info else "",
                           "quantization_level": info.quantization.decode() if info else ""}
                digest = hashlib.sha256(f"{path}:{st.st_size}:{int(st.st_mtime)}".encode()).hexdigest()
                out.append({"name": name, "digest": digest, "size": st.st_size,
                            "modified_at": datetime.fromtimestamp(st.st_mtime, timezone.utc).isoformat().replace("+00:00", "Z"),
                            "details": details})
            return out
        except Exception:
            raise RuntimeError("Failed to retrieve available models from Ollama")

    # ---- OllamaService.validateModel (:340-351): O(1) instead of a /api/tags round trip -----------
    async def validateModel(self, modelName: str) -> bool:
        return modelName in self._paths and os.path.exists(self._paths[modelName])

    def getConnectionStatus(self) -> Dict[str, Any]:
        return {"isConnected": self.isConnected, "lastHealthCheck": self.lastHealthCheck}

    # ---- prompt handling ------------------------------------------------------------------------
    def _prompt_ids(self, eng: N.Engine, request: InferenceRequest, text: Optional[str]) -> np.ndarray:
        md = request.get("metadata") or {}
        if md.get("prompt_token_ids") is not None:      # synthetic workloads: token-id prompts (SURVEY.md section 7)
            return np.asarray(md["prompt_token_ids"], dtype=np.int32)
        if not eng.info.has_tokenizer:
            raise RuntimeError("model carries no tokenizer; supply metadata.prompt_token_ids")
        ctx = md.get("context")                          # token ids of the conversation so far (OllamaService.ts:224-226)
        if self._apply_template and not md.get("raw") and not ctx:      # metadata.system / raw: OllamaService.ts:212-220
            msgs = ([{"role": "system", "content": md["system"]}] if md.get("system") else []) + [{"role": "user", "content": text or ""}]
            return eng.tokenize(self._chat_prompt(eng, msgs), add_bos=True, parse_special=True)
        if ctx:
            new = eng.tokenize(text or "", add_bos=False, parse_special=False)
            return np.concatenate([np.asarray(ctx, dtype=np.int32), np.asarray(new, dtype=np.int32)])
        return eng.tokenize(text or "", add_bos=True, parse_special=False)

    @staticmethod
    def _control_text(eng: N.Engine, tid) -> str:
        """the vocabulary text of a (control) token: gl_token_text where the engine has it; gl_token_piece renders control tokens
        as nothing (what a stream wants), so for an engine without the call the text is found by asking the tokenizer which known
        spelling parses to this id"""
        try:
            if tid is None or int(tid) < 0:
                return ""
            tt = getattr(eng, "token_text", None)              # gl_token_text: the spelling straight from the vocabulary
            if tt is not None:
                txt = tt(int(tid))
                if txt:
                    return txt
            txt = eng.token_piece(int(tid)).decode("utf-8", "replace")
            if txt:
                return txt
            for cand in ("<|begin_of_text|>", "<|end_of_text|>", "<|eot_id|>", "<s>", "</s>", "<|im_start|>", "<|im_end|>",
                         "<|endoftext|>", "<bos>", "<eos>", "<|startoftext|>"):
                ids = eng.tokenize(cand, add_bos=False, parse_special=True)
                if len(ids) == 1 and int(ids[0]) == int(tid):
                    return cand
        except Exception:
            pass
        return ""

    def _render_jinja(self, eng: N.Engine, tmpl: str, messages: List[Dict[str, Any]]) -> Optional[str]:
        """tokenizer.chat_template interpreted as what it is -- a Jinja program -- the way Ollama's runner and Hugging Face
        `apply_chat_template` do [external]: sandboxed environment, `messages`, `add_generation_prompt = True`, `bos_token` /
        `eos_token` (the GGUF's own token texts) and `raise_exception`.  None when the template cannot be rendered (a construct
        outside Jinja, a variable the host does not supply, a role the template refuses): the caller falls back to the
        template FAMILY.  A leading BOS text is dropped: the tokenizer adds the BOS id itself."""
        try:
            import jinja2
            from jinja2.sandbox import ImmutableSandboxedEnvironment
        except Exception:
            return None
        try:
            cache = self.__dict__.setdefault("_tmpl_cache", {})       # compiled templates, by template text
            if tmpl not in cache:
                env = ImmutableSandboxedEnvironment(trim_blocks=True, lstrip_blocks=True, undefined=jinja2.StrictUndefined)

                def raise_exception(msg):
                    raise jinja2.exceptions.TemplateError(msg)
                env.globals["raise_exception"] = raise_exception
                cache[tmpl] = env.from_string(tmpl)
            t = cache[tmpl]
            # the BOS / EOS spellings belong to the engine's vocabulary: kept on the engine object, not beside the template
            ctrl = getattr(eng, "_gl_ctrl_text", None)
            if ctrl is None:
                ctrl = (self._control_text(eng, getattr(eng.info, "bos_id", -1)), self._control_text(eng, getattr(eng.info, "eos_id", -1)))
                try:
                    eng._gl_ctrl_text = ctrl
                except Exception:
                    pass
            bos, eos = ctrl
            out = t.render(messages=[dict(m) for m in messages], add_generation_prompt=True, bos_token=bos, eos_token=eos)
            if bos and out.startswith(bos):
                out = out[len(bos):]
            return out if out else None
        except Exception:
            return None

    def _chat_prompt(self, eng: N.Engine, messages: List[Dict[str, Any]]) -> str:
        """messages -> prompt text.  The GGUF's chat template is rendered as Jinja (`_render_jinja`); where that is not possible
        its FAMILY is recognised from the markers it contains -- what llama.cpp's template detection does [external] -- and the
        family's framing applied: Llama-3 headers (also the default without a template), ChatML, Llama-2 / Mistral [INST].
        The gateway's own /api/chat flattening ("role: content\n...assistant:", ollama.ts:367-370) reaches generate*, not this method."""
        try:
            tmpl = eng.chat_template or ""
        except Exception:
            tmpl = ""
        if tmpl and self._jinja:
            rendered = self._render_jinja(eng, tmpl, messages)
            if rendered is not None:
                return rendered
        msgs = [(m.get("role", "user"), m.get("content", "")) for m in messages]
        if "<|im_start|>" in tmpl:                       # ChatML
            return "".join(f"<|im_start|>{r}\n{c}<|im_end|>\n" for r, c in msgs) + "<|im_start|>assistant\n"
        if "[INST]" in tmpl:                             # Llama-2 / Mistral
            system = "\n\n".join(c for r, c in msgs if r == "system")
            out, first = "", True
            for r, c in msgs:
                if r == "system":
                    continue
                if r == "assistant":
                    out += f" {c}</s>"
                    continue
                if first and system:
                    c = f"<<SYS>>\n{system}\n<</SYS>>\n\n{c}" if "<<SYS>>" in tmpl else f"{system}\n\n{c}"
                first = False
                out += f"[INST] {c} [/INST]"
            return out
        parts = [f"<|start_header_id|>{r}<|end_header_id|>\n\n{c}<|eot_id|>" for r, c in msgs]      # Llama-3 (and default)
        parts.append("<|start_header_id|>assistant<|end_header_id|>\n\n")
        return "".join(parts)

    def _stop_ids(self, eng: N.Engine, request: InferenceRequest) -> List[int]:
        return []

    def _plan(self, eng: N.Engine, ids: np.ndarray, num_predict: int, options: Dict[str, Any], on_token, fmt=None):
        """-> (num_predict, ignore_eos, sampling kw, token callback, finish(gen)): what one generation needs, however it is run.
        fmt: the request's _format keywords ({} / None: free text)."""
        kw = dict(self._sampling(options), **self._penalties(options), **(fmt or {}))
        ignore_eos = bool(options.get("ignore_eos", False))
        if fmt and ignore_eos:
            raise RuntimeError("format json cannot be combined with ignore_eos: a JSON document ends on a stop token")
        if fmt and isinstance(fmt.get("format"), dict):
            # a schema outside the subset fails the request before it runs; the engine keeps the compiled schema, and the
            # generation (or the batch runner's open) finds it again by its text
            try:
                with self._lock:
                    eng.format_schema(fmt["format"])
            except N.NativeError as ex:
                raise RuntimeError(ex.detail) from None
        # a generation that would run past the engine's context ends at it (done_reason "length") instead of failing; a prompt
        # that does not fit at all still fails (GL_ERR_CONTEXT)
        n_ctx = int(getattr(eng.info, "n_ctx", 0) or 0)
        if getattr(self, "_context_shift", False):
            # the cache shifts instead: only the output buffers (n_ctx ids) bound a generation
            if n_ctx > 0:
                num_predict = n_ctx if num_predict <= 0 else min(num_predict, n_ctx)
            elif num_predict <= 0:
                num_predict = 128
            kw["num_keep"] = self._num_keep(options)
        else:
            if num_predict <= 0:                             # -1 / -2: until EOS, bounded by the context
                num_predict = max(1, n_ctx - len(ids)) if n_ctx > 0 else 128
            if n_ctx > 0 and len(ids) < n_ctx:
                num_predict = min(num_predict, n_ctx - len(ids))
        stops = options.get("stop")
        stops = [stops] if isinstance(stops, str) else list(stops or [])
        if not stops or not eng.info.has_tokenizer:
            def finish(gen):
                gen.prompt_ids = ids
                return gen
            return num_predict, ignore_eos, kw, on_token, finish
        # stop strings: the token callback sees only released text, and cancels the native call when one completes
        filt = StopFilter(stops)

        def cb(tid: int, lp: float, piece: bytes) -> bool:
            out = filt.feed(piece)
            stop_user = bool(on_token(tid, lp, out.encode("utf-8"))) if on_token is not None else False
            return stop_user or filt.hit

        def finish(gen):
            tail = filt.flush()
            if tail and on_token is not None:
                on_token(-1, 0.0, tail.encode("utf-8"))      # held-back text of a generation that ended by length / EOS
            gen.stop_text = filt.text
            gen.stopped = filt.hit
            gen.prompt_ids = ids
            return gen
        return num_predict, ignore_eos, kw, cb, finish

    def _run(self, model: str, ids: np.ndarray, num_predict: int, options: Dict[str, Any], on_token=None, fmt=None):
        """one request at a time: the blocking gl_generate call (runs on a worker thread)"""
        eng = self._engine(model)
        num_predict, ignore_eos, kw, cb, finish = self._plan(eng, ids, num_predict, options, on_token, fmt)
        with self._lock:
            gen = eng.generate(ids, num_predict=num_predict, ignore_eos=ignore_eos, on_token=cb, **kw)
        return eng, finish(gen)

    async def _generate(self, model: str, ids: np.ndarray, num_predict: int, options: Dict[str, Any], on_token=None, fmt=None):
        """-> (engine, Generation).  With continuous batching the request becomes a sequence of the engine's batch runner and
        this coroutine just awaits its future (no thread is parked per request: 256 concurrent jobs are 256 futures); otherwise
        the blocking call runs on a worker thread.  Either way the event loop stays free for heartbeats."""
        if not self._max_batch:
            return await asyncio.to_thread(self._run, model, ids, num_predict, options, on_token, fmt)
        eng = await self._engine_async(model)
        num_predict, ignore_eos, kw, cb, finish = self._plan(eng, ids, num_predict, options, on_token, fmt)
        runner = await asyncio.to_thread(self._runner, model)
        gen = await asyncio.wrap_future(runner.submit(ids, num_predict, ignore_eos, kw, cb))
        return eng, finish(gen)

    def _sampling(self, options: Dict[str, Any]) -> Dict[str, Any]:
        """InferenceRequest.options.{temperature, top_k, top_p, seed} (client/src/types/index.ts:1-27; gateway ranges
        server/src/routes/ollama.ts:26-48) -> gl_sample_opts.  temperature 0 (or absent, with the default configuration) is
        greedy; a sampled request without a seed draws one, as Ollama does for seed 0 / absent."""
        def opt(name):
            v = options.get(name)
            return self._sampling_defaults.get(name) if v is None else v
        temperature = float(opt("temperature") or 0.0)
        if not (temperature >= 0.0) or temperature == float("inf"):
            raise RuntimeError("temperature must be a finite number >= 0")
        if temperature == 0.0:
            return {}
        top_k = int(opt("top_k") or 0)
        top_p = float(opt("top_p") if opt("top_p") is not None else 1.0)
        seed = opt("seed")
        if seed is None:
            seed = secrets.randbits(63)
        return {"temperature": temperature, "top_k": top_k, "top_p": top_p, "seed": int(seed)}

    def _penalties(self, options: Dict[str, Any]) -> Dict[str, Any]:
        """InferenceRequest.options.{repeat_penalty, repeat_last_n, presence_penalty, frequency_penalty, min_p} (validated by the
        gateway, server/src/routes/ollama.ts:26-39; the OpenAI routes map frequency_penalty / presence_penalty onto the same
        keys, openai.ts:406-410) -> the engine's penalty keywords.  {} when the request sets none of them.  A request that sets a
        penalty but no window gets Ollama's window of 64.  Out-of-range values fail the request, as a bad temperature does."""
        defaults = getattr(self, "_penalty_defaults", {})

        def opt(name):
            v = options.get(name)
            return defaults.get(name) if v is None else v
        given = {k: opt(k) for k in self.PENALTY_OPTIONS if opt(k) is not None}
        if not given:
            return {}
        out: Dict[str, Any] = {}
        for k, v in given.items():
            if isinstance(v, bool):
                raise RuntimeError(f"{k} must be a number")
            try:
                f = float(v)
            except (TypeError, ValueError):
                raise RuntimeError(f"{k} must be a number")
            if not np.isfinite(f):
                raise RuntimeError(f"{k} must be a finite number")
            if k == "repeat_last_n":
                if f != int(f) or f < -1:
                    raise RuntimeError("repeat_last_n must be an integer >= -1")
                out[k] = int(f)
            else:
                out[k] = f
        if out.get("repeat_penalty", 0.0) < 0:
            raise RuntimeError("repeat_penalty must be >= 0")
        if not 0.0 <= out.get("min_p", 0.0) <= 1.0:
            raise RuntimeError("min_p must lie in [0, 1]")
        if "repeat_last_n" not in out and any(k in out for k in ("repeat_penalty", "presence_penalty", "frequency_penalty")):
            out["repeat_last_n"] = 64
        return out

    def _format(self, request: InferenceRequest) -> Dict[str, Any]:
        """The request's output format -> the engine's `format` keyword.  metadata.format first (the gateway's Ollama routes,
        server/src/routes/ollama.ts:229, 385), then options.format (its OpenAI route, openai.ts:636-642).  "json" turns the
        JSON grammar mask on.  A JSON-schema object is enforced with json_schema=True (the engine compiles it; see
        gl_format_schema); otherwise it too turns on the JSON mask alone (valid JSON of any shape).  Absent, None or "" is free
        text ({}); anything else fails the request, as a bad temperature does."""
        md = request.get("metadata") or {}
        fmt = md.get("format")
        if fmt is None or fmt == "":
            fmt = (request.get("options") or {}).get("format")
        if fmt is None or fmt == "":
            return {}
        if isinstance(fmt, dict) and self._json_schema:
            return {"format": fmt}
        if fmt == "json" or isinstance(fmt, dict):
            return {"format": "json"}
        raise RuntimeError(f'format must be "json" or a JSON schema object, not {fmt!r}')

    def _response(self, request: InferenceRequest, eng: N.Engine, gen: N.Generation, text: str) -> InferenceResponse:
        st = gen.stats
        if getattr(gen, "stop_text", None) is not None:      # options.stop was active: the filtered text is the response
            text = gen.stop_text
        return {
            "id": request["id"],
            "model": request["model"],
            "created_at": _now_iso(),
            "response": text,
            "done": True,
            "done_reason": "stop" if (st.done_reason == 0 or getattr(gen, "stopped", False)) else "length",
            "total_duration": int(st.total_duration_ns),           # real numbers (the reference reports 0, :156-161)
            "load_duration": int(st.load_duration_ns),
            "prompt_eval_count": int(st.prompt_eval_count),
            "prompt_eval_duration": int(st.prompt_eval_duration_ns),
            "eval_count": int(st.eval_count),
            "eval_duration": int(st.eval_duration_ns),
            "system_fingerprint": "fp_gridllm_b200_native",
            # Ollama's `context` is the WHOLE conversation so far -- prompt ids then reply ids -- and the gateway round-trips it
            # (ollama.ts:143 returns it, :234 forwards it as metadata.context): a client that feeds it back continues from here
            "context": [int(t) for t in getattr(gen, "prompt_ids", [])] + [int(t) for t in gen.ids],
            "token_ids": [int(t) for t in gen.ids],                 # generated ids alone: SURVEY.md section 8f.4 (optional field)
            "logprobs": [float(x) for x in gen.logprobs],
        }

    def _text(self, eng: N.Engine, ids) -> str:
        return eng.detokenize(ids) if eng.info.has_tokenizer else ""

    # ---- OllamaService.generateResponse (:97-184) -------------------------------------------------
    async def generateResponse(self, request: InferenceRequest) -> InferenceResponse:
        try:
            options = request.get("options") or {}
            num_predict = self._num_predict(options)
            fmt = self._format(request)
            eng = await self._engine_async(request["model"])
            ids = self._prompt_ids(eng, request, request.get("prompt"))
            eng, gen = await self._generate(request["model"], ids, num_predict, options, fmt=fmt)
            return self._response(request, eng, gen, self._text(eng, gen.ids))
        except Exception as error:
            raise RuntimeError(f"Inference failed: {error}")

    # ---- OllamaService.generateStreamResponse (:186-284): async generator of {id, response, done} ----
    async def generateStreamResponse(self, request: InferenceRequest) -> AsyncGenerator[StreamResponse, None]:
        try:
            options = request.get("options") or {}
            num_predict = self._num_predict(options)
            fmt = self._format(request)
            eng = await self._engine_async(request["model"])
            ids = self._prompt_ids(eng, request, request.get("prompt"))
            loop = asyncio.get_running_loop()
            q: "asyncio.Queue" = asyncio.Queue()
            cancel = threading.Event()

            def on_token(tid: int, lp: float, piece: bytes) -> bool:      # called on an engine thread
                loop.call_soon_threadsafe(q.put_nowait, ("tok", tid, piece))
                return cancel.is_set()          # non-zero return cancels (job_cancellation, JobScheduler.ts:530-536)

            async def work():
                try:
                    _, gen = await self._generate(request["model"], ids, num_predict, options, on_token, fmt=fmt)
                    q.put_nowait(("done", gen, None))     # after every token this generation queued (same loop, FIFO)
                except Exception as ex:          # surfaced on the consumer side
                    q.put_nowait(("err", ex, None))

            task = asyncio.ensure_future(work())
            pending = b""
            try:
                while True:
                    kind, a, b = await q.get()
                    if kind == "tok":
                        pending += b or b""
                        try:
                            text = pending.decode("utf-8")
                            pending = b""
                        except UnicodeDecodeError:
                            text = ""            # wait for the rest of a multi-byte character
                        yield {"id": request["id"], "response": text, "done": False}
                    elif kind == "done":
                        yield {"id": request["id"], "response": pending.decode("utf-8", "replace"), "done": True}
                        return
                    else:
                        raise a
            finally:
                cancel.set()
                if not task.done():              # the consumer left early: the cancel flag ends the generation at its next token
                    try:
                        await task
                    except Exception:
                        pass
        except Exception as error:
            raise RuntimeError(f"Streaming inference failed: {error}")

    # ---- OllamaService.generateChatResponse (:353-449) -------------------------------------------------
    async def generateChatResponse(self, request: InferenceRequest) -> InferenceResponse:
        try:
            md = request.get("metadata") or {}
            if not md.get("messages"):
                raise RuntimeError("Chat request must include messages in metadata")
            options = request.get("options") or {}
            num_predict = self._num_predict(options)
            fmt = self._format(request)
            eng = await self._engine_async(request["model"])
            prompt = self._chat_prompt(eng, md["messages"])
            if md.get("prompt_token_ids") is not None:
                ids = np.asarray(md["prompt_token_ids"], dtype=np.int32)
            else:
                if not eng.info.has_tokenizer:
                    raise RuntimeError("model carries no tokenizer; supply metadata.prompt_token_ids")
                ids = eng.tokenize(prompt, add_bos=True, parse_special=True)
            eng, gen = await self._generate(request["model"], ids, num_predict, options, fmt=fmt)
            res = self._response(request, eng, gen, self._text(eng, gen.ids))
            res["message"] = {"role": "assistant", "content": res.pop("response")}
            return res
        except Exception as error:
            raise RuntimeError(f"Chat inference failed: {error}")

    # ---- OllamaService.generateChatStreamResponse (:451-599) ---------------------------------------------
    async def generateChatStreamResponse(self, request: InferenceRequest) -> AsyncGenerator[StreamResponse, None]:
        try:
            md = request.get("metadata") or {}
            if not md.get("messages"):
                raise RuntimeError("Chat request must include messages in metadata")
            eng = await self._engine_async(request["model"])
            sub = dict(request)
            if md.get("prompt_token_ids") is None:
                if not eng.info.has_tokenizer:
                    raise RuntimeError("model carries no tokenizer; supply metadata.prompt_token_ids")
                ids = eng.tokenize(self._chat_prompt(eng, md["messages"]), add_bos=True, parse_special=True)
                sub["metadata"] = dict(md, prompt_token_ids=[int(t) for t in ids])
            async for chunk in self.generateStreamResponse(sub):
                yield chunk
        except Exception as error:
            raise RuntimeError(f"Chat streaming inference failed: {error}")

    # ---- OllamaService.generateEmbedding (:601-665) ------------------------------------------------------
    async def generateEmbedding(self, request: InferenceRequest) -> InferenceResponse:
        try:
            inp = request.get("input")
            md = request.get("metadata") or {}
            if not inp and md.get("input_token_ids") is None:
                raise RuntimeError("Input is required for embedding requests")
            eng = await self._engine_async(request["model"])
            if md.get("input_token_ids") is not None:
                seqs = [np.asarray(s, dtype=np.int32) for s in md["input_token_ids"]]
            else:
                if not eng.info.has_tokenizer:
                    raise RuntimeError("model carries no tokenizer; supply metadata.input_token_ids")
                texts = inp if isinstance(inp, list) else [inp]
                seqs = [eng.tokenize(t, add_bos=True, parse_special=False) for t in texts]
            # metadata.truncate (OllamaService.ts:626-628): inputs longer than the context are cut to it unless truncate is false,
            # in which case the engine's context error surfaces (what /api/embed does [external])
            n_ctx = int(getattr(eng.info, "n_ctx", 0) or 0)
            if n_ctx > 0 and md.get("truncate", True) is not False:
                seqs = [s[:n_ctx] for s in seqs]

            def work():
                with self._lock:
                    return eng.embed(seqs)

            t0 = time.perf_counter_ns()
            emb, st = await asyncio.to_thread(work)
            return {"id": request["id"], "model": request["model"], "embeddings": emb.astype(float).tolist(),
                    "total_duration": time.perf_counter_ns() - t0, "load_duration": int(st.load_duration_ns),
                    "prompt_eval_count": int(st.prompt_eval_count)}
        except Exception as error:
            raise RuntimeError(f"Embedding failed: {error}")

    # ---- pullModel / deleteModel (:286-331): not reachable from WorkerClientService -------------------------
    async def pullModel(self, modelName: str) -> None:
        raise RuntimeError(f"Failed to pull model {modelName}: the native worker loads local GGUF files only")

    async def deleteModel(self, modelName: str) -> None:
        raise RuntimeError(f"Failed to delete model {modelName}: the native worker does not manage model files")
