// Drop-in replacement for client/src/services/OllamaService.ts: same 8-method surface, same
// InferenceRequest / InferenceResponse / StreamResponse types (client/src/types/index.ts), but every call goes
// to the in-process native engine (host/napi/addon.cc -> libgridllm_native.so) instead of HTTP to Ollama.
// WorkerClientService.ts needs one line changed: `new OllamaService()` -> `new NativeInferenceService()`
// (WorkerClientService.ts:32).  Not executable in the build image (no node); the Python twin
// gridllm_b200/service.py is what the tests run.
import { config } from "@/config";
import { logger } from "@/utils/logger";
import { OllamaModel, InferenceRequest, InferenceResponse, StreamResponse } from "@/types";
import * as fs from "fs";

// eslint-disable-next-line @typescript-eslint/no-var-requires
const native = require("../napi/build/Release/gridllm_native.node");

interface NativeStats {
	promptEvalCount: number; evalCount: number; promptEvalDurationNs: number; evalDurationNs: number;
	totalDurationNs: number; loadDurationNs: number; doneReason: number;
}

export class NativeInferenceService {
	private engines = new Map<string, unknown>();
	private isConnected = false;
	private lastHealthCheck = new Date();
	// model name -> GGUF path, e.g. GRIDLLM_MODELS="llama3:8b=/models/llama3-8b-q4_K_M.gguf"
	private models: Record<string, string> = Object.fromEntries(
		(process.env.GRIDLLM_MODELS || "").split(",").filter(Boolean).map((kv) => kv.split("=") as [string, string])
	);
	private device = parseInt(process.env.GRIDLLM_DEVICE || "0", 10);
	// prefixCache: a generate keeps the KV pages of the longest prefix it shares with the previous generate on the same engine
	// (a client that sends `context` back pays for its new tokens only); off by default (include/gridllm_native.h)
	private engineOptions: { prefixCache?: boolean };
	// jsonSchema: enforce a JSON-schema `format` on the GPU (gl_format_schema); off by default: a schema asks for valid JSON of
	// any shape, as before.  Same switch as gridllm_b200/service.py's json_schema.
	private jsonSchema: boolean;

	constructor(options: { prefixCache?: boolean; jsonSchema?: boolean } = {}) {
		this.engineOptions = { prefixCache: !!options.prefixCache };
		this.jsonSchema = !!options.jsonSchema;
	}

	private engine(name: string): unknown {
		if (!this.models[name]) throw new Error(`model '${name}' not found`);
		if (!this.engines.has(name)) this.engines.set(name, native.createEngine(this.models[name], this.device, this.engineOptions));
		return this.engines.get(name);
	}

	async checkHealth(): Promise<boolean> {                       // OllamaService.ts:65-83
		this.isConnected = native.deviceCount() > this.device;
		this.lastHealthCheck = new Date();
		return this.isConnected;
	}

	async getAvailableModels(): Promise<OllamaModel[]> {           // :85-95
		return Object.entries(this.models).map(([name, path]) => {
			const st = fs.statSync(path);
			return { name, digest: `${st.size}-${st.mtimeMs}`, size: st.size, modified_at: st.mtime.toISOString(),
				details: { format: "gguf", family: "llama", families: ["llama"], parameter_size: "", quantization_level: "" } };
		});
	}

	async validateModel(modelName: string): Promise<boolean> {     // :340-351, O(1) instead of GET /api/tags per job
		return !!this.models[modelName];
	}

	// GRIDLLM_SAMPLING=ollama: requests that leave temperature / top_k / top_p out inherit Ollama's documented defaults
	// (0.8 / 40 / 0.9); default: greedy, the BASELINE configuration.  GRIDLLM_APPLY_TEMPLATE=1: frame generate prompts as one user
	// turn of the model's chat template unless metadata.raw (what Ollama does).  Same switches as gridllm_b200/service.py.
	private samplingDefaults: Record<string, number> = process.env.GRIDLLM_SAMPLING === "ollama" ? { temperature: 0.8, top_k: 40, top_p: 0.9 } : {};
	private applyTemplate = process.env.GRIDLLM_APPLY_TEMPLATE === "1";

	// Optional Jinja renderer for tokenizer.chat_template: (template, variables) -> text, e.g. `(t, v) => new Template(t).render(v)`
	// from @huggingface/jinja.  gridllm_b200/service.py renders the template with sandboxed jinja2 (messages, add_generation_prompt,
	// bos_token / eos_token, raise_exception) and falls back to the family framing below when that fails; this twin does the same
	// when a renderer is injected, and uses the family framing alone otherwise (no Jinja engine is vendored here).
	public renderTemplate?: (template: string, vars: Record<string, unknown>) => string;
	public bosText = "";      // texts of the BOS / EOS control tokens for the template: native.tokenText(engine, info.bosId / eosId)
	public eosText = "";      // (filled when the engine is created)

	// messages -> prompt text.  With a renderer: the GGUF's chat template interpreted as the Jinja program it is.  Otherwise (or
	// when rendering throws) its FAMILY is recognised from the markers it contains (gl_chat_template) -- Llama-3 headers (also the
	// default), ChatML, Llama-2 / Mistral [INST] -- and that family's framing applied; same order as gridllm_b200/service.py::_chat_prompt.
	private chatPrompt(e: unknown, messages: Array<{ role: string; content: string }>): string {
		let tmpl = "";
		try { tmpl = native.chatTemplate(e) || ""; } catch { tmpl = ""; }
		if (tmpl && this.renderTemplate) {
			try {
				let out = this.renderTemplate(tmpl, { messages, add_generation_prompt: true, bos_token: this.bosText, eos_token: this.eosText,
					raise_exception: (m: string) => { throw new Error(m); } });
				if (this.bosText && out.startsWith(this.bosText)) out = out.slice(this.bosText.length);      // the tokenizer adds the BOS id itself
				if (out) return out;
			} catch { /* a template this conversation does not fit: the family framing */ }
		}
		const msgs = messages.map((m) => [m.role ?? "user", m.content ?? ""] as [string, string]);
		if (tmpl.includes("<|im_start|>"))
			return msgs.map(([r, c]) => `<|im_start|>${r}\n${c}<|im_end|>\n`).join("") + "<|im_start|>assistant\n";
		if (tmpl.includes("[INST]")) {
			const system = msgs.filter(([r]) => r === "system").map(([, c]) => c).join("\n\n");
			let out = "", first = true;
			for (const [r, c0] of msgs) {
				if (r === "system") continue;
				if (r === "assistant") { out += ` ${c0}</s>`; continue; }
				let c = c0;
				if (first && system) c = tmpl.includes("<<SYS>>") ? `<<SYS>>\n${system}\n<</SYS>>\n\n${c}` : `${system}\n\n${c}`;
				first = false;
				out += `[INST] ${c} [/INST]`;
			}
			return out;
		}
		return msgs.map(([r, c]) => `<|start_header_id|>${r}<|end_header_id|>\n\n${c}<|eot_id|>`).join("")
			+ "<|start_header_id|>assistant<|end_header_id|>\n\n";
	}

	private ids(e: unknown, request: InferenceRequest): Int32Array {
		const md = request.metadata ?? {};
		if (md.prompt_token_ids) return Int32Array.from(md.prompt_token_ids);
		const ctx: number[] | undefined = md.context;                          // conversation so far (OllamaService.ts:224-226)
		if (this.applyTemplate && !md.raw && !ctx?.length) {
			const msgs = [...(md.system ? [{ role: "system", content: md.system }] : []), { role: "user", content: request.prompt || "" }];
			return native.tokenize(e, this.chatPrompt(e, msgs), true, true);
		}
		if (ctx?.length) return Int32Array.from([...ctx, ...native.tokenize(e, request.prompt || "", false, false)]);
		return native.tokenize(e, request.prompt || "", true, false);
	}

	// options.stop: same rule as gridllm_b200/service.py::StopFilter -- end at the first stop string in the generated text,
	// hold back text that could still become one.  feed() returns the text a token releases; hit ends the native call.
	private stopFilter(stops: string[]) {
		const st = { text: "", held: "", hit: false,
			feed(piece: string): string {
				if (st.hit) return "";
				const buf = st.held + piece;
				const cuts = stops.map((s) => buf.indexOf(s)).filter((i) => i >= 0);
				if (cuts.length) { st.hit = true; st.held = ""; const out = buf.slice(0, Math.min(...cuts)); st.text += out; return out; }
				let keep = 0;
				for (const s of stops) for (let n = Math.min(s.length - 1, buf.length); n > 0; --n) if (buf.endsWith(s.slice(0, n))) { keep = Math.max(keep, n); break; }
				const out = buf.slice(0, buf.length - keep); st.held = buf.slice(buf.length - keep); st.text += out; return out;
			},
			flush(): string { const out = st.hit ? "" : st.held; st.held = ""; st.text += out; return out; } };
		return st;
	}

	// `context` is the WHOLE conversation so far -- prompt ids then reply ids: the gateway returns it (ollama.ts:143) and forwards
	// it back as metadata.context (ollama.ts:234), and a client that feeds it back must continue from here
	private toResponse(request: InferenceRequest, text: string, ids: Int32Array, st: NativeStats, promptIds?: Int32Array): InferenceResponse {
		return { id: request.id, model: request.model, created_at: new Date().toISOString(), response: text, done: true,
			done_reason: st.doneReason === 0 ? "stop" : "length", total_duration: st.totalDurationNs, load_duration: st.loadDurationNs,
			prompt_eval_count: st.promptEvalCount, prompt_eval_duration: st.promptEvalDurationNs, eval_count: st.evalCount,
			eval_duration: st.evalDurationNs, context: [...Array.from(promptIds ?? []), ...Array.from(ids)], token_ids: Array.from(ids),
			system_fingerprint: "fp_gridllm_b200_native" };
	}

	// InferenceRequest.options -> gl_sample_opts; temperature absent / 0 = greedy, a sampled request without seed draws one
	// num_predict: `options.num_predict || 128` (OllamaService.ts:105); the gateway also lets -1 / -2 through (ollama.ts:47,
	// "until EOS"): those run until the engine's context is full, like service.py::_plan
	private sampleOpts(request: InferenceRequest, e?: unknown, nPrompt = 0) {
		const o = request.options ?? {};
		const d = this.samplingDefaults;
		const temperature = o.temperature ?? d.temperature ?? 0;
		if (!(temperature >= 0) || !Number.isFinite(temperature)) throw new Error("temperature must be a finite number >= 0");
		let numPredict = o.num_predict || 128;
		const nCtx = e ? (native.engineInfo(e).nCtx as number) : 0;
		if (numPredict < 0) numPredict = nCtx > 0 ? Math.max(1, nCtx - nPrompt) : 128;
		if (nCtx > 0 && nPrompt < nCtx) numPredict = Math.min(numPredict, nCtx - nPrompt);
		return { numPredict, ignoreEos: !!o.ignore_eos, temperature, topK: o.top_k ?? d.top_k ?? 0, topP: o.top_p ?? d.top_p ?? 1,
			seed: BigInt(o.seed ?? (temperature > 0 ? Math.floor(Math.random() * 2 ** 53) : 0)), ...this.penaltyOpts(o),
			...this.formatOpts(request, e) };
	}

	// The output format -> the addon's format field; same mapping as gridllm_b200/service.py::_format.  metadata.format first (the
	// gateway's Ollama routes), then options.format (its OpenAI route).  "json" turns the JSON grammar mask on.  A JSON-schema
	// object is compiled and enforced with jsonSchema (a schema outside the subset fails the request with the library's message);
	// otherwise it too turns on the JSON mask alone (valid JSON of any shape).  Absent, null or "": free text.
	private formatOpts(request: InferenceRequest, e?: unknown): { format?: string | number } {
		let f: any = request.metadata?.format;
		if (f === undefined || f === null || f === "") f = (request.options as Record<string, any> | undefined)?.format;
		if (f === undefined || f === null || f === "") return {};
		if (f !== "json" && (typeof f !== "object" || Array.isArray(f))) throw new Error(`format must be "json" or a JSON schema object`);
		if (request.options?.ignore_eos) throw new Error("format json cannot be combined with ignore_eos: a JSON document ends on a stop token");
		if (this.jsonSchema && typeof f === "object" && e) {
			try {
				return { format: native.formatSchema(e, JSON.stringify(f)) as number };
			} catch (err: any) {
				throw new Error(String(err?.message ?? err).replace(/^gl_format_schema: (GL_ERR_[A-Z]+: )?/, ""));
			}
		}
		return { format: "json" };
	}

	// GRIDLLM_PENALTIES=ollama: requests that leave the repetition penalty out inherit Ollama's defaults (repeat_penalty 1.1 over
	// the last 64 ids); default: no penalty.  Same mapping as gridllm_b200/service.py::_penalties.
	private penaltyDefaults: Record<string, number> = process.env.GRIDLLM_PENALTIES === "ollama" ? { repeat_penalty: 1.1, repeat_last_n: 64 } : {};

	// options.{repeat_penalty, repeat_last_n, presence_penalty, frequency_penalty, min_p} (gateway: ollama.ts:26-39; the OpenAI
	// routes use the same keys) -> the addon's penalty fields.  Absent: none of them (the engine's zeros mean "off").  A penalty
	// without a window gets Ollama's window of 64.
	private penaltyOpts(o: Record<string, any>) {
		const d = this.penaltyDefaults;
		const pick = (k: string): number | undefined => (o[k] ?? d[k]);
		const out: Record<string, number> = {};
		for (const [k, name] of [["repeat_penalty", "repeatPenalty"], ["repeat_last_n", "repeatLastN"], ["presence_penalty", "presencePenalty"],
			["frequency_penalty", "frequencyPenalty"], ["min_p", "minP"]] as const) {
			const v = pick(k);
			if (v === undefined || v === null) continue;
			if (typeof v !== "number" || !Number.isFinite(v)) throw new Error(`${k} must be a finite number`);
			out[name] = v;
		}
		if (out.repeatPenalty !== undefined && out.repeatPenalty < 0) throw new Error("repeat_penalty must be >= 0");
		if (out.repeatLastN !== undefined && (!Number.isInteger(out.repeatLastN) || out.repeatLastN < -1)) throw new Error("repeat_last_n must be an integer >= -1");
		if (out.minP !== undefined && !(out.minP >= 0 && out.minP <= 1)) throw new Error("min_p must lie in [0, 1]");
		if (out.repeatLastN === undefined && (out.repeatPenalty !== undefined || out.presencePenalty !== undefined || out.frequencyPenalty !== undefined))
			out.repeatLastN = 64;
		return out;
	}

	async generateResponse(request: InferenceRequest): Promise<InferenceResponse> {   // :97-184
		try {
			const e = this.engine(request.model);
			const stop = request.options?.stop;
			const stops: string[] = (typeof stop === "string" ? [stop] : stop || []).filter(Boolean);
			const promptIds = this.ids(e, request);
			if (!stops.length) {
				const out = await native.generate(e, promptIds, this.sampleOpts(request, e, promptIds.length), null);
				return this.toResponse(request, native.detokenize(e, out.ids), out.ids, out.stats, promptIds);
			}
			const f = this.stopFilter(stops);         // a non-zero return of the token callback cancels gl_generate
			const out = await native.generate(e, promptIds, this.sampleOpts(request, e, promptIds.length),
				(_id: number, _lp: number, piece: string) => { f.feed(piece); return f.hit; });
			f.flush();
			const res = this.toResponse(request, f.text, out.ids, out.stats, promptIds);
			if (f.hit) res.done_reason = "stop";
			return res;
		} catch (error) {
			throw new Error(`Inference failed: ${error instanceof Error ? error.message : "Unknown error"}`);
		}
	}

	async *generateStreamResponse(request: InferenceRequest): AsyncGenerator<StreamResponse> {   // :186-284
		try {
			const e = this.engine(request.model);
			const queue: StreamResponse[] = [];
			let wake: (() => void) | null = null;
			const promptIds = this.ids(e, request);
			const done = native.generate(e, promptIds, this.sampleOpts(request, e, promptIds.length),
				(_id: number, _lp: number, piece: string) => { queue.push({ id: request.id, response: piece, done: false }); wake?.(); });
			let finished = false;
			done.then(() => { finished = true; wake?.(); }, () => { finished = true; wake?.(); });
			while (!finished || queue.length) {
				if (queue.length) { yield queue.shift()!; continue; }
				await new Promise<void>((r) => (wake = r));
			}
			await done;
			yield { id: request.id, response: "", done: true };
		} catch (error) {
			throw new Error(`Streaming inference failed: ${error instanceof Error ? error.message : "Unknown error"}`);
		}
	}

	async generateChatResponse(request: InferenceRequest): Promise<InferenceResponse> {   // :353-449
		if (!request.metadata?.messages) throw new Error("Chat inference failed: Chat request must include messages in metadata");
		const e = this.engine(request.model);
		const ids = request.metadata.prompt_token_ids ?? Array.from(native.tokenize(e, this.chatPrompt(e, request.metadata.messages), true, true) as Int32Array);
		const r = await this.generateResponse({ ...request, metadata: { ...request.metadata, prompt_token_ids: ids } });
		const { response, ...rest } = r;
		return { ...rest, message: { role: "assistant", content: response } };
	}

	async *generateChatStreamResponse(request: InferenceRequest): AsyncGenerator<StreamResponse> {   // :451-599
		if (!request.metadata?.messages) throw new Error("Chat streaming inference failed: Chat request must include messages in metadata");
		const e = this.engine(request.model);
		const ids = request.metadata.prompt_token_ids ?? Array.from(native.tokenize(e, this.chatPrompt(e, request.metadata.messages), true, true) as Int32Array);
		yield* this.generateStreamResponse({ ...request, metadata: { ...request.metadata, prompt_token_ids: ids } });
	}

	async generateEmbedding(request: InferenceRequest): Promise<InferenceResponse> {   // :601-665
		try {
			if (!request.input) throw new Error("Input is required for embedding requests");
			const e = this.engine(request.model);
			const texts = Array.isArray(request.input) ? request.input : [request.input];
			// metadata.truncate (OllamaService.ts:626-628): inputs longer than the context are cut to it unless truncate is false
			const nCtx = native.engineInfo(e).nCtx as number;
			const cut = request.metadata?.truncate !== false && nCtx > 0;
			const seqs = texts.map((t) => { const a = native.tokenize(e, t, true, false) as Int32Array; return cut ? a.subarray(0, nCtx) : a; });
			const offsets = new Int32Array(seqs.length + 1);
			seqs.forEach((s, i) => (offsets[i + 1] = offsets[i] + s.length));
			const flat = new Int32Array(offsets[seqs.length]);
			seqs.forEach((s, i) => flat.set(s, offsets[i]));
			const out = await native.embed(e, flat, offsets);
			const dim = out.embeddings.length / seqs.length;
			return { id: request.id, model: request.model,
				embeddings: seqs.map((_, i) => Array.from(out.embeddings.subarray(i * dim, (i + 1) * dim))),
				total_duration: out.stats.totalDurationNs, load_duration: out.stats.loadDurationNs, prompt_eval_count: out.stats.promptEvalCount };
		} catch (error) {
			throw new Error(`Embedding failed: ${error instanceof Error ? error.message : "Unknown error"}`);
		}
	}

	getConnectionStatus() { return { isConnected: this.isConnected, lastHealthCheck: this.lastHealthCheck }; }
	async pullModel(modelName: string): Promise<void> { throw new Error(`Failed to pull model ${modelName}: local GGUF files only`); }
	async deleteModel(modelName: string): Promise<void> { throw new Error(`Failed to delete model ${modelName}: not managed`); }
}

export default NativeInferenceService;
void config; void logger;
