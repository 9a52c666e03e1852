"""TEST INFRASTRUCTURE -- the context-shift rule (include/gridllm_native.h, gl_engine_opts context_shift) restated in Python,
and applied to the numpy oracle's list cache (oracle/llama_oracle.py LlamaOracle).

A shift at window W with keep count k drops positions [k, k + d), d = ceil((W - k) / 2), moves the rows [k + d, W) down to
[k, W - d), rotates each moved K row by -d positions with the fp32 cos / sin table row d (in float64, then rounded as the cache
rounds: fp16) and leaves V as it is.  Llama.cpp's K-shift, which Ollama's runner uses; parity with a real Ollama is unpinned."""
from typing import Dict, List, Sequence

import numpy as np


def keep_count(num_keep: int, n_prompt: int, W: int) -> int:
    k = n_prompt if num_keep < 0 else num_keep
    return min(k, W - 1)


def discard(W: int, k: int) -> int:
    return (W - k + 1) // 2


def cut_prompt(prompt: Sequence[int], W: int, k: int) -> List[int]:
    """a prompt of W ids or more: its first k ids plus its newest W - d - k ids"""
    p = list(prompt)
    if len(p) < W:
        return p
    tail = W - discard(W, k) - k
    return p[:k] + (p[len(p) - tail:] if tail > 0 else [])


def chunk_steps(chunk: int, remaining: int, pos: int, W: int, head_only_first: bool) -> int:
    """gl_generate's decode chunk with the option on: it ends at the window"""
    return min(chunk, remaining, W - pos + (1 if head_only_first else 0))


def rotate_back(rows: np.ndarray, d: int, cos: np.ndarray, sin: np.ndarray) -> np.ndarray:
    """R(-d) applied to K rows [..., head_dim] (adjacent pairs), float64 arithmetic on the fp32 table row d"""
    r = np.asarray(rows, dtype=np.float64)
    hd = r.shape[-1]
    p = r.reshape(r.shape[:-1] + (hd // 2, 2))
    c = cos[d].astype(np.float64)
    s = sin[d].astype(np.float64)
    out = np.empty_like(p)
    out[..., 0] = p[..., 0] * c + p[..., 1] * s
    out[..., 1] = p[..., 1] * c - p[..., 0] * s
    return out.reshape(r.shape)


def shift(orc, keep: int, d: int) -> None:
    """apply one shift to a LlamaOracle's cache (its lists hold rows 0 .. pos - 1) and lower its position by d"""
    m = orc.m
    for il in range(m.n_layer):
        ks, vs = orc.k[il], orc.v[il]
        moved = [orc._kv_round(rotate_back(np.asarray(r).reshape(m.n_head_kv, m.head_dim), d, orc.cos, orc.sin).reshape(-1))
                 for r in ks[keep + d:]]
        orc.k[il] = ks[:keep] + moved
        orc.v[il] = vs[:keep] + vs[keep + d:]
    orc.pos -= d


def greedy_with_shifts(orc, prompt: Sequence[int], n_predict: int, W: int, keep: int) -> Dict[str, np.ndarray]:
    """LlamaOracle.generate with the context shift: greedy ids, their logprobs, top-1 / top-2 margins, logits per step and
    the number of shifts"""
    orc.reset()
    d = discard(W, keep)
    logits = None
    for t in prompt:
        logits = orc.step(int(t))
    ids, lps, margins, all_logits = [], [], [], []
    n_shifts = 0
    for i in range(n_predict):
        top = int(np.argmax(logits))
        lse = logits.max() + np.log(np.exp(logits - logits.max()).sum())
        srt = np.partition(logits, -2)[-2:]
        ids.append(top)
        lps.append(float(logits[top] - lse))
        margins.append(float(srt[1] - srt[0]))
        all_logits.append(logits.astype(np.float32))
        if i == n_predict - 1:
            break
        if orc.pos == W:
            shift(orc, keep, d)
            n_shifts += 1
        logits = orc.step(top)
    return {"ids": np.array(ids, dtype=np.int32), "logprobs": np.array(lps, dtype=np.float32),
            "margins": np.array(margins, dtype=np.float32), "logits": np.stack(all_logits), "shifts": n_shifts}
