"""TEST INFRASTRUCTURE: CPU restatement of the repetition / presence / frequency penalties (gridllm_b200/csrc/penalty.cu) and of
the min-p cut of the seeded samplers (gridllm_b200/csrc/sampler.cu), on top of the draw restated in oracle/sampler.py.

Repetition penalties: Ollama's documented options repeat_penalty, repeat_last_n, presence_penalty, frequency_penalty, forwarded by
the reference (server/src/routes/ollama.ts:26-39, client/src/services/OllamaService.ts:121-125); the arithmetic is llama.cpp's
penalties sampler, which Ollama's runner uses [external: no implementation of it is in this tree].  PARITY UNPINNED against a real
Ollama, like the draw of oracle/sampler.py.
  * history H = the prompt ids of the call (BOS and any prepended context ids included), then every generated token (a drawn stop
    token ends the sequence and is never added);
  * window W = the last N entries of H: N = repeat_last_n if > 0, all of H if -1; 0 = no penalty of any kind;
  * for each distinct id t in W occurring c times: a = logit[t]; if repeat_penalty is active (> 0 and != 1)
    a = a * repeat_penalty if a <= 0 else a / repeat_penalty; logit[t] = a - (c * frequency_penalty + presence_penalty);
  * every operation is one fp32 operation rounded to nearest (no fused multiply-add): numpy float32 reproduces the kernel bit for
    bit.

min-p: after the top-p cut of oracle.sampler.distribution, keep the prefix of candidates whose weight w_j = exp((l_j - l_0) / T)
is >= min_p (off for min_p <= 0).  Both cuts are prefixes of the candidate order; the shorter wins.  The reported logprob is the
log-softmax at T = 1 of the drawn logit over the (penalised) logits, as oracle/sampler.py reports it.
"""
from __future__ import annotations

import numpy as np

from oracle import sampler as SM


def penalize(logits: np.ndarray, history, repeat_penalty: float = 1.0, repeat_last_n: int = 64, presence_penalty: float = 0.0,
             frequency_penalty: float = 0.0) -> np.ndarray:
    """The penalised copy of `logits` (float32) for a sequence whose history (prompt ids, then generated ids) is `history`."""
    out = np.array(logits, dtype=np.float32, copy=True)
    h = np.asarray(history, dtype=np.int64).reshape(-1)
    rp, pp, fp = np.float32(repeat_penalty), np.float32(presence_penalty), np.float32(frequency_penalty)
    rp_on = rp > 0 and rp != 1
    if repeat_last_n == 0 or len(h) == 0 or not (rp_on or pp != 0 or fp != 0):
        return out
    win = h if repeat_last_n < 0 else h[max(0, len(h) - int(repeat_last_n)):]
    ids, counts = np.unique(win, return_counts=True)
    a = out[ids]
    if rp_on:
        a = np.where(a <= 0, a * rp, a / rp).astype(np.float32)
    out[ids] = a - (counts.astype(np.float32) * fp + pp)
    return out


def distribution(logits: np.ndarray, temperature: float, top_k: int, top_p: float, min_p: float = 0.0):
    """oracle.sampler.distribution followed by the min-p cut: (candidate ids kept, cumulative masses) in float64."""
    ids, c = SM.distribution(logits, temperature, top_k, top_p)
    if min_p > 0.0:
        l32 = np.asarray(logits, dtype=np.float32)
        inv_t = np.float32(1.0) / np.float32(temperature)              # the same weights oracle.sampler.distribution sums
        w = np.exp((l32[ids].astype(np.float64) - float(l32[ids[0]])) * float(inv_t))
        keep = min(len(ids), int(np.count_nonzero(w >= float(np.float32(min_p)))))      # w does not increase, w[0] = 1
        ids, c = ids[:keep], c[:keep]
    return ids, c


def sample(logits: np.ndarray, temperature: float, top_k: int = 0, top_p: float = 1.0, seed: int = 0, out_index: int = 0,
           min_p: float = 0.0):
    """oracle.sampler.sample with the min-p cut: (token id, logprob, margin)."""
    l32 = np.asarray(logits, dtype=np.float32)
    if temperature <= 0 or min_p <= 0.0:
        return SM.sample(l32, temperature, top_k, top_p, seed, out_index)
    ids, c = distribution(l32, temperature, top_k, top_p, min_p)
    r = SM.uniform24(seed, out_index) * c[-1]
    j = min(int(np.searchsorted(c, r, side="right")), len(ids) - 1)
    lo = c[j - 1] if j > 0 else 0.0
    m = float(l32.max())
    lse = m + float(np.log(np.sum(np.exp(l32.astype(np.float64) - m))))
    return int(ids[j]), float(l32[ids[j]]) - lse, float(min(r - lo, c[j] - r) / c[-1])


def interval_error(logits: np.ndarray, token: int, temperature: float, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
                   out_index: int = 0, min_p: float = 0.0) -> float:
    """oracle.sampler.interval_error with the min-p cut (0 = the draw lies inside `token`'s interval, inf = not a kept candidate)."""
    ids, c = distribution(np.asarray(logits, dtype=np.float32), temperature, top_k, top_p, min_p)
    where = np.nonzero(ids == token)[0]
    if len(where) == 0:
        return float("inf")
    j = int(where[0])
    r = SM.uniform24(seed, out_index) * c[-1]
    lo = c[j - 1] if j > 0 else 0.0
    return float(max(lo - r, r - c[j], 0.0) / c[-1])
