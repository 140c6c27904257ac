"""CPU restatement of the per-token scoring contract (include/fo1.h, fo1_score_desc; vlm-fo1_b200/csrc/sampling.cuh score_row), on
top of the sampling oracle's warp(): the kept set is exactly the sampler's (top-k ties kept, top-p in the canonical order)."""
from __future__ import annotations

import numpy as np

from oracle.sampling import warp


def processed(logits, temperature: float, top_p: float, top_k: int, raw: bool = False) -> np.ndarray:
    """The scores row HF's _sample reports for this step (next_token_scores): float32 x = logits / T where the warpers keep the
    token, -inf elsewhere.  top_k == 1 keeps every token equal to the maximum (HF's TopK rule).  raw: a greedy row, the logits
    unchanged."""
    if raw:
        return np.asarray(logits, dtype=np.float32).copy()
    x, _, kept, _, _ = warp(logits, temperature, top_p, top_k)
    return np.where(kept, x, np.float32(-np.inf)).astype(np.float32)


def logprob_from(x: np.ndarray, kept: np.ndarray, token: int) -> float:
    """float64 log-probability of ``token`` given warp()'s x and kept set: (x_token - x_max) - ln(sum over the kept set of
    exp(x - x_max)); -inf for a token outside the kept set."""
    if not kept[token]:
        return -np.inf
    xmax = float(x.max())
    return (float(x[token]) - xmax) - float(np.log(np.sum(np.exp(x[kept].astype(np.float64) - xmax))))


def logprob(logits, temperature: float, top_p: float, top_k: int, token: int, raw: bool = False) -> float:
    """logprob_from() of processed()'s row.  raw: over the whole row with T = 1."""
    x, _, kept, _, _ = warp(logits, 1.0, 1.0, 0) if raw else warp(logits, temperature, top_p, top_k)
    return logprob_from(x, kept, token)
