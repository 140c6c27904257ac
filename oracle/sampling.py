"""CPU restatement of the engine's sampled decoding (include/fo1.h, fo1_sampling_desc; vlm-fo1_b200/csrc/sampling.cuh).

HF generate's sampling branch as transformers pins it: TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> softmax
-> multinomial, with the orders HF leaves open made explicit:
  * x = logits / T in float32 (IEEE division, as torch does); T == 1 leaves x as is.
  * canonical order: x descending, then token index ascending.
  * top-k (1 < k < V): keep every token with x >= the k-th largest x (ties kept).  k == 1: the arg-max, lowest index first.
  * top-p (p < 1): weights exp(x - max) in float64 over the kept tokens; keep a token iff the weight ranked above it is < p Z.
  * draw: u = (x0 >> 8) * 2^-24 of Philox4x32-10(key = (seed lo32, seed hi32), counter = (step, 0, 0, 0)); the first kept token
    whose inclusive cumulative weight exceeds u Z_kept.
Each draw also reports a decidability margin (as a fraction of Z): the distance of u Z_kept from the nearest cumulative boundary
and of p from the nearest cumulative boundary of the top-p cut.  A device result may differ from this one only where that margin
is within the device's rounding (fp32 exp, 2^-40 fixed-point weights)."""
from __future__ import annotations

import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Random123's philox4x32 with 10 rounds: ctr = 4 x uint32, key = 2 x uint32 -> 4 x uint32."""
    c = [int(v) & _MASK for v in ctr]
    k0, k1 = int(key[0]) & _MASK, int(key[1]) & _MASK
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & _MASK, (k1 + W1) & _MASK
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & _MASK, p1 & _MASK, ((p0 >> 32) ^ c[3] ^ k1) & _MASK, p0 & _MASK]
    return c


def uniform(seed: int, step: int) -> float:
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    x0 = philox4x32_10((step, 0, 0, 0), (seed & _MASK, seed >> 32))[0]
    return (x0 >> 8) * 2.0 ** -24


def scaled(logits, temperature: float) -> np.ndarray:
    x = np.asarray(logits, dtype=np.float32)
    if np.float32(temperature) != np.float32(1.0):
        x = x / np.float32(temperature)
    return x


def canonical_order(x: np.ndarray) -> np.ndarray:
    """Token indices by x descending, then index ascending (-0.0 == +0.0)."""
    return np.lexsort((np.arange(x.size), -(x.astype(np.float64) + 0.0)))


def kept_topk(x: np.ndarray, k: int) -> np.ndarray:
    """Boolean mask of the tokens the top-k stage keeps (HF TopKLogitsWarper: ties at the threshold kept)."""
    V = x.size
    if k <= 0 or k >= V:
        return np.ones(V, bool)
    thr = np.sort(x)[::-1][k - 1]
    return x >= thr


def warp(logits, temperature: float, top_p: float, top_k: int):
    """-> (x float32, order, kept mask after top-k and top-p, float64 probabilities over the vocabulary, top-p margin)."""
    x = scaled(logits, temperature)
    order = canonical_order(x)
    kept = kept_topk(x, top_k)
    xmax = float(x.max())
    w = np.where(kept, np.exp(x.astype(np.float64) - xmax), 0.0)
    margin_p = np.inf
    if top_p < 1.0:
        wo = w[order]
        Z = wo.sum()
        incl = np.cumsum(wo)
        before = incl - wo
        keep_o = (before < top_p * Z) & (wo > 0)
        keep_o[0] = True
        live = wo > 0
        margin_p = float(np.min(np.abs(incl[live] - top_p * Z)) / Z)
        k2 = np.zeros_like(kept)
        k2[order[keep_o]] = True
        kept = kept & k2
        w = np.where(kept, w, 0.0)
    probs = w / w.sum()
    return x, order, kept, probs, margin_p


def sample(logits, temperature: float, top_p: float, top_k: int, seed: int, step: int):
    """-> dict(token, margin, u): the token the contract picks and the decidability margin of the pick (fraction of Z)."""
    x = scaled(logits, temperature)
    if top_k == 1:
        return dict(token=int(np.argmax(x)), margin=np.inf, u=None)
    x, order, kept, probs, margin_p = warp(logits, temperature, top_p, top_k)
    xmax = float(x.max())
    w = np.where(kept, np.exp(x.astype(np.float64) - xmax), 0.0)[order]
    live = w > 0
    incl = np.cumsum(w)
    Z = incl[-1]
    u = uniform(seed, step)
    t = u * Z
    pos = int(np.argmax(incl > t)) if (incl > t).any() else int(np.nonzero(live)[0][-1])
    bounds = np.concatenate([[0.0], incl[live]])
    margin_u = float(np.min(np.abs(bounds - t)) / Z)
    return dict(token=int(order[pos]), margin=min(margin_u, margin_p), u=u)
