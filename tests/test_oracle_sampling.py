"""CPU checks of the sampling contract (oracle/sampling.py) and of fo1_sample_tokens' host-side argument validation."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sampling as S


@pytest.mark.parametrize("ctr,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, expect):
    """Random123's known-answer vectors of philox4x32-10."""
    assert tuple(S.philox4x32_10(ctr, key)) == expect


def _hf_chain(logits, T, p, k):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(np.asarray(logits, np.float32))[None].clone()
    ids = torch.zeros((1, 1), dtype=torch.long)
    if T != 1.0:
        s = TemperatureLogitsWarper(T)(ids, s)
    if 0 < k:
        s = TopKLogitsWarper(k)(ids, s)
    if p < 1.0:
        s = TopPLogitsWarper(p)(ids, s)
    return torch.softmax(s.double(), -1)[0].numpy()


def test_topk_matches_hf_with_ties():
    rng = np.random.default_rng(0)
    for trial in range(40):
        V = int(rng.integers(20, 400))
        row = rng.normal(0, 2, V).astype(np.float32)
        if trial % 2 == 0:      # a tie group straddling the k-th value
            row[rng.choice(V, 7, replace=False)] = np.sort(row)[::-1][min(5, V - 1)]
        for k in (2, 3, 5, 6, 10, V - 1):
            for T in (0.7, 1.0, 1.5):
                _, _, kept, _, _ = S.warp(row, T, 1.0, k)
                ref = _hf_chain(row, T, 1.0, k) > 0
                assert np.array_equal(kept, ref), (trial, k, T)


def test_topp_matches_hf_tie_free():
    rng = np.random.default_rng(1)
    for trial in range(40):
        V = int(rng.integers(50, 2000))
        row = (rng.normal(0, 1.0 + trial % 4, V)).astype(np.float32)
        row = np.unique(row)                      # tie-free: HF's sort order is then the canonical order
        rng.shuffle(row)
        for T in (0.1, 0.7, 1.0, 1.5):
            for k in (0, 50):
                for p in (0.05, 0.5, 0.9):
                    _, _, kept, probs, _ = S.warp(row, T, p, k)
                    ref = _hf_chain(row, T, p, k)
                    assert np.array_equal(kept, ref > 0), (trial, T, k, p)
                    assert np.abs(probs - ref).max() < 1e-6


def test_draws_chi_square():
    """2^16 draws of one row over (seed, step) pairs against the oracle's probabilities."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(2)
    row = rng.normal(0, 1.5, 64).astype(np.float32)
    T, p, k = 0.9, 0.95, 40
    _, order, kept, probs, _ = S.warp(row, T, p, k)
    w = probs[order]
    incl = np.cumsum(w)
    counts = np.zeros(row.size, np.int64)
    n = 1 << 16
    for i in range(n):
        u = S.uniform(seed=1000 + (i >> 8), step=i & 255)
        counts[order[min(int(np.searchsorted(incl, u * incl[-1], side="right")), row.size - 1)]] += 1
    # the tokens the draw can reach, pooled so that every expected count is >= 5
    exp = probs * n
    live = np.nonzero(exp >= 5)[0]
    rest = np.setdiff1d(np.arange(row.size), live)
    obs = np.concatenate([counts[live], [counts[rest].sum()]])
    ex = np.concatenate([exp[live], [exp[rest].sum()]])
    if ex[-1] < 5:
        obs, ex = np.concatenate([obs[:-2], [obs[-2:].sum()]]), np.concatenate([ex[:-2], [ex[-2:].sum()]])
    assert counts[~kept].sum() == 0
    assert chisquare(obs, ex).pvalue > 1e-3


def test_oracle_draw_is_the_cumulative_rule():
    """sample() picks the first kept token (canonical order) whose inclusive weight exceeds u Z."""
    rng = np.random.default_rng(3)
    row = rng.normal(0, 1, 300).astype(np.float32)
    row[10] = row[20] = row[30] = row.max() + 1.0          # a tie at the top: lowest index first
    for step in range(50):
        r = S.sample(row, 1.0, 1.0, 0, seed=7, step=step)
        x, order, kept, probs, _ = S.warp(row, 1.0, 1.0, 0)
        incl = np.cumsum(probs[order])
        assert r["token"] == order[int(np.argmax(incl > r["u"]))]
    assert S.sample(row, 1.0, 1.0, 1, seed=7, step=0)["token"] == 10


def _desc(T, p, k, seed):
    import fo1_b200
    return fo1_b200._lib.sampling_desc(T, p, k, seed)


@pytest.mark.parametrize("T,p,k,n", [
    (0.0, 0.9, 50, 1), (-1.0, 0.9, 50, 1), (float("inf"), 0.9, 50, 1), (float("nan"), 0.9, 50, 1),
    (0.7, 0.0, 50, 1), (0.7, -0.5, 50, 1), (0.7, 1.5, 50, 1), (0.7, 0.9, -1, 1), (0.7, 0.9, 50, 0),
])
def test_sample_tokens_argument_validation_without_gpu(T, p, k, n):
    """Host-side checks of fo1_sample_tokens run before any CUDA call, so they are testable on a CPU box."""
    import fo1_b200
    L = fo1_b200.lib()
    m = max(n, 1)
    sd, keep = _desc([T] * m, [p] * m, [k] * m, [1] * m)
    rc = L.fo1_sample_tokens(ctypes.c_void_p(16), 1000, n, 1000, ctypes.byref(sd), ctypes.c_void_p(16), ctypes.c_void_p(16),
                             ctypes.c_void_p(16), 1 << 20, None)
    assert rc == -1
    assert len(L.fo1_last_error()) > 0


def test_sample_tokens_workspace_bytes():
    import fo1_b200
    L = fo1_b200.lib()
    assert L.fo1_sample_tokens_workspace_bytes(3) >= 3 * 24
    assert L.fo1_sample_tokens_workspace_bytes(0) == 0
