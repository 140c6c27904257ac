"""CPU checks of the per-token scoring contract: tests/scores_oracle.py's processed / logprob against transformers' warper chain,
Fo1ForCausalLM.compute_transition_scores against transformers' own, and the host-side argument validation of fo1_score_rows and of
fo1_llm_generate with d.scores."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import scores_oracle as S


def _hf_processed(logits, T, p, k):
    """transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper output (float32 [V])."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = torch.from_numpy(np.asarray(logits, np.float32))[None].clone()
    ids = torch.zeros((1, 1), dtype=torch.long)
    if T != 1.0:
        s = TemperatureLogitsWarper(T)(ids, s)
    if 0 < k:
        s = TopKLogitsWarper(k)(ids, s)
    if p < 1.0:
        s = TopPLogitsWarper(p)(ids, s)
    return s[0].numpy()


def _same(got, ref):
    """Exactly equal: the same -inf pattern and bit-equal float32 finite values."""
    assert got.dtype == np.float32 and ref.dtype == np.float32
    assert np.array_equal(np.isneginf(got), np.isneginf(ref))
    fin = np.isfinite(ref)
    assert np.array_equal(got[fin].view(np.uint32), ref[fin].view(np.uint32))


def _check_logprob(row, T, p, k, ref):
    """scores_oracle.logprob against torch.log_softmax of the processed row, on kept tokens and one cut token."""
    ls = torch.log_softmax(torch.from_numpy(ref).double(), -1).numpy()
    kept = np.nonzero(np.isfinite(ref))[0]
    for t in kept[:: max(1, kept.size // 7)]:
        assert abs(S.logprob(row, T, p, k, int(t)) - ls[t]) < 1e-9, (T, p, k, t)
    cut = np.nonzero(~np.isfinite(ref))[0]
    if cut.size:
        assert S.logprob(row, T, p, k, int(cut[0])) == -np.inf


def test_processed_topk_matches_hf_with_ties():
    rng = np.random.default_rng(0)
    for trial in range(30):
        V = int(rng.integers(20, 400))
        row = rng.normal(0, 2, V).astype(np.float32)
        if trial % 2 == 0:      # a tie group straddling the k-th value, and one at the top
            row[rng.choice(V, 7, replace=False)] = np.sort(row)[::-1][min(5, V - 1)]
            row[rng.choice(V, 3, replace=False)] = row.max()
        for k in (1, 2, 3, 5, 6, 10, V - 1):
            for T in (0.7, 1.0, 1.5):
                ref = _hf_processed(row, T, 1.0, k)
                _same(S.processed(row, T, 1.0, k), ref)
                _check_logprob(row, T, 1.0, k, ref)


def test_processed_topp_matches_hf_tie_free():
    rng = np.random.default_rng(1)
    for trial in range(30):
        V = int(rng.integers(50, 2000))
        row = np.unique(rng.normal(0, 1.0 + trial % 4, V).astype(np.float32))    # tie-free: HF's sort order is the canonical one
        rng.shuffle(row)
        for T in (0.1, 0.7, 1.0, 1.5):
            for k in (0, 50):
                for p in (0.05, 0.5, 0.9):
                    ref = _hf_processed(row, T, p, k)
                    _same(S.processed(row, T, p, k), ref)
                    _check_logprob(row, T, p, k, ref)


def test_raw_rows():
    rng = np.random.default_rng(2)
    row = rng.normal(0, 3, 500).astype(np.float32)
    _same(S.processed(row, 0.7, 0.5, 5, raw=True), row)
    ls = torch.log_softmax(torch.from_numpy(row).double(), -1).numpy()
    for t in (0, 17, int(np.argmax(row)), 499):
        assert abs(S.logprob(row, 0.7, 0.5, 5, t, raw=True) - ls[t]) < 1e-9


def _model_cls():
    from vlm_fo1.model.fo1_model import Fo1ForCausalLM
    return Fo1ForCausalLM


@pytest.mark.parametrize("normalize", [False, True])
def test_compute_transition_scores_matches_hf(normalize):
    from transformers.generation.utils import GenerationMixin
    g = torch.Generator().manual_seed(3)
    B, P, n, V = 3, 5, 6, 40
    scores = tuple(torch.randn(B, V, generator=g) * 3 for _ in range(n))
    scores[2][1, 7:] = -float("inf")                                     # a sampled row: -inf outside the kept set
    seq = torch.randint(0, V, (B, P + n), generator=g)
    seq[1, P + 2] = 3
    stand_in = SimpleNamespace(config=SimpleNamespace(get_text_config=lambda: SimpleNamespace(vocab_size=V)))
    ref = GenerationMixin.compute_transition_scores(stand_in, seq, scores, normalize_logits=normalize)
    got = _model_cls().compute_transition_scores(None, seq, scores, normalize_logits=normalize)
    assert got.shape == (B, n) and torch.equal(got, ref)
    with pytest.raises(NotImplementedError, match="beam"):
        _model_cls().compute_transition_scores(None, seq, scores, beam_indices=torch.zeros((B, n), dtype=torch.long))


# ---------------------------------------------------------------------------------------------------------- host validation
def _lib():
    import fo1_b200
    return fo1_b200, fo1_b200.lib()


def _desc(T, p, k, n):
    import fo1_b200
    return fo1_b200._lib.sampling_desc([T] * n, [p] * n, [k] * n, [1] * n)


@pytest.mark.parametrize("case", ["n0", "ld", "ld_scores", "null_logits", "null_tokens", "null_logprobs", "temp", "raw_value"])
def test_score_rows_argument_validation_without_gpu(case):
    """fo1_score_rows checks its host arguments before any CUDA call."""
    _, L = _lib()
    P = ctypes.c_void_p(16)
    n, V, ld, lds = 2, 1000, 1000, 1000
    logits = tokens = logprobs = P
    sd, keep = _desc(0.7, 0.9, 50, 2)
    raw = None
    if case == "n0":
        n = 0
    elif case == "ld":
        ld = 999
    elif case == "ld_scores":
        lds = 10
    elif case == "null_logits":
        logits = None
    elif case == "null_tokens":
        tokens = None
    elif case == "null_logprobs":
        logprobs = None
    elif case == "temp":
        sd, keep = _desc(0.0, 0.9, 50, 2)
    elif case == "raw_value":
        raw = (ctypes.c_int32 * 2)(0, 2)
    rc = L.fo1_score_rows(logits, ld, n, V, ctypes.byref(sd), raw, tokens, logprobs, P, lds, None)
    assert rc == -1
    assert len(L.fo1_last_error()) > 0


@pytest.mark.parametrize("case", ["null_desc", "temp", "raw_value", "raw_not_greedy", "raw_temperature"])
def test_generate_sampling_and_scores_validation_without_gpu(case):
    """fo1_llm_generate checks the per-sequence host arrays of d.sampling and d.scores before it touches the model or the device."""
    F, L = _lib()
    E = __import__("importlib").import_module("vlm-fo1_b200.engine")
    d = E.GenerateDescC()
    d.n_seqs = 2
    T, k = 1.0, 1
    if case == "temp":
        T = -1.0
    if case == "raw_not_greedy":
        k = 50
    if case == "raw_temperature":
        T = 0.7
    sd, keep = _desc(T, 0.9, k, 2)
    raw = (ctypes.c_int32 * 2)(1, 3 if case == "raw_value" else 1)
    sc = F._lib.ScoreDesc(16, None, None, raw)
    d.sampling, d.scores = ctypes.pointer(sd), ctypes.pointer(sc)
    if case == "null_desc":
        rc = L.fo1_llm_generate(None, None, None)
    else:
        rc = L.fo1_llm_generate(ctypes.c_void_p(16), ctypes.byref(d), None)
    assert rc == -1
    msg = L.fo1_last_error().decode()
    assert {"null_desc": "null argument", "temp": "sampling: "}.get(case, "scores: ") in msg, msg
