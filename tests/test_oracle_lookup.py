"""oracle/lookup.py against transformers' own PromptLookupCandidateGenerator.get_candidates and n_matches expression."""
import numpy as np
import pytest
import torch

from oracle import lookup as O

P = pytest.importorskip("transformers.generation.candidate_generator")


def _hf(corpus, K, ngram, eos):
    g = P.PromptLookupCandidateGenerator(eos_token_id=torch.tensor(eos or [-1]), num_output_tokens=K, max_matching_ngram_size=ngram,
                                         max_length=10 ** 6)
    ids = torch.tensor([corpus], dtype=torch.long)
    cand, _ = g.get_candidates(ids)
    return cand[0, len(corpus):].tolist()


def _corpora(rng):
    for _ in range(60):
        L = int(rng.integers(1, 80))
        vocab = int(rng.choice([3, 8, 50, 1000]))          # small vocabularies repeat, large ones mostly do not match
        c = rng.integers(0, vocab, L).tolist()
        if rng.random() < 0.3 and L > 4:                   # placeholders, as prepare_inputs leaves them
            for j in rng.choice(L, 2, replace=False):
                c[int(j)] = int(rng.choice([-200, -300]))
        yield c


@pytest.mark.parametrize("ngram", [1, 2, 3])
def test_drafts_equal_hf(ngram):
    rng = np.random.default_rng(ngram)
    n = matched = 0
    for c in _corpora(rng):
        for K in (1, 4, 10, 16, 20):
            eos = [int(rng.integers(0, 8))] if rng.random() < 0.5 else []
            hf = _hf(c, K, ngram, eos)
            got = O.drafts(c, K, ngram, eos)
            # the engine's extra cuts: the first negative id and 16 drafts
            want = hf[:16]
            for i, t in enumerate(want):
                if t < 0:
                    want = want[:i]
                    break
            assert got == want, (c, K, ngram, eos, hf)
            assert O.drafts(c, K, ngram, eos, engine=False) == hf
            n += 1
            matched += bool(hf)
    assert 0 < matched < n            # both matches and misses were covered


def test_drafts_cap_and_no_match():
    assert O.drafts([1, 2, 3, 1, 2], 4, 2) == [3, 1, 2]
    assert O.drafts([1, 2, 3, 1, 2], 4, 2, cap=1) == [3]
    assert O.drafts([1, 2, 3, 1, 2], 4, 2, cap=0) == []
    assert O.drafts([1, 2, 3, 4], 4, 3) == []                    # no earlier occurrence of any suffix
    assert O.drafts([5, 7, 9, 5], 4, 1, stop_ids=[7]) == []      # the eos cut leaves nothing: no smaller n is tried (HF)
    assert O.drafts([5, -200, 9, 5], 4, 1) == []


def test_n_matches_equals_hf_expression():
    rng = np.random.default_rng(0)
    for _ in range(200):
        k = int(rng.integers(1, 8))
        cand = torch.from_numpy(rng.integers(0, 3, (1, k)))
        sel = torch.from_numpy(rng.integers(0, 3, (1, k + 1)))
        hf = int(((~(cand == sel[:, :-1])).cumsum(dim=-1) < 1).sum())
        assert O.n_matches(cand[0].tolist(), sel[0].tolist()) == hf
