"""CPU: oracle/beam.py against transformers' real beam search (GenerationMixin.generate with num_beams > 1) on a tiny random
Qwen2ForCausalLM built from a config.  The oracle is fed HF's own per-step log-prob rows (output_scores), and checks on the way
that the model's logits for each of its running histories are HF's rows for that beam (output_logits), so its histories are HF's
running sequences.  Sequences, beam_indices and sequences_scores must be equal; the step count must be the number of score rows."""
import itertools

import pytest
import torch

from oracle import beam as OB

V = 48          # small: eos ids are chosen often, so beams finish at every step


@pytest.fixture(scope="module")
def model():
    from transformers import Qwen2Config, Qwen2ForCausalLM
    cfg = Qwen2Config(vocab_size=V, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                      max_position_embeddings=128, tie_word_embeddings=False)
    torch.manual_seed(0)
    m = Qwen2ForCausalLM(cfg).eval()
    with torch.no_grad():
        m.lm_head.weight.mul_(8.0)        # peaked rows: scores spread over tens of nats, as a trained model's do
    return m


def _hf(model, prompt, N, T, eos, lp, es, nr, pad):
    ids = torch.tensor([prompt])
    with torch.no_grad():
        return model.generate(ids, attention_mask=torch.ones_like(ids), num_beams=N, max_new_tokens=T, do_sample=False, early_stopping=es,
                              length_penalty=lp, num_return_sequences=nr, eos_token_id=list(eos), pad_token_id=pad, output_scores=True,
                              output_logits=True, return_dict_in_generate=True)


def _check(model, prompt, N, T, eos, lp, es, nr, pad=1):
    out = _hf(model, prompt, N, T, eos, lp, es, nr, pad)
    P = len(prompt)

    def step(t, hist):
        assert t < len(out.scores), "the oracle runs more steps than HF"
        with torch.no_grad():
            x = torch.tensor([prompt + h for h in hist])
            logits = model(x).logits[:, -1].float()
        torch.testing.assert_close(logits, out.logits[t].float(), atol=1e-4, rtol=1e-4)
        return out.scores[t]

    r = OB.beam_search(step, N, OB.n_keep(N, len(eos)), T, eos, length_penalty=lp, early_stopping=es, num_return=nr)
    assert r.steps == len(out.scores)
    W = max(len(s) for s in r.sequences)
    seq = torch.tensor([prompt + s + [pad] * (W - len(s)) for s in r.sequences])
    bi = torch.tensor([b + [-1] * (W - len(b)) for b in r.beam_indices], dtype=out.beam_indices.dtype)
    assert torch.equal(out.sequences, seq), (out.sequences[:, P:], seq[:, P:])
    assert torch.equal(out.beam_indices, bi)
    assert torch.equal(out.sequences_scores, r.sequence_scores)
    return r


CASES = [  # (N, eos ids, length_penalty, early_stopping, max_new)
    (2, [3], 1.0, False, 6), (2, [3, 7], 0.0, True, 5), (2, [5], -0.5, "never", 7),
    (4, [3], 1.3, True, 6), (4, [3, 7], 1.0, "never", 6), (4, [11], 0.0, False, 8), (4, [3, 7], -0.5, False, 4),
    (8, [3], 1.0, False, 5), (8, [3, 7], 1.3, "never", 5), (8, [9], -0.5, True, 6), (8, [3, 7], 0.0, True, 4),
]


@pytest.mark.parametrize("N,eos,lp,es,T", CASES)
def test_oracle_matches_hf_beam_search(model, N, eos, lp, es, T):
    for seed in range(3):
        g = torch.Generator().manual_seed(100 * N + seed)
        prompt = torch.randint(12, V, (3 + seed,), generator=g).tolist()
        for nr in sorted({1, N // 2, N}):
            _check(model, prompt, N, T, eos, lp, es, nr)


@pytest.mark.parametrize("N,es", list(itertools.product([2, 4], [True, False, "never"])))
def test_oracle_every_beam_hits_the_limit(model, N, es):
    """No stop id the model emits: every hypothesis ends at max_new tokens."""
    r = _check(model, [20, 21, 22], N, 3, [V + 5], 1.0, es, N)
    assert all(len(s) == 3 for s in r.sequences)
