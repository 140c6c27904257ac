"""HF generate's logits processors restated in fp32 torch operations, in GenerationMixin._get_logits_processor's order:
SequenceBias -> NoRepeatNGram -> NoBadWords -> MinLength -> MinNewTokensLength -> SuppressTokens -> SuppressTokensAtBegin.

``ps`` is anything with engine.ProcessorSet's fields; ``history`` is HF's input_ids of one sequence (prompt ids, placeholders
included, then the emitted tokens) and ``prompt_len`` the prompt's length, so the output column is len(history) - prompt_len."""
import math

import torch


def _bias(scores, history, seqs):
    """SequenceBiasLogitsProcessor.__call__ for one row: length-1 biases set first, then the longer sequences added in order."""
    V = scores.shape[-1]
    bias = torch.zeros((V,), dtype=torch.float32)
    one = torch.zeros((V,), dtype=torch.float32)
    for w, b in seqs:
        if len(w) == 1:
            one[w[0]] = b
    bias += one
    for w, b in seqs:
        if len(w) == 1 or len(w) > len(history):
            continue
        match = list(history[len(history) - (len(w) - 1):]) == list(w[:-1])
        bias[w[-1]] += torch.tensor(b if match else 0.0, dtype=torch.float32)
    return scores + bias


def process(scores: torch.Tensor, history, prompt_len: int, ps) -> torch.Tensor:
    """One fp32 row [V] -> the processed row (a new tensor)."""
    x = scores.clone().float()
    L, col = len(history), len(history) - prompt_len
    V = x.shape[-1]
    if ps.sequence_bias:
        x = _bias(x, history, [(tuple(w), float(b)) for w, b in ps.sequence_bias])
    n = ps.no_repeat_ngram_size
    if n > 0 and L + 1 >= n:
        prefix = tuple(history[L - n + 1:])
        banned = [history[i + n - 1] for i in range(L - n + 1) if tuple(history[i:i + n - 1]) == prefix]
        for t in banned:
            x[t] = -math.inf                 # torch indexing: a negative id wraps to V + id
    if ps.bad_words_ids:
        x = _bias(x, history, [(tuple(w), -math.inf) for w in ps.bad_words_ids])
    vocab = torch.arange(V)
    eos = torch.isin(vocab, torch.tensor(list(ps.eos_token_ids), dtype=torch.long))
    if ps.min_length > 0 and L < ps.min_length:
        x = torch.where(eos, -math.inf, x)
    if ps.min_new_tokens > 0 and col < ps.min_new_tokens:
        x = torch.where(eos, -math.inf, x)
    if ps.suppress_tokens:
        x = torch.where(torch.isin(vocab, torch.tensor(list(ps.suppress_tokens))), -math.inf, x)
    if ps.begin_suppress_tokens and col == 0:
        x = torch.where(torch.isin(vocab, torch.tensor(list(ps.begin_suppress_tokens))), -math.inf, x)
    return x


def greedy_loop(step_logits, prompt, ps, max_new_tokens: int, eos_ids=()):
    """The greedy decode loop HF runs with these processors: ``step_logits(ids) -> fp32 [V]`` of the next position.  Returns the
    emitted tokens (the stop token included)."""
    ids = list(prompt)
    out = []
    for _ in range(max_new_tokens):
        row = process(step_logits(ids), ids, len(prompt), ps)
        t = int(torch.argmax(row))
        out.append(t)
        ids.append(t)
        if t in eos_ids:
            break
    return out
