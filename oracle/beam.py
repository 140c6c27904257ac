"""CPU restatement of transformers' beam search selection (GenerationMixin._beam_search with _get_top_k_continuations,
_get_running_beams_for_next_iteration, _update_finished_beams, _check_early_stop_heuristic and
_beam_search_has_unfinished_sequences; transformers 5.5 generation/utils.py) for ONE prompt, over log-prob rows a caller
supplies.  Every fp32 operation is the cited code's, in its order.  Where torch.topk leaves the order of equal scores
unspecified, this uses the engine's canonical order: score descending, then flat index (beam * V + token, or the position in the
merged finished set) ascending -- a stable descending sort.

A continuation "hits" the stop test if its token is one of ``stop_ids`` (HF's EosTokenCriteria; the reference's
KeywordsStoppingCriteria stops on <|im_end|>, which is also an eos id) or if it is the ``max_new``-th token (MaxLengthCriteria)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Sequence

import torch

NEG = -1.0e9


@dataclass
class Hyp:
    tokens: List[int] = field(default_factory=list)
    beam_indices: List[int] = field(default_factory=list)     # prompt * N + parent beam of each token
    logprobs: List[float] = field(default_factory=list)       # each token's log-prob under its parent's row


@dataclass
class BeamResult:
    sequences: List[List[int]]            # the best num_return hypotheses, best first
    beam_indices: List[List[int]]
    logprobs: List[List[float]]
    sequence_scores: torch.Tensor         # fp32 [num_return]
    steps: int                            # loop iterations run (rows of `scores`)
    running: List[List[List[int]]]        # running[t][j]: tokens of running beam j after step t


def _top(x: torch.Tensor, k: int) -> torch.Tensor:
    """Indices of the k largest, descending, equal values by index ascending."""
    return torch.sort(x, descending=True, stable=True).indices[:k]


def beam_search(step: Callable[[int, List[List[int]]], torch.Tensor], num_beams: int, n_keep: int, max_new: int, stop_ids: Sequence[int],
                length_penalty: float = 1.0, early_stopping=False, num_return: int = 1, beam_offset: int = 0,
                rows_are_logprobs: bool = True) -> BeamResult:
    """``step(t, histories)`` -> fp32 [N, V]: the rows of the N running beams at step t (histories: their t generated tokens), as
    log-probs, or logits when ``rows_are_logprobs`` is False (then log_softmax is applied, as HF does).  ``beam_offset``: the
    prompt's first row (prompt index * N) added to every beam index."""
    N, K = num_beams, n_keep
    stop = set(int(s) for s in stop_ids)
    run = [Hyp() for _ in range(N)]
    run_score = torch.zeros(N, dtype=torch.float32)
    run_score[1:] = NEG
    fin = [Hyp() for _ in range(N)]
    fin_score = torch.full((N,), NEG, dtype=torch.float32)
    fin_done = torch.zeros(N, dtype=torch.bool)
    unsat = torch.ones((), dtype=torch.bool)
    top_mask = torch.arange(K) < N
    running, steps = [], 0
    for t in range(max_new):
        rows = step(t, [list(h.tokens) for h in run]).to(torch.float32)
        lp = rows if rows_are_logprobs else torch.nn.functional.log_softmax(rows, dim=-1)
        V = lp.shape[1]
        acc = (lp + run_score[:, None]).reshape(N * V)
        idx = _top(acc, K)
        ts = acc[idx]
        par, tok = idx // V, idx % V
        hits = torch.tensor([t + 1 >= max_new or int(x) in stop for x in tok.tolist()], dtype=torch.bool)
        # _get_running_beams_for_next_iteration
        rs = ts + hits.to(torch.float32) * NEG
        sel = _top(rs, N)
        cand = [Hyp(run[int(p)].tokens + [int(x)], run[int(p)].beam_indices + [beam_offset + int(p)],
                    run[int(p)].logprobs + [float(lp[int(p), int(x)])]) for p, x in zip(par.tolist(), tok.tolist())]
        new_run = [cand[int(k)] for k in sel]
        new_score = rs[sel]
        # _update_finished_beams
        did = hits & top_mask
        fs = ts / ((t + 1) ** length_penalty)
        full = torch.all(fin_done) & (early_stopping is True)
        fs += full.to(torch.float32) * NEG
        fs += (~unsat).to(torch.float32) * NEG
        fs += (~did) * NEG
        merged_score = torch.cat((fin_score, fs))
        merged = fin + cand
        merged_done = torch.cat((fin_done, did))
        msel = _top(merged_score, N)
        fin = [merged[int(m)] for m in msel]
        fin_score, fin_done = merged_score[msel], merged_done[msel]
        run, run_score = new_run, new_score
        running.append([list(h.tokens) for h in run])
        steps = t + 1
        # _check_early_stop_heuristic at cur_len + 1, then _beam_search_has_unfinished_sequences
        best_len = max_new if (early_stopping == "never" and length_penalty > 0.0) else t + 1
        best = run_score[:1] / (best_len ** length_penalty)
        worst = torch.where(fin_done, torch.min(fin_score), NEG)
        unsat = unsat & torch.any(best > worst)
        go = bool(unsat) and not (bool(torch.all(fin_done)) and early_stopping is True) and not bool(torch.all(hits))
        if not go:
            break
    return BeamResult([h.tokens for h in fin[:num_return]], [h.beam_indices for h in fin[:num_return]], [h.logprobs for h in fin[:num_return]],
                      fin_score[:num_return].clone(), steps, running)


def n_keep(num_beams: int, n_eos: int) -> int:
    """HF's beams_to_keep: max(2, 1 + number of eos ids) * num_beams."""
    return max(2, 1 + n_eos) * num_beams
