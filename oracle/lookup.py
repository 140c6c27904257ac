"""Prompt-lookup decoding restated: the draft rule of transformers 5.5's PromptLookupCandidateGenerator.get_candidates with the
engine's extra cuts, and the acceptance rule of HF's assisted decoding (n_matches)."""
from typing import List, Optional, Sequence

MAX_DRAFTS = 16


def drafts(corpus: Sequence[int], num_tokens: int, max_ngram: int, stop_ids: Sequence[int] = (), cap: Optional[int] = None,
           engine: bool = True) -> List[int]:
    """The drafts of one sequence.  For n = min(max_ngram, len - 1) down to 1, the leftmost occurrence of the last n ids whose
    continuation is not empty gives the up to num_tokens ids that follow it, cut at the first stop id; the first n with such an
    occurrence decides.  ``engine``: also cut at the first negative id, at ``cap`` (max_new - emitted - 1) and at 16."""
    ids = [int(t) for t in corpus]
    L = len(ids)
    K = min(num_tokens, MAX_DRAFTS) if engine else num_tokens
    if engine and cap is not None:
        K = min(K, cap)
    if K <= 0:
        return []
    for n in range(min(max_ngram, L - 1), 0, -1):
        pat = ids[L - n:]
        for i in range(0, L - n):
            if ids[i:i + n] == pat:
                out = []
                for t in ids[i + n:min(i + n + K, L)]:
                    if t in stop_ids or (engine and t < 0):
                        break
                    out.append(t)
                return out
    return []


def n_matches(draft: Sequence[int], row_tokens: Sequence[int]) -> int:
    """HF's n_matches: the longest prefix of the drafts equal to the tokens the verify rows chose."""
    n = 0
    while n < len(draft) and int(draft[n]) == int(row_tokens[n]):
        n += 1
    return n
