"""CPU checks of teacher-forced scoring: fo1_llm_loglik's host checks (they run before anything is enqueued, on a host-only model),
the label splice against the reference's rule, the target shift, and the loss reduction against transformers' ForCausalLMLoss."""
import ctypes
import json
import os
from importlib import import_module

import numpy as np
import pytest
import torch

VOCAB = 1000
IMG, REG = -200, -300


def _lib():
    import fo1_b200
    return fo1_b200._lib, fo1_b200.lib(), import_module("vlm-fo1_b200.engine")


def _host_model(L, E):
    cfg = E.ModelConfigC()
    cfg.llm_vocab = VOCAB
    m = ctypes.c_void_p()
    assert L.fo1_model_create(ctypes.byref(cfg), ctypes.byref(m)) == 0     # host only
    return m


# each case reaches its check through one descriptor field, so the ctypes layout of fo1_loglik_desc is pinned by the messages
CASES = {
    "target_above_vocab": "sequence 1 row 3: target 1000 is outside [0, 1000) and not -100",
    "target_negative": "sequence 0 row 1: target -5 is outside [0, 1000) and not -100",
    "last_row_scored": "sequence 1: its last row (5) is scored; it has no next token",
    "prefix_row_scored": "sequence 2 row 2 is scored inside its shared prefix of 3 rows",
    "prefix_all_logits": "fo1_llm_loglik: prefix: all_logits is not available with a shared prefix",
    "prefix_group_range": "fo1_llm_loglik: prefix: sequence 0: group 3 out of range",
    "empty_sequence": "fo1_llm_loglik: sequence 1 is empty",
    "null_targets": "fo1_llm_loglik: null argument",
    "null_embeds": "fo1_llm_loglik: null argument",
    "null_positions": "fo1_llm_loglik: null argument",
    "null_logprobs": "fo1_llm_loglik: null output",
    "null_seq_logprob": "fo1_llm_loglik: null output",
    "null_seq_count": "fo1_llm_loglik: null output",
    "null_model": "fo1_llm_loglik: null argument",
    "valid": "fo1_llm_loglik: model not finalized",
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_loglik_host_checks_without_gpu(case):
    F, L, E = _lib()
    lens = [4, 6, 5]
    tg = [-100] * sum(lens)
    tg[1], tg[4 + 3], tg[10 + 3] = 7, 9, 11       # valid scored rows: none last, none inside the prefix below
    d = F.LoglikDesc()
    d.n_seqs = 3
    d.seq_lens = (ctypes.c_int32 * 3)(*lens)
    d.inputs_embeds, d.position_ids = 16, 16
    d.logprobs, d.seq_logprob, d.seq_count = 16, 16, 16
    groups, plens = [-1, 0, 0], [3]
    if case == "target_above_vocab":
        tg[4 + 3] = VOCAB
    elif case == "target_negative":
        tg[1] = -5
    elif case == "last_row_scored":
        tg[4 + 5] = 3
    elif case == "prefix_row_scored":
        tg[10 + 2] = 3
    elif case == "prefix_all_logits":
        d.all_logits = 16
    elif case == "prefix_group_range":
        groups = [3, 0, 0]
    elif case == "empty_sequence":
        d.seq_lens = (ctypes.c_int32 * 3)(4, 0, 5)
    if case != "null_targets":
        d.targets = (ctypes.c_int32 * len(tg))(*tg)
    if case == "null_embeds":
        d.inputs_embeds = None
    if case == "null_positions":
        d.position_ids = None
    for name in ("logprobs", "seq_logprob", "seq_count"):
        if case == "null_" + name:
            setattr(d, name, None)
    px = F.PrefixDesc(1, (ctypes.c_int32 * 1)(*plens), 16, 16, (ctypes.c_int32 * 3)(*groups))
    d.prefix = ctypes.pointer(px)
    m = None if case == "null_model" else _host_model(L, E)
    try:
        rc = L.fo1_llm_loglik(m, ctypes.byref(d), None)
        msg = L.fo1_last_error().decode()
    finally:
        if m is not None:
            L.fo1_model_destroy(m)
    assert rc == -1
    assert CASES[case] in msg, msg
    assert msg.startswith("fo1_llm_loglik: "), msg


def test_loglik_without_prefix_accepts_a_scored_first_row():
    """Without a shared prefix every row but a sequence's last may be scored; the call then stops at the unfinalized model."""
    F, L, E = _lib()
    lens = [3, 2]
    d = F.LoglikDesc()
    d.n_seqs = 2
    d.seq_lens = (ctypes.c_int32 * 2)(*lens)
    d.inputs_embeds, d.position_ids, d.logprobs, d.seq_logprob, d.seq_count = 16, 16, 16, 16, 16
    d.all_logits = 16
    d.targets = (ctypes.c_int32 * 5)(0, VOCAB - 1, -100, 5, -100)
    m = _host_model(L, E)
    try:
        assert L.fo1_llm_loglik(m, ctypes.byref(d), None) == -1
        assert "model not finalized" in L.fo1_last_error().decode()
    finally:
        L.fo1_model_destroy(m)


# ---------------------------------------------------------------------------------------------------------------- labels
def _reference_splice(input_ids, labels, image_rows):
    """A restatement of the reference's region branch (omchat_qwen2_5_vl.py:300-368): split the ids and labels at every image and
    region marker, keep each text segment's labels, and insert IGNORE_INDEX for each marker's feature rows (an image's merged
    tokens, one row per region)."""
    ids = torch.tensor(input_ids)
    lab = torch.tensor(labels)
    image_indices = torch.where(ids == IMG)[0].tolist()
    region_indices = torch.where(ids == REG)[0].tolist()
    special = sorted([-1] + image_indices + region_indices + [ids.shape[0]])
    out = []
    for i in range(len(special) - 1):
        out.append(lab[special[i] + 1:special[i + 1]])
        if special[i + 1] in image_indices:
            out.append(torch.full((image_rows,), -100, dtype=lab.dtype))
        elif special[i + 1] in region_indices:
            out.append(torch.full((1,), -100, dtype=lab.dtype))
    return torch.cat(out).tolist()


def _golden_prompts():
    here = os.path.join(os.path.dirname(__file__), "golden")
    prompts = []
    z = np.load(os.path.join(here, "mm_utils.npz"), allow_pickle=True)
    for k in z.files:
        a = z[k]
        if a.dtype.kind in "iu" and a.ndim == 2 and a.shape[0] == 1 and (a == IMG).any():     # the prompts prepare_inputs built
            prompts.append([int(x) for x in a[0]])
    with open(os.path.join(here, "prompt_data.json")) as fh:
        data = json.load(fh)

    def walk(x):
        if isinstance(x, list) and x and all(isinstance(t, int) for t in x) and IMG in x:
            prompts.append(list(x))
        elif isinstance(x, dict):
            for v in x.values():
                walk(v)
        elif isinstance(x, list):
            for v in x:
                walk(v)
    walk(data)
    return prompts


def test_label_splice_matches_the_reference_rule():
    P = import_module("vlm-fo1_b200.pipeline")
    prompts = _golden_prompts()
    assert len(prompts) >= 2, "the golden fixtures hold prompts with <image> and <regionN> placeholders"
    g = torch.Generator().manual_seed(0)
    n_regions = 0
    for i, ids in enumerate(prompts):
        n_regions += sum(1 for t in ids if t == REG)
        for image_rows in (1, 16, 1024):
            labels = torch.randint(0, 151643, (len(ids),), generator=g).tolist()
            labels = [-100 if (j % 3 == 0 or t in (IMG, REG)) else x for j, (t, x) in enumerate(zip(ids, labels))]
            got = P.splice_labels(ids, labels, image_rows)
            assert got == _reference_splice(ids, labels, image_rows), f"prompt {i}, {image_rows} image rows"
            assert len(got) == len(ids) - 1 + image_rows
    assert n_regions > 0, "some golden prompt has region placeholders"


def test_shift_targets_is_hf_shift():
    P = import_module("vlm-fo1_b200.pipeline")
    lab = torch.tensor([[-100, 5, 6, -100, 8]])
    shifted = torch.nn.functional.pad(lab, (0, 1), value=-100)[..., 1:]      # ForCausalLMLoss's shift
    assert P.shift_targets(lab[0].tolist()) == shifted[0].tolist()


# ---------------------------------------------------------------------------------------------------------------- loss
@pytest.mark.parametrize("case", ["ragged", "all_ignored", "one_row"])
def test_loss_reduction_equals_for_causal_lm_loss(case):
    """causal_lm_loss over per-sequence sums of log-probabilities equals transformers' ForCausalLMLoss on the same fp32 logits:
    the mean over every non-ignored shifted label of the batch (ragged counts per sequence), NaN when none is scored."""
    from transformers.loss.loss_utils import ForCausalLMLoss
    P = import_module("vlm-fo1_b200.pipeline")
    g = torch.Generator().manual_seed(1)
    V = 50
    lens = {"ragged": [7, 3, 12], "all_ignored": [4, 5], "one_row": [2]}[case]
    seq_lp, seq_n, all_logits, all_labels = [], [], [], []
    for L in lens:
        logits = torch.randn(L, V, generator=g) * 3
        labels = torch.randint(0, V, (L,), generator=g)
        if case == "all_ignored":
            labels[:] = -100
        else:
            labels[torch.rand(L, generator=g) < 0.4] = -100
            labels[1] = 3
        tg = torch.tensor(P.shift_targets(labels.tolist()))
        lp = torch.log_softmax(logits.double(), -1)
        keep = tg != -100
        seq_lp.append(float(lp[keep.nonzero().view(-1), tg[keep]].sum()))
        seq_n.append(int(keep.sum()))
        all_logits.append(logits)
        all_labels.append(labels)
    got = P.causal_lm_loss(seq_lp, seq_n)
    # HF shifts per sequence: pack the sequences as a batch of one row each and add their loss sums
    ref_sum = sum(float(ForCausalLMLoss(lg[None], lb[None], V, num_items_in_batch=1)) for lg, lb in zip(all_logits, all_labels))
    n = sum(seq_n)
    if case == "all_ignored":
        assert np.isnan(got)
        assert all(torch.isnan(ForCausalLMLoss(lg[None], lb[None], V)) for lg, lb in zip(all_logits, all_labels))
    else:
        assert got == pytest.approx(ref_sum / n, rel=1e-5)
        if len(lens) == 1:
            assert got == pytest.approx(float(ForCausalLMLoss(all_logits[0][None], all_labels[0][None], V)), rel=1e-5)
