"""-m gpu: shared-prefix generation (include/fo1.h, fo1_prefix_desc) is bit-identical to generating every sequence in full.

  1. fo1_prefix_attention against the causal varlen attention over each whole sequence, on the own rows;
  2. the pipeline at the released widths (the reduced-depth engine of test_gpu_batch_invariance.py): shared against forced-unshared
     on the same batch, both decode paths, greedy, sampled, scored and streamed, and against each sample alone where the decode
     attention splits the keys as it does for one sequence;
  3. the towers run once per unique image;
  4. num_return_sequences on the fabricated checkpoint.
Every comparison is torch.equal."""
from importlib import import_module

import numpy as np
import pytest
import torch

from tests.test_gpu_batch_invariance import _first_diff, _sample, _splits, pipe  # noqa: F401 (pipe: fixture)
from tests.test_gpu_sampling import fab  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def _eng_mod():
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine")


# ------------------------------------------------------------------------------------------------------- 1. the attention
PREFIXES = [1, 63, 64, 65, 127, 128, 129, 1195, 3000]


@pytest.mark.parametrize("own", [1, 2, 17, 64, 130])
def test_prefix_attention_equals_full_causal(own):
    """One launch: a sequence per prefix length plus a loner (P = 0), each with `own` own rows, against the causal attention over
    each whole sequence alone (whose query tiles and key tiles start at the sequence start, as the prefill's tile table makes them)."""
    E, ops = _eng_mod(), import_module("vlm-fo1_b200.ops")
    qh, kvh, hd = 16, 2, 128
    pre = PREFIXES + [0]
    n = len(pre)
    lens = [p + own for p in pre]
    cap = (max(lens) + 1 + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(own)
    kc = torch.randn(n, cap, kvh * hd, device="cuda", generator=g).bfloat16()      # finite everywhere, also past each sequence
    vc = torch.randn(n, cap, kvh * hd, device="cuda", generator=g).bfloat16()
    scale = hd ** -0.5
    q_own, ref = [], []
    for b in range(n):
        q = (torch.randn(lens[b], qh * hd, device="cuda", generator=g) * 2.0).bfloat16()
        cu = torch.tensor([0, lens[b]], dtype=torch.int32, device="cuda")
        full = ops.attention_varlen(q, kc[b, :lens[b]], vc[b, :lens[b]], cu, lens[b], qh, kvh, hd, scale, causal=True)
        q_own.append(q[pre[b]:]); ref.append(full[pre[b]:])
    got = E.prefix_attention(torch.cat(q_own), kc, vc, pre, [own] * n, qh, kvh, scale)
    ref = torch.cat(ref)
    assert torch.isfinite(ref.float()).all()
    off = np.cumsum([0] + [own] * n)
    for b in range(n):
        a, r = got[off[b]:off[b + 1]], ref[off[b]:off[b + 1]]
        assert torch.equal(a, r), f"P={pre[b]} own={own}: {_first_diff(a, r)}"


# ------------------------------------------------------------------------------------------------------- 2. the pipeline
MAX_NEW = 6
TAIL = [151645, 198, 151644, 77091, 198]


def _prompt(base, q, fill=0, head=None):
    """The base prompt through its last region placeholder, `fill` filler tokens, a 15-30 token question of its own, the turn tail.
    head: a first token of its own (the prompt then shares no row with the others)."""
    cut = max(i for i, t in enumerate(base.input_ids) if t == -300) + 1
    gq = torch.Generator().manual_seed(500 + q)
    question = [1000 + q] + torch.randint(0, 151643, (14 + q % 16,), generator=gq).tolist()
    ids = list(base.input_ids[:cut]) + [7] * fill + question + TAIL
    if head is not None:
        ids[0] = head
    return ids


def _ask(base, ids, clone=True):
    """A question about base's image: fresh tensors of the same content (what prepare_inputs builds every call)."""
    P = import_module("vlm-fo1_b200.pipeline")
    t = (lambda x: x.clone()) if clone else (lambda x: x)
    return P.SampleInputs(ids, t(base.pixel_values), base.grid_hw, t(base.image_aux), t(base.boxes))


def _fill_for(base, residue):
    """Filler tokens that make the shared prefix (in spliced rows) == residue mod 64."""
    cut = max(i for i, t in enumerate(base.input_ids) if t == -300) + 1
    rows = cut - 1 + base.grid_hw[0] * base.grid_hw[1] // 4
    return (residue - rows) % 64


def _run(pipe, samples, shared, sampling=None, scored=False, stream=False):
    pipe._share_inputs = shared
    cols = []
    try:
        on = (lambda lo, hi, t, l: cols.append((lo, hi, t.copy(), l.copy()))) if stream else None
        out = pipe.generate(samples, MAX_NEW, stop_ids=[], early_exit_interval=0, want_prefill_logits=True, want_logits=True,
                            sampling=sampling, want_logprobs=scored, want_scores=scored, on_tokens=on)
    finally:
        pipe._share_inputs = True
    res = {k: out[k].clone() for k in ("tokens", "lens", "prefill_logits", "logits") + (("logprobs", "scores") if scored else ())}
    res["path"] = pipe.eng.last_decode_path()
    if stream:
        B = len(samples)
        toks = np.zeros((B, MAX_NEW), np.int32)
        for lo, hi, t, _ in cols:
            toks[:, lo:hi] = t
        res["streamed"] = torch.from_numpy(toks)
        res["streamed_lens"] = torch.from_numpy(cols[-1][3])
    return res


def _assert_same(a, b, what, rows=None):
    rows = range(a["tokens"].shape[0]) if rows is None else rows
    for key in ("tokens", "lens", "logprobs", "streamed", "streamed_lens"):
        if key in a:
            assert torch.equal(a[key], b[key]), f"{what} {key}: {a[key].tolist()} vs {b[key].tolist()}"
    assert torch.equal(a["prefill_logits"], b["prefill_logits"]), f"{what} prefill logits: {_first_diff(a['prefill_logits'], b['prefill_logits'])}"
    for key in ("logits", "scores"):
        if key not in a:
            continue
        for r in rows:
            for t in range(int(a["lens"][r])):       # rows past a sequence's stop column are unspecified
                x, y = a[key][t, r], b[key][t, r]
                assert torch.equal(x, y), f"{what} {key} column {t} row {r}: {_first_diff(x, y)}"


def _check(pipe, samples, what, expect_path, alone=False, **kw):
    shared = _run(pipe, samples, True, **kw)
    ref = _run(pipe, samples, False, **kw)
    assert shared["path"] == ref["path"] == expect_path, what
    _assert_same(ref, shared, what)
    if alone:
        for b, s in enumerate(samples):
            one = _run(pipe, [s], False)
            sub = {k: (v[b:b + 1] if k in ("tokens", "lens", "prefill_logits") else v[:, b:b + 1]) for k, v in shared.items()
                   if k in ("tokens", "lens", "prefill_logits", "logits")}
            _assert_same(one, sub, f"{what} sample {b} alone")


BASE = (150, 112, 3)


@pytest.mark.parametrize("B", [2, 8, 20])
def test_shared_greedy_persistent(pipe, B):
    base = _sample(*BASE)
    samples = [_ask(base, _prompt(base, q), clone=q % 2 == 1) for q in range(B)]
    _check(pipe, samples, f"greedy B={B}", 1, alone=_splits(B, False) == _splits(1, False))


@pytest.mark.parametrize("B,no_mega", [(33, False), (8, True)])
def test_shared_greedy_per_kernel(pipe, B, no_mega, monkeypatch):
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    base = _sample(*BASE)
    samples = [_ask(base, _prompt(base, q)) for q in range(B)]
    _check(pipe, samples, f"per-kernel B={B}", 0)


def test_shared_sampled_scored_streamed(pipe):
    E = _eng_mod()
    base = _sample(*BASE)
    samples = [_ask(base, _prompt(base, q)) for q in range(6)] + [_ask(base, _prompt(base, 2))]     # identical prompts too
    B = len(samples)
    sampling = E.Sampling([0.8] * B, [0.9] * B, [40] * B, [11 + b for b in range(B)])
    _check(pipe, samples, "sampled, scored", 1, sampling=sampling, scored=True)
    _check(pipe, samples, "sampled, streamed", 1, sampling=sampling, stream=True)


def test_two_groups_and_loners_interleaved(pipe):
    a, b = _sample(*BASE), _sample(160, 168, 5)
    samples = [_ask(a, _prompt(a, 0)), _sample(170, 56, 1), _ask(b, _prompt(b, 1)), _ask(a, _prompt(a, 2)), _sample(171, 112, 2),
               _ask(b, _prompt(b, 3)), _ask(a, _prompt(a, 4))]
    _check(pipe, samples, "two groups and loners", 1)


@pytest.mark.parametrize("residue", [0, 1, 63])
def test_prefix_length_at_key_tile_edges(pipe, residue):
    base = _sample(*BASE)
    fill = _fill_for(base, residue)
    samples = [_ask(base, _prompt(base, q, fill)) for q in range(3)]
    _check(pipe, samples, f"P mod 64 = {residue}", 1, alone=True)


def test_group_sharing_only_the_towers(pipe):
    base = _sample(*BASE)
    samples = [_ask(base, _prompt(base, q, head=9000 + q)) for q in range(3)]
    P = import_module("vlm-fo1_b200.pipeline")
    assert P.shared_prefix_groups([s.input_ids for s in samples], [0, 0, 0], [16] * 3, [100] * 3) == []
    _check(pipe, samples, "towers only", 1, alone=True)


# ------------------------------------------------------------------------------------------------------- 3. towers once
def test_towers_run_once_per_unique_image(pipe, monkeypatch):
    seen = {"vit": 0, "davit": 0}
    eng = pipe.eng
    vit, davit = eng.vit_forward, eng.davit_forward

    def count_vit(px, grids):
        seen["vit"] += len(px)
        return vit(px, grids)

    def count_davit(images):
        seen["davit"] += len(images)
        return davit(images)
    monkeypatch.setattr(eng, "vit_forward", count_vit)
    monkeypatch.setattr(eng, "davit_forward", count_davit)
    a, b = _sample(*BASE), _sample(160, 168, 5)
    samples = [_ask(a, _prompt(a, q)) for q in range(5)] + [_ask(b, _prompt(b, q)) for q in range(3)] + [_sample(170, 56, 1)]
    _run(pipe, samples, True)
    assert seen == {"vit": 3, "davit": 3}
    seen.update(vit=0, davit=0)
    _run(pipe, samples, False)
    assert seen == {"vit": 9, "davit": 9}


# ------------------------------------------------------------------------------------------------------- 4. num_return_sequences
def test_num_return_sequences(fab):
    _, model, kw = fab
    n = 4
    a = dict(kw(0, temperature=0.7, top_p=0.9), streamer=None)      # prepare_inputs attaches a TextStreamer, which takes one sequence
    P = a["inputs"].shape[1]
    torch.manual_seed(5)
    got = model.generate(**a, num_return_sequences=n)
    torch.manual_seed(5)
    ref = model.generate_batch([a] * n)
    pad = model.default_stop_ids[0]
    T = max(r.shape[1] for r in ref) - P
    assert got.shape == (n, P + T)
    for i, r in enumerate(ref):
        m = r.shape[1]
        assert torch.equal(got[i, :m], r[0]), i
        assert bool((got[i, m:] == pad).all()), i
    torch.manual_seed(5)
    d = model.generate(**a, num_return_sequences=n, return_dict_in_generate=True, output_scores=True, output_logits=True)
    assert torch.equal(d.sequences, got)
    assert len(d.scores) == len(d.logits) == T and all(s.shape[0] == n for s in d.scores + d.logits)
    with pytest.raises(ValueError, match="num_return_sequences"):
        model.generate(**kw(0, temperature=0.0, top_p=0.05), num_return_sequences=2)
    with pytest.raises(ValueError, match="streamer"):
        model.generate(**kw(0, temperature=0.7, top_p=0.9), num_return_sequences=2)
