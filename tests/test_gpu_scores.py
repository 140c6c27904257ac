"""-m gpu: per-token scoring (csrc/sampling.cuh score_row) -- the row routine through fo1_score_rows against the CPU oracle
(tests/scores_oracle.py over oracle/sampling.py), both decode paths of the engine (the persistent kernel and FO1_NO_MEGA=1's per-kernel graph), and the model's
generate surface (return_dict_in_generate, output_scores / output_logits, compute_transition_scores, output_logprobs)."""
import gzip
import json
import os

import numpy as np
import pytest
import torch

from oracle import sampling as S
from tests import scores_oracle as SO
from tests.test_gpu_decode_mega import _batch, _engine
from tests.test_gpu_sampling import _rows

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARGIN = 1e-6      # of Z: a top-p cut closer than this to a cumulative boundary is left undecided (as test_gpu_sampling)
LP_TOL = 2e-5      # fp32 rounding bound of a log-probability: fp32 exp, 2^-40 fixed-point weights, fp32 result


def _eng_mod():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine")


def _div(row, T):
    """row / T on the device as an IEEE fp32 division (a Python scalar divisor would be turned into a multiply)."""
    return row / torch.full_like(row, T) if T != 1.0 else row


@pytest.mark.parametrize("V", [151936, 32000])
def test_score_rows_matches_oracle(V):
    E = _eng_mod()
    rng = np.random.default_rng(V + 1)
    rows = _rows(V, rng)
    hole = rng.normal(0, 2.0, V).astype(np.float32)
    hole[rng.choice(V, V // 10, replace=False)] = -np.inf                     # rows with -inf entries
    rows.append(hole)
    combos = [(k, p) for k in (0, 1, 50, 1000, V) for p in (0.05, 0.9, 1.0)]
    checked = 0
    for ri, row in enumerate(rows):
        dev_row = torch.from_numpy(row).cuda()
        for T in (0.1, 0.7, 1.0, 1.5):
            plans = []
            for k, p in combos:
                x, order, kept, _, margin_p = S.warp(row, T, p, k)
                kept_idx = order[kept[order]]                                # kept tokens, canonical order
                toks = [int(kept_idx[0]), int(kept_idx[-1]), int(kept_idx[rng.integers(kept_idx.size)])]
                cut = np.nonzero(~kept)[0]
                if cut.size:
                    toks.append(int(cut[rng.integers(cut.size)]))
                plans.append((k, p, x, kept, margin_p, toks))
            n = sum(len(pl[5]) for pl in plans)
            lg = dev_row.view(1, -1).expand(n, -1).contiguous()
            Ts, Ps, Ks, tok = [], [], [], []
            for k, p, _, _, _, toks in plans:
                Ts += [T] * len(toks); Ps += [p] * len(toks); Ks += [k] * len(toks); tok += toks
            lp, sc = E.score_rows(lg, torch.tensor(tok, dtype=torch.int32), Ts, Ps, Ks, want_scores=True)
            lp, sc = lp.cpu().numpy(), sc
            x_dev = _div(dev_row, T).cpu().numpy()
            j = 0
            for k, p, x, kept, margin_p, toks in plans:
                fin = torch.isfinite(sc[j]).cpu().numpy()
                if margin_p > MARGIN:
                    checked += 1
                    assert np.array_equal(fin, kept & np.isfinite(x)), (V, ri, T, k, p)      # a kept -inf logit stays -inf
                    got = sc[j].cpu().numpy()
                    assert np.array_equal(got[fin].view(np.uint32), x_dev[fin].view(np.uint32)), (V, ri, T, k, p)
                    for i, t in enumerate(toks):
                        ref = SO.logprob_from(x, kept, t)
                        if ref == -np.inf:
                            assert lp[j + i] == -np.inf, (V, ri, T, k, p, t, lp[j + i])
                        else:
                            assert abs(lp[j + i] - ref) <= LP_TOL, (V, ri, T, k, p, t, lp[j + i], ref)
                j += len(toks)
    assert checked >= 0.5 * len(rows) * 4 * len(combos), checked
    # raw rows: the logits unchanged, log-probabilities over the whole row (T = 1), whatever the row's sampling parameters
    dev = torch.from_numpy(np.stack(rows)).cuda()
    n = dev.shape[0]
    tok = [int(np.argmax(r)) if i % 2 else int(rng.integers(V)) for i, r in enumerate(rows)]
    for kw in (dict(), dict(temperature=[0.7] * n, top_p=[0.5] * n, top_k=[5] * n, raw_rows=[1] * n)):
        lp, sc = E.score_rows(dev, torch.tensor(tok, dtype=torch.int32), want_scores=True, **kw)
        assert torch.equal(sc, dev)
        for i, r in enumerate(rows):
            ref = SO.logprob(r, 1.0, 1.0, 0, tok[i], raw=True)
            assert abs(float(lp[i]) - ref) <= LP_TOL or (ref == -np.inf and float(lp[i]) == -np.inf), (i, float(lp[i]), ref)


# ---------------------------------------------------------------------------------------------------------- decode paths
@pytest.fixture(scope="module")
def engine():
    return _engine()


def _gen(eng, emb, pos, lens, deltas, T, sampling, stop_ids, scored, raw_rows=None):
    kw = dict(want_logprobs=True, want_scores=True, want_logits=True, want_prefill_logits=True, raw_rows=raw_rows) if scored else {}
    return eng.generate(emb, pos, lens, deltas, T, stop_ids=list(stop_ids), pad_id=0, early_exit_interval=2, sampling=sampling, **kw)


def _check_rows(out, lens_out, params, raw):
    """Per (sequence, column): scores / logits / logprobs against the contract."""
    toks, lp, sc, lg = out["tokens"].cpu(), out["logprobs"], out["scores"], out["logits"]
    assert torch.equal(lg[0], out["prefill_logits"])                         # column 0 is the prefill's last-position row
    for b, n in enumerate(lens_out):
        assert torch.all(lp[b, n:] == 0), b                                  # 0 past out_lens
        for t in range(n):
            tok = int(toks[b, t])
            if raw[b]:
                assert torch.equal(sc[t, b], lg[t, b]), (b, t)
                assert int(torch.argmax(lg[t, b])) == tok, (b, t)            # the row of this step and slot
            else:
                T, p, k = params[b]
                x = _div(lg[t, b], T)
                fin = torch.isfinite(sc[t, b])
                assert torch.equal(sc[t, b][fin], x[fin]) and bool(fin[tok]), (b, t)
                _, _, kept, _, margin_p = S.warp(lg[t, b].cpu().numpy(), T, p, k)
                if margin_p > MARGIN:
                    assert np.array_equal(fin.cpu().numpy(), kept), (b, t)
            ref = float(torch.log_softmax(sc[t, b].double(), -1)[tok])
            assert abs(float(lp[b, t]) - ref) <= LP_TOL, (b, t, float(lp[b, t]), ref)


@pytest.mark.parametrize("B,no_mega", [(1, False), (5, False), (20, False), (1, True), (5, True), (20, True), (40, True)])
@pytest.mark.parametrize("sampled", [False, True])
def test_decode_paths_scored(engine, B, no_mega, sampled, monkeypatch):
    eng, _ = engine
    E = _eng_mod()
    monkeypatch.setenv("FO1_MEGA_MAX_B", "32")
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [41 + 37 * (b % 5) for b in range(B)]
    emb, pos, deltas = _batch(lens, seed=100 + B)
    T = 10
    params = [(0.7, 0.9, 50)] * B
    samp = E.Sampling([0.7] * B, [0.9] * B, [50] * B, [500 + b for b in range(B)]) if sampled else None
    free = _gen(eng, emb, pos, lens, deltas, T, samp, [], False)
    stop = int(free["tokens"][0, 3])                                         # sequences end at different columns
    base = _gen(eng, emb, pos, lens, deltas, T, samp, [stop], False)
    out = _gen(eng, emb, pos, lens, deltas, T, samp, [stop], True)
    assert eng.last_decode_path() == (0 if no_mega or B > 32 else 1)
    assert torch.equal(base["tokens"], out["tokens"]) and torch.equal(base["lens"], out["lens"])
    lens_out = out["lens"].cpu().tolist()
    assert min(lens_out) < T
    _check_rows(out, lens_out, params, [not sampled] * B)


@pytest.mark.parametrize("no_mega", [False, True])
def test_mixed_batch_raw_and_topk1_rows(engine, no_mega, monkeypatch):
    """A raw (greedy) row scores its logits; a top_k = 1 sampled row keeps every maximum: logprob 0, or -ln(ties)."""
    eng, _ = engine
    E = _eng_mod()
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [120, 77, 200, 64]
    emb, pos, deltas = _batch(lens, seed=8)
    params = [(0.7, 0.9, 50), (1.0, 1.0, 1), (0.7, 1.0, 1), (1.5, 0.5, 0)]
    raw = [0, 1, 0, 0]
    samp = E.Sampling([p[0] for p in params], [p[1] for p in params], [p[2] for p in params], [1, 2, 3, 4])
    T = 10
    base = _gen(eng, emb, pos, lens, deltas, T, samp, [], False)
    out = _gen(eng, emb, pos, lens, deltas, T, samp, [], True, raw_rows=raw)
    assert torch.equal(base["tokens"], out["tokens"])
    _check_rows(out, [T] * 4, params, raw)
    for t in range(T):
        x = _div(out["logits"][t, 2], 0.7)
        ties = int((x == x.max()).sum())
        assert abs(float(out["logprobs"][2, t]) + np.log(ties)) <= LP_TOL, (t, ties)


# ---------------------------------------------------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def fab(tmp_path_factory):
    from importlib import import_module
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    E = _eng_mod(); FB = import_module("vlm-fo1_b200.fabricate")
    root = tmp_path_factory.mktemp("scores")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(root / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(REPO, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    tokenizer, model, procs = load_pretrained_model(model_path, device="cuda:0")
    sizes = {im["file_name"]: (im["width"], im["height"]) for im in fx["instances"]["images"]}
    src = ImageSource(str(root / "none"), str(root / "synth"))
    msgs = []
    for d in fx["coco"][:3]:
        msgs.append([{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                                  {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}])

    def kw(i, **k):
        return prepare_inputs(model_path, model, procs, tokenizer, msgs[i], device="cuda:0", max_tokens=10, **k)
    return model, kw


@pytest.mark.parametrize("sampled", [False, True])
def test_generate_return_dict(fab, sampled):
    model, kw = fab
    a = kw(0, temperature=0.7 if sampled else 0.0, top_p=0.9)
    assert a["do_sample"] is sampled
    torch.manual_seed(4)
    plain = model.generate(**a)
    torch.manual_seed(4)
    out = model.generate(**a, return_dict_in_generate=True, output_scores=True, output_logits=True)
    assert torch.equal(out.sequences, plain)
    n = plain.shape[1] - a["inputs"].shape[1]
    assert len(out.scores) == n and len(out.logits) == n and out.scores[0].shape == out.logits[0].shape and out.scores[0].shape[0] == 1
    assert out.past_key_values is None and out.attentions is None and out.hidden_states is None
    if not sampled:
        assert all(torch.equal(s, l) for s, l in zip(out.scores, out.logits))
    ts = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=True)
    torch.manual_seed(4)
    (seq, lp), = model.generate_batch([a], output_logprobs=True)
    assert torch.equal(seq, plain) and lp.shape == (1, n)
    assert torch.allclose(lp, ts.float(), atol=LP_TOL, rtol=0), (lp, ts)
    # only the dict carries scores: without return_dict_in_generate nothing changes
    torch.manual_seed(4)
    t = model.generate(**a, output_scores=True, return_dict_in_generate=False)
    assert isinstance(t, torch.Tensor) and torch.equal(t, plain)


def test_generate_outputs_contract(fab):
    model, kw = fab
    a = kw(1, temperature=0.0, top_p=0.9)
    for field in ("output_attentions", "output_hidden_states"):
        with pytest.raises(NotImplementedError, match=field):
            model.generate(**a, return_dict_in_generate=True, **{field: True})
    plain = model.generate(**a)
    gc = dict(model.generation_config)
    try:       # generation_config.json's fields apply as in HF; the call's kwargs win
        model.generation_config.update(return_dict_in_generate=True, output_scores=True)
        out = model.generate(**a)
        assert torch.equal(out.sequences, plain) and len(out.scores) == plain.shape[1] - a["inputs"].shape[1] and out.logits is None
        assert isinstance(model.generate(**a, return_dict_in_generate=False), torch.Tensor)
    finally:
        model.generation_config.clear()
        model.generation_config.update(gc)


def test_generate_batch_per_dict_outputs(fab):
    """Element b is what generate(**batch[b]) returns, a greedy sample in a sampled batch scored on its raw logits."""
    model, kw = fab
    kws = [dict(kw(0, temperature=0.7, top_p=0.9), return_dict_in_generate=True, output_scores=True), kw(1, temperature=0.7, top_p=0.9),
           dict(kw(2, temperature=0.0, top_p=0.9), return_dict_in_generate=True, output_scores=True, output_logits=True)]
    torch.manual_seed(6)
    res = model.generate_batch(kws, output_logprobs=True)
    (d0, lp0), (t1, lp1), (d2, lp2) = res
    assert isinstance(t1, torch.Tensor) and d0.logits is None and d2.logits is not None
    assert all(torch.equal(s, l) for s, l in zip(d2.scores, d2.logits))        # the raw row: scores are its logits
    for d, lp in ((d0, lp0), (d2, lp2)):
        ts = model.compute_transition_scores(d.sequences, d.scores, normalize_logits=True)
        assert torch.allclose(lp, ts.float(), atol=LP_TOL, rtol=0)
