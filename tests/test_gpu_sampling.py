"""-m gpu: sampled decoding (csrc/sampling.cuh) -- the standalone kernel against the CPU oracle (oracle/sampling.py), both decode
paths of the engine (the persistent kernel and FO1_NO_MEGA=1's per-kernel graph) and the model's generate surface."""
import gzip
import json
import os

import numpy as np
import pytest
import torch

from oracle import sampling as S
from tests.test_gpu_decode_mega import NEAR_TIE, _batch, _engine

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# of Z: a draw closer than this to a cumulative boundary is left undecided.  The kernel's cumulative weights differ from the oracle's
# float64 ones by the fp32 exp (a few 1e-7 relative) and the 2^-40 fixed-point rounding of each weight: well under 1e-6 of Z.
MARGIN = 1e-6


def _eng_mod():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine")


def _rows(V, rng):
    rows = [rng.normal(0, s, V).astype(np.float32) for s in (0.5, 2.0, 6.0)]
    tie = np.round(rng.normal(0, 2.0, V) * 2).astype(np.float32) / 2          # a few dozen values shared by thousands of tokens
    dom = rng.normal(0, 1.0, V).astype(np.float32)
    dom[int(rng.integers(V))] = 30.0                                           # one dominant token
    return rows + [tie, dom]


class _Oracle:
    """The oracle's kept set and cumulative weights of one (row, T, p, k), then any number of draws."""

    def __init__(self, row, T, p, k):
        self.k1 = k == 1
        x, self.order, kept, probs, self.margin_p = S.warp(row, T, p, k)
        self.argmax = int(np.argmax(x))
        w = probs[self.order]
        self.live = w > 0
        self.incl = np.cumsum(w)

    def draw(self, seed, step):
        if self.k1:
            return self.argmax, np.inf
        Z = self.incl[-1]
        t = S.uniform(seed, step) * Z
        pos = int(np.searchsorted(self.incl, t, side="right"))
        bounds = np.concatenate([[0.0], self.incl[self.live]])
        return int(self.order[min(pos, self.order.size - 1)]), min(float(np.min(np.abs(bounds - t)) / Z), self.margin_p)


@pytest.mark.parametrize("V", [151936, 32000])
def test_kernel_matches_oracle(V):
    E = _eng_mod()
    rng = np.random.default_rng(V)
    n_draw = 6
    checked = undecided = 0
    bounded = bounded_undecided = 0     # draws among at most 1000 candidates (top-k 1, 50, 1000)
    for ri, row in enumerate(_rows(V, rng)):
        dev = torch.from_numpy(row).cuda().view(1, -1).expand(n_draw, -1).contiguous()
        for T in (0.1, 0.7, 1.0, 1.5):
            for k in (0, 1, 50, 1000, V):
                for p in (0.05, 0.5, 0.9, 1.0):
                    seeds = [int(rng.integers(0, 2 ** 63)) for _ in range(n_draw)]
                    steps = torch.tensor([int(rng.integers(0, 4096)) for _ in range(n_draw)], dtype=torch.int32)
                    got = E.sample_tokens(dev, [T] * n_draw, [p] * n_draw, [k] * n_draw, seeds, steps.cuda()).cpu().tolist()
                    orc = _Oracle(row, T, p, k)
                    for j in range(n_draw):
                        tok, margin = orc.draw(seeds[j], int(steps[j]))
                        if k == 1:
                            assert got[j] == tok, (ri, T, k, p)                # k = 1 is the arg-max, bit for bit
                        if 1 <= k <= 1000:
                            bounded += 1
                            bounded_undecided += int(margin <= MARGIN)
                        if margin > MARGIN:
                            checked += 1
                            assert got[j] == tok, (V, ri, T, k, p, j, got[j], tok, margin)
                        else:
                            undecided += 1
    # Over all 151936 tokens of a flat row (small spread, high temperature, no top-k) the cumulative boundaries lie a few 1e-6 of Z
    # apart, so many of those draws are undecidable by construction; among at most 1000 candidates almost none may be.
    assert bounded_undecided < 0.01 * bounded, (bounded_undecided, bounded)
    assert checked >= 0.5 * (checked + undecided), (undecided, checked)


def test_kernel_reproducible_and_row_independent():
    E = _eng_mod()
    rng = np.random.default_rng(9)
    V = 151936
    rows = torch.from_numpy(np.stack(_rows(V, rng))).cuda()
    n = rows.shape[0]
    args = ([0.7] * n, [0.9] * n, [50] * n, list(range(11, 11 + n)))
    a = E.sample_tokens(rows, *args, step=5)
    b = E.sample_tokens(rows, *args, step=5)
    assert torch.equal(a, b)
    for i in range(n):                                                   # alone, and as the last row of a launch of two
        one = E.sample_tokens(rows[i:i + 1], [0.7], [0.9], [50], [11 + i], step=5)
        two = E.sample_tokens(rows[[0, i]], [0.7] * 2, [0.9] * 2, [50] * 2, [11, 11 + i], step=5)
        assert int(one[0]) == int(a[i]) == int(two[1])


def _gen(eng, emb, pos, lens, deltas, T, sampling, stop_ids=(), pad_id=0, interval=0):
    return eng.generate(emb, pos, lens, deltas, T, stop_ids=list(stop_ids), pad_id=pad_id, early_exit_interval=interval, sampling=sampling)


def _samp(E, B, T=1.0, p=1.0, k=0, seeds=None):
    return E.Sampling([T] * B, [p] * B, [k] * B, list(seeds) if seeds is not None else [100 + b for b in range(B)])


@pytest.fixture(scope="module")
def engine():
    return _engine()


@pytest.mark.parametrize("B,no_mega", [(5, False), (20, False), (5, True), (40, False)])
def test_engine_topk1_is_greedy_and_reproducible(engine, B, no_mega, monkeypatch):
    eng, _ = engine
    E = _eng_mod()
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [37 + 29 * (b % 7) for b in range(B)]
    emb, pos, deltas = _batch(lens, seed=B)
    T = 12
    greedy = _gen(eng, emb, pos, lens, deltas, T, None)
    k1 = _gen(eng, emb, pos, lens, deltas, T, _samp(E, B, T=0.7, p=0.9, k=1))
    assert eng.last_decode_path() == (0 if no_mega or B > 32 else 1)
    assert torch.equal(greedy["tokens"], k1["tokens"])
    s1 = _gen(eng, emb, pos, lens, deltas, T, _samp(E, B, T=1.0, p=0.95, k=50))
    s2 = _gen(eng, emb, pos, lens, deltas, T, _samp(E, B, T=1.0, p=0.95, k=50))
    assert torch.equal(s1["tokens"], s2["tokens"]) and torch.equal(s1["lens"], s2["lens"])
    assert not torch.equal(s1["tokens"], greedy["tokens"])


@pytest.mark.parametrize("no_mega", [False, True])
def test_engine_slots_seeds_batch_size_and_stop_ids(engine, no_mega, monkeypatch):
    eng, _ = engine
    E = _eng_mod()
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [200, 333, 200, 91]
    emb, pos, deltas = _batch(lens, seed=3)
    emb[533:733] = emb[0:200]                                          # sequence 2 == sequence 0
    T = 12
    same = _gen(eng, emb, pos, lens, deltas, T, _samp(E, 4, seeds=[7, 8, 7, 9]))["tokens"].cpu()
    assert torch.equal(same[0], same[2])
    diff = _gen(eng, emb, pos, lens, deltas, T, _samp(E, 4, seeds=[7, 8, 6, 9]))["tokens"].cpu()
    assert not torch.equal(diff[0], diff[2])
    assert torch.equal(diff[0], same[0])                               # a row depends on its own seed only
    one = _gen(eng, emb[:200], pos[:, :200].contiguous(), [200], [0], T, _samp(E, 1, seeds=[7]))["tokens"].cpu()
    assert torch.equal(one[0], same[0])                                # B = 1 against B = 4
    stop = int(same[1, 3])
    out2 = _gen(eng, emb, pos, lens, deltas, T, _samp(E, 4, seeds=[7, 8, 7, 9]), stop_ids=[stop], pad_id=7, interval=2)
    t2, l2 = out2["tokens"].cpu(), out2["lens"].cpu().tolist()
    for i in range(4):
        row = same[i].tolist()
        n = row.index(stop) + 1 if stop in row else T
        assert l2[i] == n and t2[i].tolist() == row[:n] + [7] * (T - n), (i, l2, t2[i].tolist(), row)


@pytest.mark.parametrize("no_mega", [False, True])
def test_engine_steps_and_seeds_teacher_forced(engine, no_mega, monkeypatch):
    """Every sampled token is the oracle's draw (same seed, step = output column) on the logits of its prefix re-scored through the
    prefill, wherever the draw is decidable: its margin exceeds the logit error between the decode step and the prefill, taken as
    the larger of 6 sigma of the difference measured between two prefills and NEAR_TIE of the logits' spread (the bound
    test_gpu_decode_mega.py establishes for two summation orders of the same bf16 data)."""
    eng, sd = engine
    E = _eng_mod()
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [150, 260]
    emb, pos, deltas = _batch(lens, seed=11)
    T, Tmp, k, seeds = 16, 1.0, 3, [12345, 2 ** 40 + 3]
    out = _gen(eng, emb, pos, lens, deltas, T, E.Sampling([Tmp] * 2, [1.0] * 2, [k] * 2, seeds))["tokens"].cpu()
    table = sd["embed_tokens.weight"]
    starts = [0, lens[0], lens[0] + lens[1]]
    decided = 0
    for i in range(2):
        full = torch.cat([emb[starts[i]:starts[i + 1]], table[out[i, :T - 1].long().cuda()].to(torch.bfloat16)])
        n = full.shape[0]
        fpos = torch.arange(n, dtype=torch.int32).view(1, -1).expand(3, -1).contiguous()
        all_lg = eng.generate(full, fpos, [n], [0], 0, stop_ids=[], pad_id=0, want_all_logits=True, early_exit_interval=0)["all_logits"].cpu()
        for t in range(T):
            P = lens[i] + t
            ppos = torch.arange(P, dtype=torch.int32).view(1, -1).expand(3, -1).contiguous()
            lg = eng.generate(full[:P].contiguous(), ppos, [P], [0], 1, stop_ids=[], pad_id=0, want_prefill_logits=True,
                              early_exit_interval=0)["prefill_logits"][0].cpu()
            # logit error: the same position scored by two prefills of different lengths, and the decode / prefill bound
            err = max(6 * float((lg - all_lg[P - 1]).float().std()), NEAR_TIE * float(lg.std()))
            row = lg.numpy().astype(np.float32)
            tok, margin = _Oracle(row, Tmp, 1.0, k).draw(seeds[i], t)
            top = np.sort(row)[::-1]
            # decidable: the top-k set is not a near-tie (k-th against (k+1)-th logit) and the draw clears twice the error
            # (a logit error e moves a weight by a factor exp(+-e / T))
            if top[k - 1] - top[k] > 2 * err and margin > 2 * err / Tmp:
                decided += 1
                assert int(out[i, t]) == tok, (i, t, int(out[i, t]), tok, margin, err)
    assert decided >= 8, decided


# ---------------------------------------------------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def fab(tmp_path_factory):
    from importlib import import_module
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    E = _eng_mod(); FB = import_module("vlm-fo1_b200.fabricate")
    root = tmp_path_factory.mktemp("samp")
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
    for d in fx["coco"][:6]:
        msgs.append([{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                                  {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}])

    def kw(i, **k):
        return prepare_inputs(model_path, model, procs, tokenizer, msgs[i], device="cuda:0", max_tokens=10, **k)
    return model_path, model, kw


def test_generate_sampled_reproducible(fab):
    _, model, kw = fab
    a = kw(0, temperature=0.7, top_p=0.9)
    assert a["do_sample"] is True
    torch.manual_seed(3)
    x = model.generate(**a)
    torch.manual_seed(3)
    y = model.generate(**a)
    P = a["inputs"].shape[1]
    assert x.dim() == 2 and x.shape[0] == 1 and x.shape[1] > P and torch.equal(x[0, :P].cpu(), a["inputs"][0].cpu())
    assert torch.equal(x, y)


def test_generate_batch_sampled_equals_one_by_one(fab):
    _, model, kw = fab
    kws = [kw(i, temperature=0.7, top_p=0.9) for i in range(5)] + [kw(5, temperature=0.0, top_p=0.05)]     # one greedy sample too
    torch.manual_seed(21)
    batch = model.generate_batch(kws)
    torch.manual_seed(21)
    ones = [model.generate(**k) for k in kws]
    for i, (k, one, got) in enumerate(zip(kws, ones, batch)):
        P = k["inputs"].shape[1]
        assert one.shape[1] > P
        assert one.shape == got.shape and torch.equal(one, got), (i, one[0, P:].tolist(), got[0, P:].tolist())


def test_generate_argument_contract(fab, tmp_path):
    model_path, model, kw = fab
    a = kw(0, temperature=0.0, top_p=0.05)
    with pytest.raises(ValueError):
        model.generate(**dict(a, do_sample=True, temperature=0.0))
    # the reference callers' greedy kwargs: exactly the greedy pipeline's output
    assert a["do_sample"] is False
    got = model.generate(**a)
    s, stop, samp = model._sample(**{k: v for k, v in a.items() if k in ("inputs", "images", "images_aux", "image_grid_thws", "bbox_list")})
    ref = model.pipeline.generate([s], 10, sorted(set(stop)), pad_id=stop[0], early_exit_interval=8)
    n = int(ref["lens"][0])
    assert samp is None and torch.equal(got[0, a["inputs"].shape[1]:].cpu(), ref["tokens"][0, :n].long().cpu())
    # a processor the engine does not implement is refused on the sampled path only
    gc = dict(model.generation_config)
    try:
        model.generation_config["repetition_penalty"] = 1.05
        with pytest.raises(NotImplementedError, match="repetition_penalty"):
            model.generate(**kw(0, temperature=0.7, top_p=0.9))
        assert torch.equal(model.generate(**a), got)
    finally:
        model.generation_config.clear()
        model.generation_config.update(gc)


def test_generation_config_file_is_read(fab, tmp_path):
    import shutil
    from vlm_fo1.model.builder import load_pretrained_model
    model_path, _, _ = fab
    dst = tmp_path / os.path.basename(model_path)
    shutil.copytree(model_path, dst)
    gp = dst / "generation_config.json"
    gc = json.load(open(gp)) if gp.exists() else {}
    gc.update(repetition_penalty=1.05, top_k=7)
    json.dump(gc, open(gp, "w"))
    _, model, _ = load_pretrained_model(str(dst), device="cuda:0")           # loading never refuses
    assert model.generation_config["repetition_penalty"] == 1.05
    with pytest.raises(NotImplementedError):
        model._sampling_params(0.7, 0.9, None, {})
    model.generation_config.pop("repetition_penalty")
    assert model._sampling_params(0.7, 0.9, None, {}) == (0.7, pytest.approx(0.9), 7)
