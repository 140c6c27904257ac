"""-m gpu: streamed decoding (include/fo1.h, fo1_stream_desc) -- both decode paths publish every output column into pinned host
memory while the loop stays on the device: the published columns equal the outputs, streaming changes no token / score / logit,
the host really sees columns while the device decodes, a cancel stops every sequence after the column recorded next, callback
errors stop the device and propagate, and the HF streamer surface of Fo1ForCausalLM.generate follows HF's put / end order."""
import gzip
import json
import os
import threading

import numpy as np
import pytest
import torch

from tests.test_gpu_decode_mega import _batch, _engine

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mods():
    from importlib import import_module
    import fo1_b200
    return fo1_b200._lib, import_module("vlm-fo1_b200.engine")


@pytest.fixture(scope="module")
def engine():
    return _engine()


class Recorder:
    """on_tokens that keeps every call; ``cancel_at``: return True once that many columns are visible; ``raise_at``: raise this
    exception instead once that many columns are visible."""

    def __init__(self, eng, cancel_at=None, raise_at=None, exc=None):
        self.eng, self.cancel_at, self.raise_at, self.exc = eng, cancel_at, raise_at, exc
        self.calls = []

    def __call__(self, lo, hi, toks, lens):
        F, _ = _mods()
        done_now = bool(int(self.eng._stream_buf[2][0]) & F.FO1_STREAM_DONE)
        assert toks.dtype == np.int32 and lens.dtype == np.int32 and toks.shape == (lens.shape[0], hi - lo)
        self.calls.append((lo, hi, toks, lens.copy(), done_now))
        if self.raise_at is not None and hi >= self.raise_at:
            raise self.exc
        return self.cancel_at is not None and hi >= self.cancel_at

    def check_published(self, out):
        """Chunks are contiguous and non-empty; concatenated they equal out_tokens up to the last column published, the final lens
        equal out_lens, and the final progress is done | max(out_lens)."""
        F, _ = _mods()
        assert self.calls and self.calls[0][0] == 0
        for (_, hi0, *_), (lo1, hi1, *_) in zip(self.calls, self.calls[1:]):
            assert lo1 == hi0 and hi1 > lo1
        toks = np.concatenate([c[2] for c in self.calls], axis=1)
        lens = out["lens"].cpu().numpy()
        hi = self.calls[-1][1]
        assert hi == lens.max()
        assert np.array_equal(toks, out["tokens"][:, :hi].cpu().numpy())
        for b, n in enumerate(lens):
            assert np.array_equal(toks[b, :n], out["tokens"][b, :n].cpu().numpy())
        assert np.array_equal(self.calls[-1][3], lens)
        assert int(self.eng._stream_buf[2][0]) == F.FO1_STREAM_DONE | int(lens.max())


def _gen(eng, x, T, samp=None, stop=(), scored=False, on_tokens=None):
    emb, pos, lens, deltas = x
    kw = dict(want_logprobs=True, want_scores=True, want_logits=True, want_prefill_logits=True) if scored else {}
    return eng.generate(emb, pos, lens, deltas, T, stop_ids=list(stop), pad_id=0, early_exit_interval=2, sampling=samp, on_tokens=on_tokens, **kw)


def _inputs(B, seed):
    lens = [41 + 37 * (b % 5) for b in range(B)]
    emb, pos, deltas = _batch(lens, seed=seed)
    return emb, pos, lens, deltas


@pytest.mark.parametrize("B,no_mega", [(1, False), (5, False), (20, False), (5, True), (40, True)])
@pytest.mark.parametrize("mode", ["greedy", "sampled", "scored"])
def test_streamed_equals_unstreamed(engine, B, no_mega, mode, monkeypatch):
    eng, _ = engine
    _, E = _mods()
    monkeypatch.setenv("FO1_MEGA_MAX_B", "32")
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    x = _inputs(B, 300 + B)
    T = 12
    samp = E.Sampling([0.7] * B, [0.9] * B, [50] * B, [700 + b for b in range(B)]) if mode == "sampled" else None
    scored = mode == "scored"
    free = _gen(eng, x, T, samp)
    for stop in ([], [int(free["tokens"][0, 3])]):                       # no stop id; a stop id that ends sequence 0 mid-run
        base = _gen(eng, x, T, samp, stop, scored)
        rec = Recorder(eng)
        out = _gen(eng, x, T, samp, stop, scored, on_tokens=rec)
        assert eng.last_decode_path() == (0 if no_mega or B > 32 else 1)
        for k in ("tokens", "lens") + (("logprobs", "prefill_logits") if scored else ()):
            assert torch.equal(base[k], out[k]), k
        if scored:                                                         # rows past a sequence's stop are unspecified
            for b, n in enumerate(out["lens"].cpu().tolist()):
                assert torch.equal(base["scores"][:n, b], out["scores"][:n, b]) and torch.equal(base["logits"][:n, b], out["logits"][:n, b])
        rec.check_published(out)
        if stop:
            assert int(out["lens"][0]) <= 4


@pytest.mark.parametrize("no_mega", [False, True])
def test_columns_arrive_while_decoding(engine, no_mega, monkeypatch):
    eng, _ = engine
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    x = _inputs(2, 11)
    rec = Recorder(eng)
    out = eng.generate(*x, 1024, stop_ids=[], pad_id=0, early_exit_interval=8, on_tokens=rec)
    assert eng.last_decode_path() == (0 if no_mega else 1)
    assert len(rec.calls) >= 2
    assert not rec.calls[0][4] and rec.calls[0][1] < 1024                 # the first call came while the device was decoding
    rec.check_published(out)


@pytest.mark.parametrize("no_mega", [False, True])
def test_cancel_cuts_every_sequence(engine, no_mega, monkeypatch):
    eng, _ = engine
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    x = _inputs(3, 12)
    T = 2048
    base = eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8)
    rec = Recorder(eng, cancel_at=8)
    out = eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8, on_tokens=rec)
    lens = out["lens"].cpu().tolist()
    L = lens[0]
    assert all(n == L for n in lens) and 8 <= L < T, lens
    assert torch.equal(out["tokens"][:, :L], base["tokens"][:, :L])
    assert bool((out["tokens"][:, L:] == 0).all())
    rec.check_published(out)
    again = eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8)
    assert torch.equal(again["tokens"], base["tokens"]) and torch.equal(again["lens"], base["lens"])


@pytest.mark.parametrize("exc", [ValueError("callback failed"), KeyboardInterrupt()])
@pytest.mark.parametrize("no_mega", [False, True])
def test_callback_error_stops_and_propagates(engine, exc, no_mega, monkeypatch):
    eng, _ = engine
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    x = _inputs(2, 13)
    T = 512
    base = eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8)
    threads = threading.active_count()
    with pytest.raises(type(exc)) as info:
        eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8, on_tokens=Recorder(eng, raise_at=4, exc=exc))
    assert info.value is exc
    assert threading.active_count() == threads
    again = eng.generate(*x, T, stop_ids=[], pad_id=0, early_exit_interval=8)
    assert torch.equal(again["tokens"], base["tokens"]) and torch.equal(again["lens"], base["lens"])


def test_pageable_buffers_are_refused_without_launch(engine, monkeypatch):
    eng, _ = engine
    F, _ = _mods()
    import fo1_b200
    x = _inputs(2, 14)
    # ordinary (pageable) host tensors in place of the pinned buffers
    monkeypatch.setattr(eng, "_stream_buffers", lambda B, T: (torch.zeros(B * T, dtype=torch.int32), torch.zeros(B, dtype=torch.int32),
                                                               torch.zeros(32, dtype=torch.int32)))
    torch.cuda.synchronize()
    n0 = fo1_b200.lib().fo1_launch_count()
    threads = threading.active_count()
    with pytest.raises(F.Fo1Error, match="pinned"):
        eng.generate(*x, 8, stop_ids=[], pad_id=0, on_tokens=Recorder(eng))
    assert fo1_b200.lib().fo1_launch_count() == n0
    assert threading.active_count() == threads


def test_zero_new_tokens_is_done_at_once(engine):
    eng, _ = engine
    F, _ = _mods()
    rec = Recorder(eng)
    eng.generate(*_inputs(2, 15), 0, stop_ids=[], pad_id=0, on_tokens=rec)
    assert rec.calls == []
    assert int(eng._stream_buf[2][0]) == F.FO1_STREAM_DONE


# ---------------------------------------------------------------------------------------------------------- HF surface
@pytest.fixture(scope="module")
def fab(tmp_path_factory):
    from importlib import import_module
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    _, E = _mods()
    FB = import_module("vlm-fo1_b200.fabricate")
    root = tmp_path_factory.mktemp("stream")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(root / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(REPO, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    tokenizer, model, procs = load_pretrained_model(model_path, device="cuda:0")
    sizes = {im["file_name"]: (im["width"], im["height"]) for im in fx["instances"]["images"]}
    src = ImageSource(str(root / "none"), str(root / "synth"))
    d = fx["coco"][0]
    msg = [{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                        {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}]

    def kw(**k):
        return prepare_inputs(model_path, model, procs, tokenizer, msg, device="cuda:0", max_tokens=24, **k)
    return model, tokenizer, kw


class RecordingStreamer:
    def __init__(self, fail_at=None):
        self.events, self.fail_at = [], fail_at

    def put(self, value):
        if self.fail_at is not None and sum(e[0] == "put" for e in self.events) + 1 == self.fail_at:
            raise RuntimeError("streamer failed")
        self.events.append(("put", value.clone()))

    def end(self):
        self.events.append(("end", None))


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return (torch.equal(a.sequences, b.sequences) and (a.scores is None) == (b.scores is None)
            and (a.scores is None or all(torch.equal(x, y) for x, y in zip(a.scores, b.scores))))


@pytest.mark.parametrize("case", ["greedy", "sampled", "return_dict"])
def test_streamer_put_order(fab, case):
    model, _, kw = fab
    a = kw(temperature=0.7 if case == "sampled" else 0.0, top_p=0.9)
    extra = dict(return_dict_in_generate=True, output_scores=True) if case == "return_dict" else {}
    torch.manual_seed(21)
    plain = model.generate(**dict(a, streamer=None), **extra)
    rs = RecordingStreamer()
    torch.manual_seed(21)
    got = model.generate(**dict(a, streamer=rs), **extra)
    assert _same(got, plain)
    seq = got if isinstance(got, torch.Tensor) else got.sequences
    new = seq[0, a["inputs"].shape[1]:].cpu()
    kinds = [e[0] for e in rs.events]
    assert kinds[-1] == "end" and kinds.count("end") == 1
    puts = [e[1] for e in rs.events if e[0] == "put"]
    assert torch.equal(puts[0], a["inputs"].cpu())
    assert all(p.dtype == torch.int64 and p.device.type == "cpu" and p.shape == (1,) for p in puts[1:])
    assert torch.equal(torch.cat(puts[1:]) if len(puts) > 1 else torch.zeros(0, dtype=torch.int64), new)


def test_text_iterator_streamer(fab):
    from transformers import TextIteratorStreamer
    model, tok, kw = fab
    a = kw(temperature=0.0, top_p=0.9)
    plain = model.generate(**dict(a, streamer=None))
    streamer = TextIteratorStreamer(tok, skip_prompt=True, skip_special_tokens=True)
    th = threading.Thread(target=model.generate, kwargs=dict(a, streamer=streamer))
    th.start()
    text = "".join(streamer)
    th.join()
    assert text == tok.decode(plain[0, a["inputs"].shape[1]:], skip_special_tokens=True)


def test_streamer_error_propagates(fab):
    model, _, kw = fab
    a = kw(temperature=0.0, top_p=0.9)
    plain = model.generate(**dict(a, streamer=None))
    assert plain.shape[1] - a["inputs"].shape[1] >= 4, "the 5th put must be a generated token"
    threads = threading.active_count()
    with pytest.raises(RuntimeError, match="streamer failed"):
        model.generate(**dict(a, streamer=RecordingStreamer(fail_at=5)))
    assert threading.active_count() == threads
    assert torch.equal(model.generate(**dict(a, streamer=None)), plain)
