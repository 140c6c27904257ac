"""-m gpu: fo1_llm_generate called directly through ctypes with a descriptor filled by hand: every option NULL (greedy), d.sampling,
and d.sampling with d.scores (greedy or sampled).  Each must give Engine.generate's tokens, lengths, step count and scores bit for bit
on both decode paths."""
import ctypes as C

import pytest
import torch

from tests.test_gpu_decode_mega import _batch, _engine

pytestmark = pytest.mark.gpu


def _mods():
    from importlib import import_module
    import fo1_b200
    return fo1_b200._lib, import_module("vlm-fo1_b200.engine")


@pytest.fixture(scope="module")
def engine():
    return _engine()[0]


def _direct(eng, mode, emb, pos, lens, T, stop, samp):
    """One fo1_llm_generate call with the options `mode` names, in a descriptor filled as Engine.generate fills it."""
    F, E = _mods()
    B, V, dev = len(lens), eng.cfg.llm["vocab_size"], eng.device
    toks = torch.empty((B, T), dtype=torch.int32, device=dev)
    out_lens = torch.zeros((B,), dtype=torch.int32, device=dev)
    pos = pos.to(dev, torch.int32).contiguous()
    sl, rd = (C.c_int32 * B)(*lens), (C.c_int32 * B)(*([0] * B))
    st = (C.c_int32 * max(len(stop), 1))(*stop)
    d = E.GenerateDescC()
    d.n_seqs, d.seq_lens, d.rope_deltas, d.stop_ids, d.n_stop_ids = B, sl, rd, st, len(stop)
    d.inputs_embeds, d.position_ids = emb.data_ptr(), pos.data_ptr()
    d.max_new_tokens, d.pad_id, d.early_exit_interval = T, 0, 2
    d.out_tokens, d.out_lens = toks.data_ptr(), out_lens.data_ptr()
    L, stream = F.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if samp is not None:
        sd, _keep = F.sampling_desc(samp.temperature, samp.top_p, samp.top_k, samp.seed)     # (the arrays must outlive the call)
        d.sampling = C.pointer(sd)
    out = dict()
    if mode == "scored":
        out["logprobs"] = torch.empty((B, T), dtype=torch.float32, device=dev)
        out["scores"] = torch.empty((T, B, V), dtype=torch.float32, device=dev)
        out["logits"] = torch.empty((T, B, V), dtype=torch.float32, device=dev)
        desc = F.ScoreDesc(out["logprobs"].data_ptr(), out["scores"].data_ptr(), out["logits"].data_ptr(), None)
        d.scores = C.pointer(desc)
    F.check(L.fo1_llm_generate(eng._h, C.byref(d), stream), "fo1_llm_generate")
    torch.cuda.synchronize()
    return dict(out, tokens=toks, lens=out_lens, steps_run=d.steps_run)


@pytest.mark.parametrize("no_mega", [False, True])
@pytest.mark.parametrize("mode,sampled", [("greedy", False), ("sampled", True), ("scored", False), ("scored", True)])
def test_hand_filled_descriptor_equals_generate(engine, mode, sampled, no_mega, monkeypatch):
    _, E = _mods()
    if no_mega:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    lens = [41, 78, 115]
    emb, pos, _ = _batch(lens, seed=17)
    B, T = len(lens), 10
    samp = E.Sampling([0.7] * B, [0.9] * B, [50] * B, [900 + b for b in range(B)]) if sampled else None
    scored = mode == "scored"
    kw = dict(want_logprobs=True, want_scores=True, want_logits=True) if scored else {}
    free = engine.generate(emb, pos, lens, [0] * B, T, stop_ids=[], pad_id=0, early_exit_interval=2, sampling=samp)
    stop = [int(free["tokens"][0, 3])]                                     # ends sequence 0 mid-run
    ref = engine.generate(emb, pos, lens, [0] * B, T, stop_ids=stop, pad_id=0, early_exit_interval=2, sampling=samp, **kw)
    out = _direct(engine, mode, emb, pos, lens, T, stop, samp)
    assert engine.last_decode_path() == (0 if no_mega else 1)
    assert out["steps_run"] == ref["steps_run"]
    for k in ("tokens", "lens") + (("logprobs",) if scored else ()):
        assert torch.equal(out[k], ref[k]), k
    assert int(out["lens"][0]) <= 4
    if scored:                                                             # rows past a sequence's stop are unspecified
        for b, n in enumerate(out["lens"].cpu().tolist()):
            assert torch.equal(out["scores"][:n, b], ref["scores"][:n, b]) and torch.equal(out["logits"][:n, b], ref["logits"][:n, b])
