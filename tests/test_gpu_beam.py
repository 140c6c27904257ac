"""-m gpu: beam search on the device (csrc/beam.cu, fo1_llm_generate with d.beam) at the 3B widths (2 decoder layers, vocabulary 20000,
non-unit norm gains and non-zero biases: tests/test_gpu_decode_parity.py's model).

  1. Selection is HF's, bit for bit: the engine's own per-step log-prob rows (`scores`) fed to oracle/beam.py (the restatement of
     transformers' _beam_search, pinned against HF's generate by tests/test_oracle_beam.py) reproduce its tokens, lengths,
     beam_indices, sequences_scores and steps with torch.equal.  N = 2, 4, 8; 1 and 3 prompts; every early_stopping value;
     stop ids taken from a free run so that some beams end early.
  2. Each `scores` row is log_softmax of its `logits` row within 1e-5 + 1e-6 |lp| (torch's fp32 log_softmax on the CPU).
  3. The K/V reorder: every beam row's logits at every step pass test_gpu_decode_parity's (A) / (B) bounds against the fp32
     oracle decoder teacher-forced on THAT beam's history (the oracle's running histories).  Negative control: the history the
     row's cache slot would hold without the reorder misses the bound.
  4. Column 0: the N rows of a prompt carry identical bits, equal to its prefill row.
  5. Batch invariance: each prompt of a batch of S = 2 .. 4 prompts (S * N <= 16 rows: the decode-attention split stays at 8 on a
     132-SM H100) equals the same prompt alone, bit for bit.
  6. End to end through Fo1ForCausalLM on a fabricated checkpoint: HF's output types and shapes, sequences_scores * len^lp equal to
     the sum of generate_batch's per-token log-probs, which equal HF's compute_transition_scores on the outputs; generate_batch
     equals one-by-one generate; the towers run once per unique image."""
import gzip
import json
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import beam as OB
from tests.golden_io import nerr, rerr
from tests.test_gpu_decode_parity import TOL_B, _model, _mods, a_bound, make_seq

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_COLS = 12
V = 20000


@pytest.fixture(scope="module")
def model():
    return _model()


@pytest.fixture(scope="module")
def pool():
    grids = [(8, 12), None, (12, 12), (4, 4)]
    return [make_seq(L, gr, 5000 + i) for i, (L, gr) in enumerate(zip([150, 37, 300, 64], grids))]


def run(eng, seqs, N, T=T_COLS, stop=(), es=False, lp=1.0, nr=None, logits=False, logprobs=False):
    E, _, _ = _mods()
    emb = torch.cat([s.emb for s in seqs]).cuda()
    pos = torch.cat([s.pos for s in seqs], dim=1).contiguous()
    beams = E.Beams(N, OB.n_keep(N, len(stop)), lp, es, nr or N)
    out = eng.generate(emb, pos, [s.L for s in seqs], [s.delta for s in seqs], T, list(stop), 0, want_prefill_logits=True,
                       early_exit_interval=4, want_scores=True, want_logits=logits, want_logprobs=logprobs, beams=beams)
    torch.cuda.synchronize()
    assert eng.last_decode_path() == 0
    return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def oracle_of(out, b, N, T, stop, es, lp, nr):
    return OB.beam_search(lambda t, hist: out["scores"][t, b * N:(b + 1) * N], N, OB.n_keep(N, len(stop)), T, stop, length_penalty=lp,
                          early_stopping=es, num_return=nr, beam_offset=b * N)


def check_selection(out, S, N, T, stop, es, lp, nr):
    for b in range(S):
        r = oracle_of(out, b, N, T, stop, es, lp, nr)
        rows = slice(b * nr, (b + 1) * nr)
        tok = torch.tensor([s + [0] * (T - len(s)) for s in r.sequences], dtype=torch.int32)
        bi = torch.tensor([x + [-1] * (T - len(x)) for x in r.beam_indices], dtype=torch.int32)
        assert int(out["beam_steps"][b]) == r.steps, (b, out["beam_steps"], r.steps)
        assert torch.equal(out["lens"][rows], torch.tensor([len(s) for s in r.sequences], dtype=torch.int32))
        assert torch.equal(out["tokens"][rows], tok), (b, out["tokens"][rows], tok)
        assert torch.equal(out["beam_indices"][rows], bi)
        assert torch.equal(out["sequence_scores"][rows], r.sequence_scores)
    return r


def stops_from(out, N, k=2):
    """up to k token ids from the middle of a free run's hypotheses: stop on them and some beams end early"""
    cand = out["tokens"][:, 2:5].flatten().tolist()
    return sorted(set(cand))[:k]


SEL_CASES = [(2, 1, False, 1.0), (2, 3, True, 0.0), (4, 1, "never", 1.3), (4, 3, False, -0.5), (8, 1, True, 1.0), (8, 3, "never", 0.0),
             (4, 3, True, 1.0), (8, 1, False, 1.3)]


@pytest.mark.parametrize("N,S,es,lp", SEL_CASES)
def test_selection_is_hf_bit_for_bit(model, pool, N, S, es, lp):
    eng, _ = model
    seqs = pool[:S]
    free = run(eng, seqs, N, es=es, lp=lp, logits=True)
    check_selection(free, S, N, T_COLS, (), es, lp, N)
    # 2. log-softmax bound on every row the loop wrote
    for b in range(S):
        for t in range(int(free["beam_steps"][b])):
            sc, lg = free["scores"][t, b * N:(b + 1) * N], free["logits"][t, b * N:(b + 1) * N]
            ref = torch.log_softmax(lg, dim=-1)
            assert bool(((sc - ref).abs() <= 1e-5 + 1e-6 * ref.abs()).all()), (b, t, float((sc - ref).abs().max()))
    # with stop ids: beams end early, the finished set fills before max_new
    stop = stops_from(free, N)
    out = run(eng, seqs, N, stop=stop, es=es, lp=lp, nr=max(1, N // 2))
    check_selection(out, S, N, T_COLS, stop, es, lp, max(1, N // 2))
    if lp <= 1.0:          # (a penalty above 1 favours the long hypotheses: the short ones finish but are not returned)
        assert int(out["lens"].min()) < T_COLS, out["lens"]


def test_column0_rows_identical(model, pool):
    eng, _ = model
    N, S = 4, 3
    out = run(eng, pool[:S], N, logits=True)
    for b in range(S):
        for j in range(N):
            assert torch.equal(out["logits"][0, b * N + j], out["prefill_logits"][b])
            assert torch.equal(out["scores"][0, b * N + j], out["scores"][0, b * N])


@pytest.mark.parametrize("N,S", [(4, 2), (4, 4), (8, 2), (2, 3)])
def test_batch_invariance(model, pool, N, S):
    eng, _ = model
    seqs = pool[:S]
    stop = stops_from(run(eng, seqs[:1], N), N, 1)
    both = run(eng, seqs, N, stop=stop, es=False, lp=1.0, nr=2)
    for b in range(S):
        alone = run(eng, [seqs[b]], N, stop=stop, es=False, lp=1.0, nr=2)
        rows = slice(2 * b, 2 * b + 2)
        assert torch.equal(both["tokens"][rows], alone["tokens"]) and torch.equal(both["lens"][rows], alone["lens"])
        assert torch.equal(both["sequence_scores"][rows], alone["sequence_scores"])
        bi = both["beam_indices"][rows]
        assert torch.equal(torch.where(bi >= 0, bi - b * N, bi), alone["beam_indices"])
        steps = int(alone["beam_steps"][0])
        assert int(both["beam_steps"][b]) == steps
        assert torch.equal(both["scores"][:steps, b * N:(b + 1) * N], alone["scores"][:steps])


def test_kv_reorder_against_fp32_decoder(model, pool):
    """3: each running beam's rows against the oracle decoder on its own history; the un-reordered history must miss."""
    eng, orc = model
    N, S, T = 4, 2, 8
    seqs = pool[:S]
    out = run(eng, seqs, N, T=T, logits=True)
    tol_b = TOL_B[0]
    moved = 0
    for b, seq in enumerate(seqs):
        r = oracle_of(out, b, N, T, (), False, 1.0, N)
        steps = r.steps
        for j in range(N):
            hists = [[]] + [r.running[t - 1][j] for t in range(1, steps)]
            got = out["logits"][:steps, b * N + j]
            ref = torch.stack([orc.rows(seq, h, True)[-1] for h in hists])
            f32 = torch.stack([orc.rows(seq, h, False)[-1] for h in hists])
            ra = rerr(got, f32) / a_bound(ref, f32)
            rb = max(nerr(got[t], ref[t]) for t in range(steps)) / tol_b
            assert ra <= 1.0 and rb <= 1.0, (b, j, ra, rb)
            # the tokens fed to slot j, step by step: what its cache would hold without the reorder
            fed = [[r.running[s][j][s] for s in range(t)] for t in range(steps)]
            if fed != hists:
                moved += 1
                ctrl = torch.stack([orc.rows(seq, h, False)[-1] for h in fed])
                miss = max(rerr(got, ctrl) / a_bound(ref, f32), max(nerr(got[t], ctrl[t]) for t in range(steps)) / tol_b)
                assert miss > 1.0, (b, j, miss)
    assert moved > 0, "no beam changed parent: the reorder was not exercised"


# ---------------------------------------------------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def fab(tmp_path_factory):
    from importlib import import_module
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    E, _, _ = _mods()
    FB = import_module("vlm-fo1_b200.fabricate")
    root = tmp_path_factory.mktemp("beam")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(root / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(REPO, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    tokenizer, mdl, procs = load_pretrained_model(model_path, device="cuda:0")
    sizes = {im["file_name"]: (im["width"], im["height"]) for im in fx["instances"]["images"]}
    src = ImageSource(str(root / "none"), str(root / "synth"))
    msgs = []
    for d in fx["coco"][:3]:
        msgs.append([{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                                  {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}])

    def kw(i, **k):
        return prepare_inputs(model_path, mdl, procs, tokenizer, msgs[i], device="cuda:0", max_tokens=10, **k)
    return mdl, kw


def test_generate_beam_end_to_end(fab):
    from transformers.generation.utils import GenerateBeamDecoderOnlyOutput, GenerationMixin
    mdl, kw = fab
    a = kw(0, temperature=0.0, top_p=0.9)
    a.pop("streamer", None)                             # prepare_inputs' TextStreamer: HF refuses it with beams
    N, nr, lp = 4, 3, 1.3
    plain = mdl.generate(**a, num_beams=N, num_return_sequences=nr, length_penalty=lp)
    out = mdl.generate(**a, num_beams=N, num_return_sequences=nr, length_penalty=lp, return_dict_in_generate=True, output_scores=True,
                       output_logits=True)
    assert isinstance(out, GenerateBeamDecoderOnlyOutput) and torch.equal(out.sequences, plain)
    P = a["inputs"].shape[1]
    W = plain.shape[1] - P
    assert plain.shape[0] == nr and plain.dtype == torch.long and out.sequences_scores.shape == (nr,)
    assert out.beam_indices.shape == (nr, W) and len(out.scores) == len(out.logits) and out.scores[0].shape == (N, out.logits[0].shape[1])
    assert len(out.scores) >= W
    (seq, lps), = mdl.generate_batch([dict(a, num_beams=N, num_return_sequences=nr, length_penalty=lp)], output_logprobs=True)
    assert torch.equal(seq, plain) and lps.shape == (nr, W)
    lens = (out.beam_indices >= 0).sum(-1)
    assert torch.allclose(out.sequences_scores * lens.float() ** lp, lps.sum(-1), atol=1e-4, rtol=1e-5)
    vocab = out.scores[0].shape[1]
    stand_in = SimpleNamespace(config=SimpleNamespace(get_text_config=lambda: SimpleNamespace(vocab_size=vocab)))
    ts = GenerationMixin.compute_transition_scores(stand_in, out.sequences, out.scores, out.beam_indices)
    assert torch.equal(ts.float().cpu(), lps.cpu())
    with pytest.raises(NotImplementedError):           # beam_indices stays refused by the model's own method
        mdl.compute_transition_scores(out.sequences, out.scores, out.beam_indices)


def test_generate_batch_beams_equals_generate_and_shares_towers(fab, monkeypatch):
    mdl, kw = fab
    kws = [dict(kw(i, temperature=0.0, top_p=0.9), num_beams=2, num_return_sequences=2, early_stopping=True) for i in (0, 1, 0)]
    for k in kws:
        k.pop("streamer", None)
    one = [mdl.generate(**k) for k in kws]
    eng = mdl.pipeline.eng
    runs = []
    vit = eng.vit_forward
    monkeypatch.setattr(eng, "vit_forward", lambda px, grids: (runs.append(len(px)), vit(px, grids))[1])
    batch = mdl.generate_batch(kws)
    assert sum(runs) == 2, runs                          # samples 0 and 2 share their image
    for a, b in zip(one, batch):
        assert torch.equal(a, b)
    d = mdl.generate_batch([dict(k, return_dict_in_generate=True, output_scores=True) for k in kws])
    for k, x in zip(kws, d):
        ref = mdl.generate(**k, return_dict_in_generate=True, output_scores=True)
        assert torch.equal(x.sequences, ref.sequences) and torch.equal(x.beam_indices, ref.beam_indices)
        assert torch.equal(x.sequences_scores, ref.sequences_scores)
        assert len(x.scores) == len(ref.scores) and all(torch.equal(p, q) for p, q in zip(x.scores, ref.scores))
