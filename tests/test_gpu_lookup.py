"""Prompt-lookup decoding on the device: the draft kernel against oracle/lookup.py, and every lookup call bit-identical (torch.equal)
to the plain per-kernel call (FO1_NO_MEGA=1) at the same batch: tokens, lengths, pad tails, logprobs and every scores / logits row
up to each length.  Random-init model at the 3B widths, as in test_gpu_decode_parity.py."""
import numpy as np
import pytest
import torch

from oracle import lookup as O
from tests.test_gpu_decode_parity import _model, _mods, make_seq
from tests.test_gpu_sampling import fab  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
VOCAB = 20000


@pytest.fixture(scope="module")
def eng():
    e, _ = _model(vocab=VOCAB, layers=2, seed=41)
    return e


def test_draft_kernel_equals_oracle():
    E, _, _ = _mods()
    rng = np.random.default_rng(5)
    for K in (1, 4, 16):
        for ngram in (1, 2, 3):
            corp = [rng.integers(0, int(rng.choice([3, 10, 500])), int(rng.integers(1, 300))).tolist() for _ in range(37)]
            corp[0][0:2] = [-200, -300]
            ld = max(len(c) for c in corp)
            dev = torch.zeros((len(corp), ld), dtype=torch.int32)
            for b, c in enumerate(corp):
                dev[b, :len(c)] = torch.tensor(c)
            lens = torch.tensor([len(c) for c in corp], dtype=torch.int32)
            emitted = torch.from_numpy(rng.integers(0, 20, len(corp))).to(torch.int32)
            stop = [1, 7]
            d, n = E.lookup_drafts(dev.cuda(), lens.cuda(), K, ngram, stop, emitted.cuda(), 20)
            d, n = d.cpu(), n.cpu()
            for b, c in enumerate(corp):
                want = O.drafts(c, K, ngram, stop, cap=20 - int(emitted[b]) - 1)
                assert d[b, :int(n[b])].tolist() == want, (b, K, ngram)


def _batch(B, L0=40):
    seqs = [make_seq(L0 + 7 * (b % 5), None, 100 + b, vocab=VOCAB) for b in range(B)]
    return (torch.cat([s.emb for s in seqs]).cuda(), torch.cat([s.pos for s in seqs], 1).cuda(), [s.L for s in seqs],
            [s.delta for s in seqs])


def _run(eng, monkeypatch, batch, T, stop, sampling=None, scored=False, lookup=None):
    monkeypatch.setenv("FO1_NO_MEGA", "1")
    emb, pos, lens, deltas = batch
    out = eng.generate(emb, pos, lens, deltas, T, stop_ids=stop, pad_id=3, early_exit_interval=4, sampling=sampling,
                       want_logprobs=scored, want_scores=scored, want_logits=scored, lookup=lookup)
    torch.cuda.synchronize()
    return out


def _assert_same(a, b, scored):
    assert torch.equal(a["lens"], b["lens"])
    assert torch.equal(a["tokens"], b["tokens"])          # tokens up to each length, and pad from there to the end
    if scored:
        assert torch.equal(a["logprobs"], b["logprobs"])
        for s, n in enumerate(a["lens"].tolist()):
            assert torch.equal(a["scores"][:n, s], b["scores"][:n, s])
            assert torch.equal(a["logits"][:n, s], b["logits"][:n, s])


def _sampling(E, B, greedy=False):
    if greedy:
        return None
    return E.Sampling([0.7] * B, [0.9] * B, [50] * B, [1000 + b for b in range(B)])


@pytest.mark.parametrize("B", [1, 8, 17, 33])
@pytest.mark.parametrize("mode", ["greedy", "sampled", "scored"])
def test_lookup_bit_identical_to_plain(eng, monkeypatch, B, mode):
    E, _, _ = _mods()
    batch = _batch(B)
    T = 24
    samp = None if mode != "sampled" else _sampling(E, B)
    scored = mode == "scored"
    plain = _run(eng, monkeypatch, batch, T, [], samp, scored)
    toks = plain["tokens"].cpu().tolist()
    # stop ids taken from the plain output: sequences end at different steps (and the stop ids lie inside the corpora)
    stop = sorted({toks[b][T // 2 + b % 7] for b in range(0, B, 3)})
    plain = _run(eng, monkeypatch, batch, T, stop, samp, scored)
    toks = plain["tokens"].cpu().tolist()
    acc_total = {}
    for K in (1, 4, 16):
        for kind in ("full", "partial", "none"):
            if kind == "full":
                corpus = [t for t in toks]                                  # the plain run's own output
            elif kind == "partial":
                corpus = [t[: T // 2] + [(x + 1) % VOCAB for x in t[T // 2:]] for t in toks]
            else:
                corpus = [[] for _ in toks]
            lk = E.Lookup(num_tokens=K, max_ngram=3, corpus=corpus)
            out = _run(eng, monkeypatch, batch, T, stop, samp, scored, lk)
            _assert_same(out, plain, scored)
            acc_total[(K, kind)] = int(out["lookup_accepted"].sum())
    for K in (1, 4, 16):
        assert acc_total[(K, "full")] > 0 and acc_total[(K, "partial")] > 0, acc_total


def test_lookup_max_new_mid_step(eng, monkeypatch):
    """max_new_tokens is reached inside a step: the drafts are capped and the call ends through the early-exit poll."""
    E, _, _ = _mods()
    batch = _batch(8)
    for T in (2, 5, 9):
        plain = _run(eng, monkeypatch, batch, T, [])
        corpus = plain["tokens"].cpu().tolist()
        out = _run(eng, monkeypatch, batch, T, [], lookup=E.Lookup(16, 2, corpus))
        _assert_same(out, plain, False)
        assert out["steps_run"] <= T - 1


def test_lookup_shared_prefix(eng, monkeypatch):
    """A shared-prefix batch (the prefill of fo1_llm_generate with d.prefix) decodes with lookup as the same call without it."""
    E, _, _ = _mods()
    B, P = 6, 30
    s0 = make_seq(P + 10, None, 7, vocab=VOCAB)
    seqs = [make_seq(P + 10, None, 200 + b, vocab=VOCAB) for b in range(B)]
    embs = [torch.cat([s0.emb[:P], s.emb[P:]]) for s in seqs]
    pos = s0.pos
    prefix = E.Prefix(lens=[P], embeds=s0.emb[:P].cuda(), position_ids=pos[:, :P].cuda(), seq_group=[0] * B)
    own = torch.cat([e[P:] for e in embs]).cuda()
    own_pos = torch.cat([pos[:, P:]] * B, 1).cuda()
    monkeypatch.setenv("FO1_NO_MEGA", "1")
    T = 16
    plain = eng.generate(own, own_pos, [P + 10] * B, [s0.delta] * B, T, stop_ids=[], pad_id=3, early_exit_interval=4, prefix=prefix)
    corpus = plain["tokens"].cpu().tolist()
    out = eng.generate(own, own_pos, [P + 10] * B, [s0.delta] * B, T, stop_ids=[], pad_id=3, early_exit_interval=4, prefix=prefix,
                       lookup=E.Lookup(4, 2, corpus))
    _assert_same(out, plain, False)
    assert int(out["lookup_accepted"].sum()) > 0


def test_hf_generate_and_batch(fab, monkeypatch):
    """Fo1ForCausalLM.generate(prompt_lookup_num_tokens=10) equals the plain per-kernel generate; generate_batch equals one-by-one.
    Each call's engine output is recorded; a second pass puts the plain answer in front of the corpus the model passes (the
    prompt ids), so that drafts are accepted and the comparison is not plain decoding against itself."""
    _, model, kw = fab
    E, _, _ = _mods()
    monkeypatch.setenv("FO1_NO_MEGA", "1")
    pipe, outs, extra = model.pipeline, [], {}
    real = pipe.generate

    def recorded(samples, *a, **k):
        lk = k.get("lookup")
        if lk is not None and extra:
            # the answer first: its first token's leftmost occurrence is then the answer's own start, not a prompt id
            k["lookup"] = E.Lookup(lk.num_tokens, lk.max_ngram, [extra[tuple(s.input_ids)] + list(s.input_ids) for s in samples])
        out = real(samples, *a, **k)
        outs.append(out)
        return out
    monkeypatch.setattr(pipe, "generate", recorded)
    for echo in (False, True):
        outs.clear()
        if echo:    # no stop id: the answers run to max_new_tokens, so there is something to accept
            monkeypatch.setattr(model, "default_stop_ids", [])
        for i in range(3):
            a = kw(i)
            a["streamer"] = None        # prepare_inputs adds a TextStreamer, and a streamed call runs without lookup
            if echo:
                a.pop("stopping_criteria", None)
            plain = model.generate(**a)
            P = a["inputs"].shape[1]
            if echo:
                extra[tuple(a["inputs"][0].tolist())] = plain[0, P:].tolist()
            got = model.generate(**a, prompt_lookup_num_tokens=10)
            assert torch.equal(plain, got), (i, echo)
        if echo:
            acc = [int(o["lookup_accepted"].sum()) for o in outs if "lookup_accepted" in o]
            assert sum(acc) > 0, (acc, [o["lens"].tolist() for o in outs])
    monkeypatch.undo()
    monkeypatch.setenv("FO1_NO_MEGA", "1")
    kws = [kw(i, temperature=0.7, top_p=0.9) for i in range(4)] + [kw(4)]
    for k in kws:
        k["prompt_lookup_num_tokens"] = 4
        k["streamer"] = None
    torch.manual_seed(5)
    batch = model.generate_batch(kws)
    torch.manual_seed(5)
    ones = [model.generate(**k) for k in kws]
    for i, (one, got) in enumerate(zip(ones, batch)):
        assert one.shape == got.shape and torch.equal(one, got), i
