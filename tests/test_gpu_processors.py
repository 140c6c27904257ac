"""Logits processors on the device: fo1_logits_process against oracle/processors.py bit for bit, and teacher-forced end-to-end calls on
both decode paths (every scores row equals the oracle applied to its raw logits row and the sequence's history; the token is the
choice rule on it).  Random-init model at the 3B widths, as in test_gpu_decode_parity.py."""
import numpy as np
import pytest
import torch

from oracle import processors as O
from oracle import sampling as OS
from tests.test_gpu_decode_parity import _model, _mods, make_seq
from tests.test_gpu_slots import fab_model  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
VOCAB = 20000
STOP = [17, 29]


@pytest.fixture(scope="module")
def eng():
    e, _ = _model(vocab=VOCAB, layers=2, seed=43)
    return e


def _E():
    return _mods()[0]


def _sets():
    S = _E().ProcessorSet
    return {
        "ngram": S(no_repeat_ngram_size=3),
        "ngram1": S(no_repeat_ngram_size=1),
        "bad": S(bad_words_ids=((11,), (4, 5), (5, 6, 7), (3, 4, 5), (8, 8))),
        "bias": S(sequence_bias=(((7,), 1.5), ((2, 7), -0.25), ((1, 2, 7), 3.0), ((3,), -2.0), ((8, 3), 0.125))),
        "min": S(min_length=1300, eos_token_ids=(17, 29)),
        "min_new": S(min_new_tokens=9, eos_token_ids=(17, 29)),
        "suppress": S(suppress_tokens=(0, 1, 2), begin_suppress_tokens=(9, 10)),
        "all": S(no_repeat_ngram_size=2, bad_words_ids=tuple((int(a), int(b)) for a, b in zip(range(30, 50), range(50, 70))) + ((12,),),
                 sequence_bias=(((4,), 0.5), ((2, 4), 1.0), ((9, 9), -3.0)), min_length=40, min_new_tokens=5, eos_token_ids=(17, 29),
                 suppress_tokens=(0,), begin_suppress_tokens=(1,)),
    }


@pytest.mark.parametrize("name", ["ngram", "ngram1", "bad", "bias", "min", "min_new", "suppress", "all"])
def test_row_routine_equals_oracle(name):
    E = _E()
    ps = _sets()[name]
    rng = np.random.default_rng(len(name))
    V, n = 4096, 12
    prompts, outs, cols = [], [], []
    for r in range(n):
        P = int(rng.choice([5, 60, 1200]))
        hi = int(rng.choice([4, 20, 4096]))             # small alphabets repeat n-grams and complete bad words / biases
        p = rng.integers(0, hi, P).tolist()
        p[0] = -200                                       # a placeholder id
        c = int(rng.choice([0, 1, 3, 200, 4800]))
        o = rng.integers(0, min(hi, V), c).tolist()
        if r % 3 == 0 and c >= 4:
            o[-3:] = p[1:4] if P >= 4 else o[-3:]        # an n-gram across the prompt / output boundary
        prompts.append(p); outs.append(o); cols.append(c)
    ld = max(max(cols), 1)
    out_t = torch.zeros((n, ld), dtype=torch.int32)
    for r, o in enumerate(outs):
        out_t[r, :len(o)] = torch.tensor(o, dtype=torch.int32) if o else out_t[r, :0]
    rows = torch.randn((n, V)) * 3
    dev = rows.cuda()
    sets = [ps if r != n - 1 else None for r in range(n)]          # the last row has no set: never edited
    E.logits_process(dev, E.Processors(sets, prompts), out_t.cuda(), cols)
    got = dev.cpu()
    for r in range(n):
        want = O.process(rows[r], prompts[r] + outs[r], len(prompts[r]), ps) if sets[r] is not None else rows[r]
        assert torch.equal(got[r], want), (name, r)


def _batch(B, L0=40):
    seqs = [make_seq(L0 + 7 * (b % 5), None, 200 + b, vocab=VOCAB) for b in range(B)]
    return (torch.cat([s.emb for s in seqs]).cuda(), torch.cat([s.pos for s in seqs], 1).cuda(), [s.L for s in seqs],
            [s.delta for s in seqs])


def _prompts(B):
    rng = np.random.default_rng(7)
    return [[-200] + rng.integers(30, 70, 30 + b % 4).tolist() for b in range(B)]


def _gen(eng, monkeypatch, B, T, mega, sets=None, sampling=None, scored=True, stream=False, stop=STOP):
    if mega:
        monkeypatch.delenv("FO1_NO_MEGA", raising=False)
    else:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    E = _E()
    emb, pos, lens, deltas = _batch(B)
    pr = E.Processors(sets, _prompts(B)) if sets is not None else None
    cols = []
    on = (lambda lo, hi, t, ln: cols.append(hi)) if stream else None
    out = eng.generate(emb, pos, lens, deltas, T, stop_ids=stop, pad_id=3, early_exit_interval=4, sampling=sampling, want_logprobs=scored,
                       want_scores=scored, want_logits=scored, on_tokens=on, processors=pr)
    torch.cuda.synchronize()
    out["path"] = eng.last_decode_path()
    return out


def _check_teacher_forced(out, sets, prompts, greedy, seeds=None):
    lens = out["lens"].cpu().tolist()
    toks = out["tokens"].cpu()
    for b, ps in enumerate(sets):
        for c in range(lens[b]):
            raw = out["logits"][c, b].cpu()
            hist = prompts[b] + toks[b, :c].tolist()
            want = O.process(raw, hist, len(prompts[b]), ps) if ps is not None else raw
            assert torch.equal(out["scores"][c, b].cpu(), want), (b, c)
            if greedy:
                assert int(toks[b, c]) == int(torch.argmax(want)), (b, c)
            else:       # the draw on the processed row (T 1, no cut), where the float64 oracle decides it
                d = OS.sample(want.numpy(), 1.0, 1.0, 0, seeds[b], c)
                assert torch.isfinite(want[int(toks[b, c])]), (b, c)
                if d["margin"] > 1e-6:
                    assert int(toks[b, c]) == d["token"], (b, c)


@pytest.mark.parametrize("B,mega", [(1, True), (8, True), (17, True), (33, False)])
@pytest.mark.parametrize("mode", ["greedy", "sampled"])
def test_teacher_forced_end_to_end(eng, monkeypatch, B, mega, mode):
    E = _E()
    S = _sets()
    names = ["all", "ngram", "bad", "bias", "min", "min_new", "suppress", "ngram1"]
    sets = [S[names[b % len(names)]] if b % 4 != 3 else None for b in range(B)]
    sampling = E.Sampling([1.0] * B, [1.0] * B, [0] * B, list(range(B))) if mode == "sampled" else None
    out = _gen(eng, monkeypatch, B, 24, mega, sets, sampling)
    assert out["path"] == (1 if mega else 0)
    _check_teacher_forced(out, sets, _prompts(B), mode == "greedy", seeds=list(range(B)))
    # rows without a set are bit-identical to the call without processors
    plain = _gen(eng, monkeypatch, B, 24, mega, None, sampling)
    for b, ps in enumerate(sets):
        if ps is None:
            n = int(plain["lens"][b])
            assert int(out["lens"][b]) == n and torch.equal(out["tokens"][b], plain["tokens"][b]), b
            assert torch.equal(out["logprobs"][b, :n], plain["logprobs"][b, :n]), b


def test_streamed_and_unscored_equal_scored(eng, monkeypatch):
    S = _sets()
    sets = [S["all"], None, S["ngram"], S["bad"]]
    a = _gen(eng, monkeypatch, 4, 24, True, sets)
    b = _gen(eng, monkeypatch, 4, 24, True, sets, scored=False, stream=True)
    c = _gen(eng, monkeypatch, 4, 24, True, sets, scored=False)
    for o in (b, c):
        assert torch.equal(a["tokens"], o["tokens"]) and torch.equal(a["lens"], o["lens"])


def _ngrams(seq, n):
    return [tuple(seq[i:i + n]) for i in range(len(seq) - n + 1)]


def _new_repeats(seq, P, n):
    """n-grams that end in the output (index >= P) and occurred earlier in seq: what no_repeat_ngram_size=n forbids."""
    seen, rep = set(), []
    for i in range(len(seq) - n + 1):
        g = tuple(seq[i:i + n])
        if i + n - 1 >= P and g in seen:
            rep.append(g)
        seen.add(g)
    return rep


def test_non_vacuous(eng, monkeypatch):
    """Each processor changes what the seeded call emits, and the constraint then holds everywhere: the plain greedy call repeats a
    3-gram, emits a bigram and stops at column 2 on a stop id; with no_repeat_ngram_size=3 no 3-gram repeats in prompt + output, with
    the bigram banned it never appears in the output, and with min_new_tokens=12 no sequence stops before column 12."""
    B, T = 4, 48
    S = _E().ProcessorSet
    prompts = _prompts(B)
    plain = _gen(eng, monkeypatch, B, T, True, None, scored=False, stop=[])
    toks = [plain["tokens"][b, :int(plain["lens"][b])].tolist() for b in range(B)]
    # n-grams
    assert any(_new_repeats(prompts[b] + toks[b], len(prompts[b]), 3) for b in range(B))
    out = _gen(eng, monkeypatch, B, T, True, [S(no_repeat_ngram_size=3)] * B, scored=False, stop=[])
    for b in range(B):
        assert not _new_repeats(prompts[b] + out["tokens"][b, :int(out["lens"][b])].tolist(), len(prompts[b]), 3), b
    # bad words: each sequence's own first output bigram
    sets = [S(bad_words_ids=(tuple(toks[b][4:6]),)) for b in range(B)]
    out = _gen(eng, monkeypatch, B, T, True, sets, scored=False, stop=[])
    for b in range(B):
        seq = prompts[b][-1:] + out["tokens"][b, :int(out["lens"][b])].tolist()
        assert tuple(toks[b][4:6]) not in _ngrams(seq, 2), b
    # min_new_tokens: the stop ids are the tokens the plain call emits at column 2
    stop = sorted({toks[b][2] for b in range(B)})
    early = _gen(eng, monkeypatch, B, T, True, None, scored=False, stop=stop)
    assert all(int(x) <= 3 for x in early["lens"].tolist())
    out = _gen(eng, monkeypatch, B, T, True, [S(min_new_tokens=12, eos_token_ids=tuple(stop))] * B, scored=False, stop=stop)
    assert all(int(x) >= 12 for x in out["lens"].tolist()), out["lens"]


def test_neutral_processors_are_the_plain_call(eng, monkeypatch):
    for mega in (True, False):
        plain = _gen(eng, monkeypatch, 3, 16, mega, None)
        neutral = _gen(eng, monkeypatch, 3, 16, mega, [None, None, None])
        for k in ("tokens", "lens", "scores", "logits", "logprobs"):
            assert torch.equal(plain[k], neutral[k]), k
        assert plain["path"] == neutral["path"]


@pytest.mark.parametrize("mega", [True, False])
def test_slot_pool_equals_static_batch(eng, monkeypatch, mega):
    if mega:
        monkeypatch.delenv("FO1_NO_MEGA", raising=False)
    else:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    E = _E()
    S = _sets()
    N, T = 4, 20
    sets = [S["all"], None, S["ngram"], S["bad"]]
    static = _gen(eng, monkeypatch, N, T, mega, sets, scored=False)
    emb, pos, lens, deltas = _batch(N)
    prompts = _prompts(N)
    with E.SlotPool(eng, N, max(lens) + T + 1, T, STOP, 3) as pool:
        pool.admit(list(range(N)), emb, pos, lens, torch.tensor(deltas, dtype=torch.int32), [T] * N, processors=E.Processors(sets, prompts))
        pool.decode(0)
        torch.cuda.synchronize()
        for b in range(N):
            n = int(static["lens"][b])
            assert int(pool.lens[b]) == n, b
            assert torch.equal(pool.tokens[b, :n], static["tokens"][b, :n]), b


def _plain_kw(kw, i):
    return kw(i, max_new=24)


def test_model_entry_points_with_processors(fab_model):
    """Fo1ForCausalLM with processors, up from the kwargs: generate_batch (per-sample sets, two requests on one image: the shared
    prefix path) and generate_iter (3 slots for 7 requests: slots reused with other sets, and requests without processors admitted into
    a pool that has them) equal generate alone for every request (at most 8 sequences on the persistent kernel); the processors change
    the output and the banned bigram never appears."""
    _, model, kw = fab_model
    plain = [model.generate(**_plain_kw(kw, i))[0].tolist() for i in range(6)]
    P = [len(_plain_kw(kw, i)["inputs"][0]) for i in range(6)]
    gen = [plain[i][P[i]:] for i in range(6)]
    extra = [dict(no_repeat_ngram_size=2), dict(bad_words_ids=[gen[1][2:4]]), dict(min_new_tokens=20), {},
             dict(sequence_bias=[[[gen[4][1]], -30.0]]), dict(suppress_tokens=[gen[5][0]], no_repeat_ngram_size=3), dict(bad_words_ids=[gen[0][1:3]])]
    items = [0, 1, 2, 3, 4, 5, 0]
    kws = [dict(_plain_kw(kw, i), **e) for i, e in zip(items, extra)]
    alone = [model.generate(**dict(k))[0].tolist() for k in kws]
    assert alone[1] != plain[1] and alone[4] != plain[4] and alone[5] != plain[5]
    assert tuple(gen[1][2:4]) not in _ngrams(alone[1][P[1] - 1:], 2)
    assert tuple(gen[0][1:3]) not in _ngrams(alone[6][P[0] - 1:], 2)
    batch = model.generate_batch([dict(k) for k in kws])
    for j, r in enumerate(batch):
        assert r[0].tolist() == alone[j], j
    got = dict(model.generate_iter([dict(k) for k in kws], batch_size=3))
    for j in range(len(kws)):
        assert got[j][0].tolist() == alone[j], j


def test_model_num_return_sequences_with_processors(fab_model):
    """num_return_sequences copies (the shared-prefix path) with processors: every scores row is the oracle applied to the raw logits
    row and that copy's history (temperature 1, no cut), and no output token completes a 2-gram seen before."""
    _, model, kw = fab_model
    k = dict(kw(2, max_new=16, temperature=1.0, top_p=1.0), top_k=0, do_sample=True, num_return_sequences=3, no_repeat_ngram_size=2,
             return_dict_in_generate=True, output_scores=True, output_logits=True)
    prompt = k["inputs"][0].tolist()
    out = model.generate(**k)
    ps = _E().ProcessorSet(no_repeat_ngram_size=2)
    seqs = out.sequences.tolist()
    for r in range(3):
        new = seqs[r][len(prompt):]
        n = len(out.scores)
        for c in range(n):
            if c > 0 and new[c - 1] in (151645, 151643):      # past this copy's stop: rows unspecified
                break
            want = O.process(out.logits[c][r].cpu(), prompt + new[:c], len(prompt), ps)
            assert torch.equal(out.scores[c][r].cpu(), want), (r, c)
        assert not _new_repeats(prompt + [t for t in new if t not in (151645, 151643)], len(prompt), 2), r
