"""CPU: the argument handling of the logits processors -- Fo1ForCausalLM._processors' reading of the call's kwargs, else
generation_config.json, HF's ValueErrors, neutral values, the refusals, and fo1_llm_generate's host checks of d.processors (before any
CUDA call).  The model tests record the pipeline call instead of running it (tests/test_beam_args.py)."""
import ctypes
from types import SimpleNamespace

import pytest

from tests.test_beam_args import _Stop, _call, _kw, _lib, _model  # noqa: F401

VOCAB = 1000


def _m(gc=None):
    m = _model(generation_config=gc)
    m.engine = SimpleNamespace(cfg=SimpleNamespace(llm={"vocab_size": VOCAB}))
    return m


def test_neutral_values_give_none_and_the_old_call():
    m = _m()
    plain = _call(m)
    assert "processors" not in plain
    for kw in (dict(no_repeat_ngram_size=0), dict(min_length=0), dict(min_new_tokens=0), dict(suppress_tokens=[]),
               dict(begin_suppress_tokens=[]), dict(remove_invalid_values=False), dict(guidance_scale=1.0)):
        assert m._processors(kw) is None, kw
        assert _call(m, **kw) == plain, kw


def test_kwargs_then_generation_config():
    m = _m(dict(no_repeat_ngram_size=4, eos_token_id=[7, 8], suppress_tokens=[1, 2000]))
    ps = m._processors({})
    assert ps.no_repeat_ngram_size == 4 and ps.suppress_tokens == (1,)           # an id past the vocabulary is dropped, as HF's isin
    ps = m._processors(dict(no_repeat_ngram_size=2, min_new_tokens=3))
    assert ps.no_repeat_ngram_size == 2 and ps.min_new_tokens == 3 and ps.eos_token_ids == (7, 8)
    ps = _m()._processors(dict(min_length=9))
    assert ps.min_length == 9
    assert ps.eos_token_ids == ()                     # the default stop ids lie past VOCAB: dropped, as HF's isin drops them
    ps = m._processors(dict(min_length=9, eos_token_id=[7]))
    assert ps.min_length == 9 and ps.eos_token_ids == (7,)
    c = _call(m, bad_words_ids=[[5, 6], [7], [9]], sequence_bias=[[[3], 1.0], [[4, 3], -2.0]])
    ps = c["processors"].sets[0]
    assert ps.bad_words_ids == ((5, 6), (9,))                                     # HF drops a bad word equal to an eos id
    assert ps.sequence_bias == (((3,), 1.0), ((4, 3), -2.0))


@pytest.mark.parametrize("kw", [dict(no_repeat_ngram_size=1.5), dict(bad_words_ids=[]), dict(bad_words_ids=[[-1]]),
                                dict(sequence_bias=[]), dict(sequence_bias=[[[3], 1]]), dict(min_length=2.5),
                                dict(bad_words_ids=[[5000]]), dict(sequence_bias=[[[5000], 1.0]])])
def test_hf_value_errors(kw):
    with pytest.raises(ValueError):
        _m()._processors(kw)


@pytest.mark.parametrize("kw", [dict(forced_bos_token_id=1), dict(forced_eos_token_id=2), dict(exponential_decay_length_penalty=(2, 1.5)),
                                dict(guidance_scale=2.0), dict(prefix_allowed_tokens_fn=lambda b, ids: [1]), dict(remove_invalid_values=True),
                                dict(renormalize_logits=True), dict(watermarking_config=object()), dict(top_h=0.5),
                                dict(logits_processor=[object()])])
def test_unimplemented_processors_refused(kw):
    m = _m()
    with pytest.raises(NotImplementedError):
        m.generate(**_kw(**kw))
    with pytest.raises(NotImplementedError):
        m.generate_batch([_kw(**kw)])
    with pytest.raises(NotImplementedError):
        list(m.generate_iter([_kw(**kw)]))


def test_beams_and_lookup_with_processors_refused():
    m = _m()
    for extra in (dict(num_beams=2), dict(prompt_lookup_num_tokens=4)):
        with pytest.raises(NotImplementedError):
            m.generate(**_kw(no_repeat_ngram_size=3, **extra))
        with pytest.raises(NotImplementedError):
            m.generate_batch([_kw(no_repeat_ngram_size=3, **extra)])


def test_repetition_penalty_contract_unchanged():
    m = _m()
    assert "processors" not in _call(m, repetition_penalty=1.05)          # greedy ignores it, as before
    with pytest.raises(NotImplementedError):
        m.generate(**_kw(do_sample=True, temperature=0.7, repetition_penalty=1.05))


def test_sampled_path_accepts_no_repeat_ngram():
    c = _call(_m(), do_sample=True, temperature=0.7, no_repeat_ngram_size=3)
    assert c["processors"].sets[0].no_repeat_ngram_size == 3 and c["sampling"] is not None


CHECKS = {  # case: (field edits, expected text)
    "set_range": (dict(seq_set=[2]), "set 2 out of range"),
    "prompt_id": (dict(prompt=[-2000]), "prompt id -2000"),
    "ngram_negative": (dict(ng=[-1]), "must be >= 0"),
    "id_range": (dict(ids=[5, VOCAB]), "out of range [0, 1000)"),
    "bias_nan": (dict(bias=[float("nan")]), "not finite"),
    "empty_sequence": (dict(seq_off=[0, 0]), "sequence 0 is empty"),
    "offsets_decrease": (dict(eos=[1, 0]), "eos_offsets"),
}


@pytest.mark.parametrize("case", sorted(CHECKS))
def test_generate_processors_desc_host_checks(case):
    F, L, E = _lib()
    edits, text = CHECKS[case]
    cfg = E.ModelConfigC()
    cfg.llm_vocab = VOCAB
    m = ctypes.c_void_p()
    assert L.fo1_model_create(ctypes.byref(cfg), ctypes.byref(m)) == 0
    d = E.GenerateDescC()
    d.n_seqs = 1
    d.seq_lens = (ctypes.c_int32 * 1)(3)
    d.max_new_tokens = 4
    f = dict(seq_set=[0], prompt=[1, 2, 3], poff=[0, 3], ng=[2], ml=[0], mn=[0], eos=[0, 1], sup=[1, 1], bsup=[1, 1], bias_off=[0, 1],
             bad_off=[1, 1], seq_off=[1, 2], bias=[0.5], ids=[5, 6])
    f.update(edits)
    i32 = lambda v: (ctypes.c_int32 * len(v))(*v)
    pr = F.ProcessorDesc(1, i32(f["seq_set"]), i32(f["prompt"]), i32(f["poff"]), i32(f["ng"]), i32(f["ml"]), i32(f["mn"]), i32(f["eos"]),
                         i32(f["sup"]), i32(f["bsup"]), i32(f["bias_off"]), i32(f["bad_off"]), len(f["bias"]), i32(f["seq_off"]),
                         (ctypes.c_float * 1)(*f["bias"]), len(f["ids"]), i32(f["ids"]))
    d.processors = ctypes.pointer(pr)
    rc = L.fo1_llm_generate(m, ctypes.byref(d), None)
    msg = L.fo1_last_error().decode()
    assert rc == -1 and "fo1_llm_generate: processors: " in msg and text in msg, (case, rc, msg)
    L.fo1_model_destroy(m)


def test_processor_desc_packs_each_set_and_sequence():
    _, _, E = _lib()
    S = E.ProcessorSet
    a = S(min_length=5, eos_token_ids=(17, 29), suppress_tokens=(3,), bad_words_ids=((4, 5),), sequence_bias=(((7,), 1.0), ((2, 7), -0.5)))
    b = S(begin_suppress_tokens=(9,), bad_words_ids=((11,),))
    d, k = E._processor_desc(E.Processors([a, None, b, a], [[1], [2], [3, 4], [5]]), 4)
    ids, so = list(k["ids"]), list(k["seq_off"])
    seq = lambda i: tuple(ids[so[i]:so[i + 1]])
    lst = lambda key, s: tuple(ids[k[key][s]:k[key][s + 1]])
    assert list(k["seq_set"]) == [0, -1, 1, 0] and d.n_sets == 2                 # equal sets packed once
    assert lst("eos", 0) == (17, 29) and lst("sup", 0) == (3,) and lst("bsup", 1) == (9,) and lst("eos", 1) == ()
    bias_off, bad_off = list(k["bias_off"]), list(k["bad_off"])
    assert [seq(i) for i in range(bias_off[0], bias_off[1])] == [(7,), (2, 7)] and list(k["bias"])[:2] == [1.0, -0.5]
    assert [seq(i) for i in range(bad_off[0], bad_off[1])] == [(4, 5)] and [seq(i) for i in range(bad_off[1], bad_off[2])] == [(11,)]
    assert list(k["prompt"])[:5] == [1, 2, 3, 4, 5] and list(k["poff"]) == [0, 1, 2, 4, 5]


def test_min_new_tokens_takes_precedence_over_min_length():
    """HF's _prepare_generated_length: with min_new_tokens set (even to 0), min_length is replaced by prompt length + min_new_tokens."""
    m = _m(dict(min_length=30, eos_token_id=[7]))
    ps = m._processors(dict(min_new_tokens=2))
    assert ps.min_new_tokens == 2 and ps.min_length == 0 and ps.eos_token_ids == (7,)
    assert m._processors(dict(min_new_tokens=0)) is None
    assert m._processors({}).min_length == 30
