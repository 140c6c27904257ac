"""CPU: the argument handling of prompt-lookup decoding -- fo1_llm_generate's host checks of d.lookup, which run before any CUDA call,
and Fo1ForCausalLM.generate / generate_batch's reading of prompt_lookup_num_tokens and max_matching_ngram_size.  The model tests
record the pipeline call instead of running it (tests/test_beam_args.py)."""
import ctypes

import pytest

from tests.test_beam_args import _Stop, _call, _kw, _lib, _model

VOCAB = 1000

LOOKUP_CASES = {  # case: (num_tokens, max_ngram, offsets, corpus present, expected text)
    "num_tokens_0": (0, 2, [0, 1, 2], True, "num_tokens 0"),
    "max_ngram_0": (4, 0, [0, 1, 2], True, "max_ngram 0"),
    "offsets_null": (4, 2, None, True, "null corpus_offsets"),
    "offsets_start": (4, 2, [1, 1, 2], True, "corpus_offsets[0] = 1"),
    "offsets_decrease": (4, 2, [0, 2, 1], True, "decrease at sequence 1"),
    "corpus_null": (4, 2, [0, 1, 2], False, "null corpus"),
}


@pytest.mark.parametrize("case", sorted(LOOKUP_CASES))
def test_generate_lookup_desc_validation_without_gpu(case):
    F, L, E = _lib()
    K, ng, offs, has_corpus, text = LOOKUP_CASES[case]
    cfg = E.ModelConfigC()
    cfg.llm_vocab = VOCAB
    m = ctypes.c_void_p()
    assert L.fo1_model_create(ctypes.byref(cfg), ctypes.byref(m)) == 0     # host only
    d = E.GenerateDescC()
    d.n_seqs = 2
    d.seq_lens = (ctypes.c_int32 * 2)(3, 3)
    d.max_new_tokens = 8
    ids = (ctypes.c_int32 * 2)(5, 6)
    off = (ctypes.c_int32 * 3)(*offs) if offs is not None else None
    lk = F.LookupDesc(K, ng, ids if has_corpus else None, off, None, None)
    d.lookup = ctypes.pointer(lk)
    rc = L.fo1_llm_generate(m, ctypes.byref(d), None)
    msg = L.fo1_last_error().decode()
    assert rc == -1, (case, rc, msg)
    assert "fo1_llm_generate: lookup: " in msg and text in msg, msg
    L.fo1_model_destroy(m)


def test_lookup_drafts_checks_without_gpu():
    F, L, E = _lib()
    for K, ng, text in ((0, 2, "num_tokens 0"), (17, 2, "num_tokens 17"), (4, 0, "max_ngram 0")):
        assert L.fo1_lookup_drafts(16, 4, 16, 1, K, ng, None, 0, None, 0, 16, 16, None) == -1
        assert text in L.fo1_last_error().decode()


def test_kwargs_then_generation_config():
    m = _model()
    plain = _call(m)
    assert "lookup" not in plain
    c = _call(m, prompt_lookup_num_tokens=10)
    assert (c["lookup"].num_tokens, c["lookup"].max_ngram, c["lookup"].corpus) == (10, 2, None)
    c = _call(m, prompt_lookup_num_tokens=3, max_matching_ngram_size=4)
    assert (c["lookup"].num_tokens, c["lookup"].max_ngram) == (3, 4)
    m = _model(generation_config=dict(prompt_lookup_num_tokens=5, max_matching_ngram_size=1))
    c = _call(m)
    assert (c["lookup"].num_tokens, c["lookup"].max_ngram) == (5, 1)
    c = _call(m, prompt_lookup_num_tokens=7)
    assert (c["lookup"].num_tokens, c["lookup"].max_ngram) == (7, 1)


@pytest.mark.parametrize("extra", [dict(prompt_lookup_num_tokens=0), dict(prompt_lookup_num_tokens=-1),
                                   dict(prompt_lookup_num_tokens=4, max_matching_ngram_size=0)])
def test_non_positive_raises_hf_value_error(extra):
    with pytest.raises(ValueError, match="Invalid max_matching_ngram_size or num_output_tokens"):
        _model().generate(**_kw(**extra))


def test_beams_and_streamer_leave_the_call_as_today():
    m = _model()
    assert _call(m, num_beams=2, prompt_lookup_num_tokens=4) == _call(m, num_beams=2)

    class S:
        def put(self, x):
            pass

        def end(self):
            pass
    a = _call(m, streamer=S(), prompt_lookup_num_tokens=4)
    b = _call(m, streamer=S())
    a.pop("on_tokens"); b.pop("on_tokens")
    assert a == b


def test_generate_batch_one_lookup_setting():
    m = _model()
    with pytest.raises(_Stop):
        m.generate_batch([_kw(prompt_lookup_num_tokens=4), _kw(prompt_lookup_num_tokens=4)])
    assert m.pipeline.calls[-1]["lookup"].num_tokens == 4 and m.pipeline.calls[-1]["n"] == 2
    with pytest.raises(NotImplementedError, match="prompt_lookup_num_tokens"):
        m.generate_batch([_kw(prompt_lookup_num_tokens=4), _kw()])


def test_num_return_sequences_with_lookup_raises_hf_value_error():
    with pytest.raises(ValueError, match="num_return_sequences has to be 1 when doing assisted generate"):
        _model().generate(**_kw(prompt_lookup_num_tokens=4, num_return_sequences=2, do_sample=True, temperature=0.7))
