"""CPU: the argument handling of beam search -- fo1_llm_generate's host checks of d.beam, which run before any CUDA call, and
Fo1ForCausalLM.generate / generate_batch's reading of num_beams, length_penalty, early_stopping and num_return_sequences, with
HF's refusals.  The model tests record the pipeline call instead of running it."""
import ctypes
from importlib import import_module

import pytest
import torch

VOCAB = 1000


def _lib():
    import fo1_b200
    return fo1_b200._lib, fo1_b200.lib(), import_module("vlm-fo1_b200.engine")


BEAM_CASES = {  # case: (field overrides, expected text)
    "one_beam": (dict(num_beams=1), "num_beams 1"),
    "too_many_beams": (dict(num_beams=17, n_keep=34, num_return=1), "num_beams 17"),
    "return_zero": (dict(num_return=0), "num_return 0"),
    "return_above_beams": (dict(num_return=5), "num_return 5"),
    "keep_below_2n": (dict(n_keep=7), "n_keep 7"),
    "keep_above_limit": (dict(n_keep=129), "n_keep 129"),
    "keep_above_vocab": (dict(num_beams=16, n_keep=128, num_return=1), None),      # with a 100-token vocabulary below
    "lp_nan": (dict(length_penalty=float("nan")), "length_penalty"),
    "lp_inf": (dict(length_penalty=float("inf")), "length_penalty"),
    "early_stopping_3": (dict(early_stopping=3), "early_stopping 3"),
    "max_new_zero": ({}, "max_new_tokens 0"),
    "all_logits": ({}, "all_logits"),
    "null_scores": (dict(sequence_scores=None), "null output"),
    "null_beam_indices": (dict(beam_indices=None), "null output"),
    "null_steps": (dict(steps_run=None), "null output"),
    "null_tokens": ({}, "null output"),
}


@pytest.mark.parametrize("case", sorted(BEAM_CASES))
def test_generate_beam_desc_validation_without_gpu(case):
    F, L, E = _lib()
    over, text = BEAM_CASES[case]
    cfg = E.ModelConfigC()
    cfg.llm_vocab = 100 if case == "keep_above_vocab" else VOCAB
    m = ctypes.c_void_p()
    assert L.fo1_model_create(ctypes.byref(cfg), ctypes.byref(m)) == 0     # host only
    d = E.GenerateDescC()
    d.n_seqs = 2
    d.max_new_tokens = 0 if case == "max_new_zero" else 8
    d.out_tokens, d.out_lens = (None if case == "null_tokens" else 16), 16
    if case == "all_logits":
        d.all_logits = 16
    f = dict(num_beams=4, n_keep=8, length_penalty=1.0, early_stopping=0, num_return=2, sequence_scores=16, beam_indices=16, steps_run=16,
             scores=None, logits=None, logprobs=None)
    f.update(over)
    bm = F.BeamDesc(**f)
    d.beam = ctypes.pointer(bm)
    rc = L.fo1_llm_generate(m, ctypes.byref(d), None)
    msg = L.fo1_last_error().decode()
    assert rc == -1, (case, rc, msg)
    assert "fo1_llm_generate: beam: " in msg and (text is None or text in msg), msg
    if case == "keep_above_vocab":
        assert "vocab 100" in msg
    L.fo1_model_destroy(m)


def test_generate_with_beam_null_model():
    F, L, E = _lib()
    d = E.GenerateDescC()
    bm = F.BeamDesc(num_beams=4, n_keep=8, num_return=1)
    d.beam = ctypes.pointer(bm)
    assert L.fo1_llm_generate(None, ctypes.byref(d), None) == -1
    assert "null argument" in L.fo1_last_error().decode()


def test_beams_early_stopping_codes():
    _, _, E = _lib()
    assert [E.Beams(2, 4, early_stopping=v).code() for v in (False, True, "never")] == [0, 1, 2]
    with pytest.raises(ValueError):
        E.Beams(2, 4, early_stopping="always").code()


# ---------------------------------------------------------------------------------------------------------------- Fo1ForCausalLM
class _Recorder:
    def __init__(self):
        self.calls = []

    def generate(self, samples, max_new_tokens, stop_ids, **kw):
        self.calls.append(dict(n=len(samples), max_new_tokens=max_new_tokens, stop_ids=list(stop_ids), **kw))
        raise _Stop()


class _Stop(Exception):
    pass


def _model(generation_config=None, stop_ids=(151645, 151643)):
    M = import_module("vlm_fo1.model.fo1_model")
    m = M.Fo1ForCausalLM.__new__(M.Fo1ForCausalLM)
    m._P = import_module("vlm-fo1_b200.pipeline")
    m.pipeline = _Recorder()
    m.default_stop_ids = list(stop_ids)
    m.generation_config = dict(generation_config or {})
    return m


def _kw(**extra):
    kw = dict(inputs=torch.tensor([[1, 2, 3]]), images=[torch.zeros(4, 8)], images_aux=[torch.zeros(3, 16, 16)],
              image_grid_thws=torch.tensor([[1, 2, 2]]), bbox_list=[torch.zeros(0, 4)], max_new_tokens=5)
    kw.update(extra)
    return kw


def _call(m, **kw):
    with pytest.raises(_Stop):
        m.generate(**_kw(**kw))
    return m.pipeline.calls[-1]


def test_greedy_num_beams_1_is_the_old_call():
    m = _model()
    plain = _call(m)
    one = _call(m, num_beams=1)
    assert plain == one
    assert "beams" not in plain and plain["sampling"] is None


def test_beam_call_reads_kwargs_then_generation_config():
    m = _model(dict(num_beams=4, length_penalty=0.5, early_stopping="never", eos_token_id=[151645, 151643]))
    c = _call(m)
    b = c["beams"]
    assert (b.num_beams, b.n_keep, b.length_penalty, b.early_stopping, b.num_return) == (4, 12, 0.5, "never", 1)
    c = _call(m, num_beams=2, length_penalty=2.0, early_stopping=True, num_return_sequences=2)
    b = c["beams"]
    assert (b.num_beams, b.n_keep, b.length_penalty, b.early_stopping, b.num_return) == (2, 6, 2.0, True, 2)
    assert c["pad_id"] == 151645                      # HF: pad_token_id or eos_token_id[0]
    c = _call(_model(), num_beams=3)
    assert c["beams"].n_keep == 9 and c["beams"].length_penalty == 1.0 and c["beams"].early_stopping is False


@pytest.mark.parametrize("extra,exc,text", [
    (dict(do_sample=True, num_beams=2), NotImplementedError, "num_beams"),
    (dict(num_beams=2, streamer=object()), ValueError, "`streamer` cannot be used with beam search"),
    (dict(num_beams=2, num_return_sequences=3), ValueError, "has to be smaller or equal to `num_beams`"),
    (dict(num_beams=4, num_beam_groups=2), NotImplementedError, "num_beam_groups"),
    (dict(num_beams=4, diversity_penalty=0.5), NotImplementedError, "diversity_penalty"),
    (dict(num_beams=4, constraints=[object()]), NotImplementedError, "constraints"),
    (dict(num_beams=4, early_stopping="sometimes"), ValueError, "early_stopping"),
])
def test_beam_refusals(extra, exc, text):
    m = _model()
    with pytest.raises(exc, match=text.replace("(", r"\(").replace("`", "`")):
        m.generate(**_kw(**extra))
    assert m.pipeline.calls == []


def test_generate_batch_needs_one_beam_setting():
    m = _model()
    with pytest.raises(NotImplementedError, match="same num_beams"):
        m.generate_batch([_kw(num_beams=2), _kw(num_beams=4)])
    with pytest.raises(NotImplementedError, match="same num_beams"):
        m.generate_batch([_kw(num_beams=2), _kw()])
    with pytest.raises(_Stop):
        m.generate_batch([_kw(num_beams=2), _kw(num_beams=2)])
    c = m.pipeline.calls[-1]
    assert c["n"] == 2 and c["beams"].num_beams == 2
