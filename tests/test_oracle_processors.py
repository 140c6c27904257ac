"""CPU: oracle/processors.py against transformers' own logits processors, as GenerationMixin._get_logits_processor builds them from a
GenerationConfig, and the oracle's greedy loop against HF's real greedy generate on a tiny random Qwen2ForCausalLM."""
from importlib import import_module

import pytest
import torch

from oracle import processors as O

V = 64
PROMPT_LEN = 12


def _set(**kw):
    return import_module("vlm-fo1_b200.engine").ProcessorSet(**kw)


def _tiny():
    from transformers import Qwen2Config, Qwen2ForCausalLM
    torch.manual_seed(0)
    cfg = Qwen2Config(vocab_size=V, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                      max_position_embeddings=256)
    return Qwen2ForCausalLM(cfg).eval()


def _hf_list(model, gc_kw, prompt_len):
    from transformers import GenerationConfig
    gc = GenerationConfig(**gc_kw)
    gc._eos_token_tensor = torch.tensor(gc_kw.get("eos_token_id", [5, 6]) if isinstance(gc_kw.get("eos_token_id", [5, 6]), list)
                                        else [gc_kw["eos_token_id"]])
    return model._get_logits_processor(generation_config=gc, input_ids_seq_length=prompt_len, encoder_input_ids=None,
                                       prefix_allowed_tokens_fn=None, logits_processor=None, device="cpu")


# (HF generation-config kwargs, the same as a ProcessorSet, history)
CASES = {
    "ngram_in_prompt": (dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=2), [1, 2, 3, 1, 2, 4, 9, 8, 7, 3, 2, 1]),
    "ngram_across_boundary": (dict(no_repeat_ngram_size=3), dict(no_repeat_ngram_size=3),
                              [7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 3, 7, 8, 9, 3, 7]),
    "ngram_1": (dict(no_repeat_ngram_size=1), dict(no_repeat_ngram_size=1), list(range(20, 32)) + [40]),
    "ngram_negative_placeholder": (dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=2),
                                   [3, -20, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 3, -20, 4, 3]),
    "bad_words": (dict(bad_words_ids=[[9], [3, 4], [4, 5, 6], [5, 6, 7], [2, 3]]),
                  dict(bad_words_ids=((9,), (3, 4), (4, 5, 6), (5, 6, 7), (2, 3))), [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 4, 5, 6, 2]),
    "sequence_bias": (dict(sequence_bias=[[[7], 1.5], [[2, 7], -0.25], [[1, 2, 7], 3.0], [[3], -2.0], [[8, 3], 0.125]]),
                      dict(sequence_bias=(((7,), 1.5), ((2, 7), -0.25), ((1, 2, 7), 3.0), ((3,), -2.0), ((8, 3), 0.125))),
                      [9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 9, 1, 2]),
    "min_length_below": (dict(min_length=14), dict(min_length=14, eos_token_ids=(5, 6)), list(range(13))),
    "min_length_at": (dict(min_length=13), dict(min_length=13, eos_token_ids=(5, 6)), list(range(13))),
    "min_new_below": (dict(min_new_tokens=2), dict(min_new_tokens=2, eos_token_ids=(5, 6)), list(range(13))),
    "min_new_at": (dict(min_new_tokens=1), dict(min_new_tokens=1, eos_token_ids=(5, 6)), list(range(13))),
    "suppress": (dict(suppress_tokens=[1, 2, 63]), dict(suppress_tokens=(1, 2, 63)), list(range(14))),
    "begin_suppress_col0": (dict(begin_suppress_tokens=[4, 5]), dict(begin_suppress_tokens=(4, 5)), list(range(12))),
    "begin_suppress_col1": (dict(begin_suppress_tokens=[4, 5]), dict(begin_suppress_tokens=(4, 5)), list(range(13))),
    "all": (dict(no_repeat_ngram_size=2, bad_words_ids=[[3, 4], [11]], sequence_bias=[[[4], 0.5], [[2, 4], 1.0]], min_length=30,
                 min_new_tokens=5, suppress_tokens=[0], begin_suppress_tokens=[1]),
            dict(no_repeat_ngram_size=2, bad_words_ids=((3, 4), (11,)), sequence_bias=(((4,), 0.5), ((2, 4), 1.0)), min_length=30,
                 min_new_tokens=5, suppress_tokens=(0,), begin_suppress_tokens=(1,), eos_token_ids=(5, 6)),
            [1, 2, 3, 4, 2, 3, 1, 2, 3, 9, 10, 11, 2, 3]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_equals_hf_processors(case):
    model = _tiny()
    gc_kw, ps_kw, hist = CASES[case]
    hf = _hf_list(model, dict(gc_kw, eos_token_id=[5, 6]), PROMPT_LEN)
    ps = _set(**ps_kw)
    g = torch.Generator().manual_seed(len(case))
    for trial in range(4):
        row = torch.randn((1, V), generator=g) * 4
        ref = hf(torch.tensor([hist]), row.clone())[0]
        got = O.process(row[0], hist, PROMPT_LEN, ps)
        assert torch.equal(got, ref), (case, trial)


def test_oracle_greedy_loop_equals_hf_generate():
    model = _tiny()
    prompt = [3, 7, 7, 1, 2, 3, 4, 9, 9, 10]
    gc_kw = dict(no_repeat_ngram_size=2, bad_words_ids=[[12], [7, 1]], min_new_tokens=4, suppress_tokens=[0], sequence_bias=[[[2], -1.0]])
    with torch.no_grad():
        out = model.generate(torch.tensor([prompt]), attention_mask=torch.ones((1, len(prompt)), dtype=torch.long), do_sample=False,
                             max_new_tokens=12, eos_token_id=[5, 6], pad_token_id=0, **gc_kw)
    hf = out[0, len(prompt):].tolist()
    ps = _set(no_repeat_ngram_size=2, bad_words_ids=((12,), (7, 1)), min_new_tokens=4, suppress_tokens=(0,), sequence_bias=(((2,), -1.0),),
              eos_token_ids=(5, 6))

    def step(ids):
        with torch.no_grad():
            return model(torch.tensor([ids])).logits[0, -1].float()
    ours = O.greedy_loop(step, prompt, ps, 12, eos_ids=(5, 6))
    assert ours == hf[:len(ours)] and (len(ours) == len(hf) or all(t == 0 for t in hf[len(ours):]))


def _model_with(gc):
    from types import SimpleNamespace

    from tests.test_beam_args import _model
    m = _model(generation_config=gc)
    m.engine = SimpleNamespace(cfg=SimpleNamespace(llm={"vocab_size": V}))
    return m


@pytest.mark.parametrize("kw", [dict(min_length=30, min_new_tokens=2), dict(min_length=30, min_new_tokens=0), dict(min_length=30),
                                dict(min_new_tokens=5)])
def test_min_lengths_through_the_kwargs_equal_hf_generate(kw):
    """Fo1ForCausalLM._processors' reading of min_length / min_new_tokens (min_new_tokens takes precedence, HF's
    _prepare_generated_length), run through the oracle's greedy loop, against HF's real generate."""
    model = _tiny()
    prompt = [3, 7, 7, 1, 2, 3, 4, 9, 9, 10]

    def step(ids):
        with torch.no_grad():
            return model(torch.tensor([ids])).logits[0, -1].float()
    plain = O.greedy_loop(step, prompt, _set(), 8)
    eos = plain[3]                      # the plain run emits this at column 3: the min lengths decide whether it stops there
    with torch.no_grad():
        out = model.generate(torch.tensor([prompt]), attention_mask=torch.ones((1, len(prompt)), dtype=torch.long), do_sample=False,
                             max_new_tokens=12, eos_token_id=[eos], pad_token_id=0, **kw)
    hf = out[0, len(prompt):].tolist()
    ps = _model_with(dict(eos_token_id=[eos]))._processors(dict(kw))
    ours = O.greedy_loop(step, prompt, ps if ps is not None else _set(), 12, eos_ids=(eos,))
    assert ours == hf[:len(ours)] and all(t == 0 for t in hf[len(ours):]), (ours, hf)
