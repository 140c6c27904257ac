"""The object ``load_pretrained_model`` returns in place of the reference's ``OmChatQwen25VLForCausalLM``
(vlm_fo1/model/language_model/omchat_qwen2_5_vl.py:28-41): same ``.config`` attributes the callers read, same
``.generate(**kwargs)`` contract (mm_utils.py:640-654 builds the kwargs; returns LongTensor [1, P + T] whose first P
columns are ``inputs``, or HF's GenerateDecoderOnlyOutput with ``return_dict_in_generate=True``), everything underneath
delegated to the H100 engine."""
from __future__ import annotations

import math
from importlib import import_module
from types import SimpleNamespace
from typing import List, Optional

import torch


# generation_config.json fields of logits processors the engine does not implement, with HF GenerationConfig's neutral defaults.
# On the sampled path a non-neutral value is refused (honour or refuse, never ignore); greedy decoding does not read them.
_UNSUPPORTED_PROCESSORS = (("repetition_penalty", 1.0), ("min_p", None), ("typical_p", 1.0), ("epsilon_cutoff", 0.0),
                           ("eta_cutoff", 0.0), ("num_beams", 1))

# HF logits processors the engine does not implement, with their neutral values: a non-neutral value is refused on every path
_UNIMPLEMENTED_PROCESSORS = (("forced_bos_token_id", None), ("forced_eos_token_id", None), ("exponential_decay_length_penalty", None),
                             ("guidance_scale", 1.0), ("prefix_allowed_tokens_fn", None), ("remove_invalid_values", False),
                             ("renormalize_logits", False), ("watermarking_config", None), ("top_h", None))


class Fo1ForCausalLM:
    def __init__(self, engine, config: SimpleNamespace, vt_mode: str, stop_ids: List[int], roi_size: int = 7, apply_pos_embed: bool = True,
                 generation_config: Optional[dict] = None):
        P = import_module("vlm-fo1_b200.pipeline")
        self.engine = engine
        self.config = config
        self.pipeline = P.Fo1Pipeline(engine, vt_mode=vt_mode, image_token_id=config.image_token_id,
                                      vision_start_token_id=config.vision_start_token_id, video_token_id=config.video_token_id,
                                      roi_size=roi_size, apply_pos_embed=apply_pos_embed)
        self._P = P
        self.default_stop_ids = list(stop_ids)
        self.device = engine.device
        self.dtype = torch.bfloat16
        self.generation_config = dict(generation_config or {})

    # nn.Module-ish no-ops the callers invoke
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def get_model(self):
        return self

    def _sampling_params(self, temperature, top_p, top_k, kwargs):
        """(T, p, k) of a sampled call, validated as HF's warpers validate them; unsupported processors are refused."""
        gc = self.generation_config
        for name, neutral in _UNSUPPORTED_PROCESSORS:
            v = kwargs.get(name, gc.get(name, neutral))
            if v is not None and v != neutral:
                raise NotImplementedError(f"{name}={v!r} is not supported by the fo1-b200 engine's sampled decoding "
                                          "(it implements temperature, top_k and top_p)")
        T = 1.0 if temperature is None else float(temperature)
        if not (T > 0.0) or not math.isfinite(T):
            raise ValueError(f"`temperature` (={temperature}) has to be a strictly positive float when do_sample=True")
        p = 1.0 if top_p is None else float(top_p)
        if not (0.0 < p <= 1.0):
            raise ValueError(f"`top_p` has to be a float in (0, 1], but is {top_p}")
        k = gc.get("top_k", 50) if top_k is None else top_k
        k = 0 if k is None else int(k)
        if k < 0:
            raise ValueError(f"`top_k` has to be a non-negative integer, but is {top_k}")
        return T, p, k

    def _processors(self, kwargs):
        """None (no logits processor: today's path) or the engine.ProcessorSet of a call: sequence_bias, no_repeat_ngram_size,
        bad_words_ids, min_length, min_new_tokens, suppress_tokens and begin_suppress_tokens from the call's kwargs, else
        generation_config.json, validated by transformers' own processor classes (their ValueErrors).  As in HF's generate, a
        min_new_tokens (even 0) overrides min_length: HF sets min_length = prompt length + min_new_tokens.  The eos ids MinLength and
        MinNewTokens mask are HF's: eos_token_id, else the model's default stop ids.  Ids outside the vocabulary in the suppress and
        eos lists are dropped, as HF's isin masks drop them.  HF processors the engine does not implement raise NotImplementedError
        when non-neutral."""
        gc = self.generation_config
        get = lambda name: kwargs[name] if kwargs.get(name) is not None else gc.get(name)
        for name, neutral in _UNIMPLEMENTED_PROCESSORS:
            v = get(name)
            if v is not None and v != neutral:
                raise NotImplementedError(f"{name}={v!r} is not supported by the fo1-b200 engine (its logits processors are sequence_bias, "
                                          "no_repeat_ngram_size, bad_words_ids, min_length, min_new_tokens, suppress_tokens and "
                                          "begin_suppress_tokens)")
        if kwargs.get("logits_processor"):
            raise NotImplementedError("a custom logits_processor list is not supported by the fo1-b200 engine (its processors run on the device)")
        from transformers.generation import logits_process as LP
        E = import_module("vlm-fo1_b200.engine")
        V = self._vocab()
        in_vocab = lambda ids: tuple(int(t) for t in ids if V is None or 0 <= int(t) < V)
        eos = kwargs.get("eos_token_id")
        eos = gc.get("eos_token_id", self.default_stop_ids) if eos is None else eos
        eos = [] if eos is None else ([int(eos)] if isinstance(eos, int) else [int(t) for t in eos])

        def vocab_check(seqs):
            bad = [t for w in seqs for t in w if V is not None and t >= V]
            if bad:
                raise ValueError(f"The model vocabulary size is {V}, but the following tokens were being biased: {bad}")
        f = {}
        ng = get("no_repeat_ngram_size")
        if ng is not None and ng > 0:
            f["no_repeat_ngram_size"] = LP.NoRepeatNGramLogitsProcessor(ng).ngram_size
        sb = get("sequence_bias")
        if sb is not None:
            d = LP.SequenceBiasLogitsProcessor(sequence_bias=sb).sequence_bias
            vocab_check(d)
            f["sequence_bias"] = tuple((tuple(int(t) for t in k), float(v)) for k, v in d.items())
        bw = get("bad_words_ids")
        if bw is not None:
            d = LP.NoBadWordsLogitsProcessor(bw, eos or None).sequence_bias
            vocab_check(d)
            if d:
                f["bad_words_ids"] = tuple(tuple(int(t) for t in k) for k in d)
        ml, mn = get("min_length"), get("min_new_tokens")
        if mn is not None:      # HF's _prepare_generated_length: min_new_tokens takes precedence, min_length becomes P + min_new_tokens
            ml = None
        if ml is not None and eos and ml > 0:
            f["min_length"] = LP.MinLengthLogitsProcessor(ml, eos).min_length
        if mn is not None and eos and mn > 0:
            f["min_new_tokens"] = LP.MinNewTokensLengthLogitsProcessor(0, mn, eos).min_new_tokens
        if "min_length" in f or "min_new_tokens" in f:
            f["eos_token_ids"] = in_vocab(eos)
        for name in ("suppress_tokens", "begin_suppress_tokens"):
            v = get(name)
            if v is not None and in_vocab(v):
                f[name] = in_vocab(v)
        return E.ProcessorSet(**f) if f else None

    def _vocab(self):
        eng = getattr(self, "engine", None)
        return eng.cfg.llm["vocab_size"] if eng is not None else None

    def _outputs(self, kwargs):
        """None (a bare LongTensor, as today) or (output_scores, output_logits) of a return_dict_in_generate call.  Like HF, the
        fields come from the call's kwargs, else from generation_config.json, and only the dict carries them.  Attentions and
        hidden states are refused: the decode loop never materialises them."""
        gc = self.generation_config

        def get(name):
            v = kwargs.get(name)
            return bool(gc.get(name, False) if v is None else v)
        if not get("return_dict_in_generate"):
            return None
        for name in ("output_attentions", "output_hidden_states"):
            if get(name):
                raise NotImplementedError(f"{name}=True is not supported by the fo1-b200 engine's generate (its output dict carries "
                                          "sequences, scores and logits)")
        return get("output_scores"), get("output_logits")

    def _result(self, out, b, inputs, want):
        """Sample b of an engine output -> what generate returns: LongTensor [1, P + n], or the output dict when ``want`` is set."""
        n = int(out["lens"][b])
        new = out["tokens"][b, :n].to(torch.long)
        full = torch.cat([inputs[0].to(new.device), new]).unsqueeze(0)
        if want is None:
            return full
        from transformers.generation.utils import GenerateDecoderOnlyOutput
        rows = lambda key: tuple(out[key][t, b:b + 1] for t in range(n))       # n device views [1, V], the stop token's included
        # past_key_values is None: the K/V cache lives in the engine and is reused by its next call
        return GenerateDecoderOnlyOutput(sequences=full, scores=rows("scores") if want[0] else None,
                                         logits=rows("logits") if want[1] else None, past_key_values=None)

    def compute_transition_scores(self, sequences, scores, beam_indices=None, normalize_logits=False):
        """HF's GenerationMixin.compute_transition_scores without beams: ``scores`` is the tuple generate returned (n tensors
        [batch, V]) -> [batch, n], the score of each generated token (its log-probability with ``normalize_logits``).  V is the
        rows' width (HF reads config.get_text_config(), which this config does not have)."""
        if beam_indices is not None:
            raise NotImplementedError("beam_indices: the fo1-b200 engine has no beam search")
        n, V = len(scores), scores[0].shape[-1]
        stacked = torch.stack(scores).reshape(n, -1).transpose(0, 1)           # [batch * V, n]
        if normalize_logits:
            stacked = torch.nn.functional.log_softmax(stacked.reshape(-1, V, n), dim=1).reshape(-1, n)
        beams = torch.arange(scores[0].shape[0], device=sequences.device).view(-1, 1)
        return stacked.gather(0, sequences[:, sequences.shape[-1] - n:] + beams * V)

    def _sample(self, inputs=None, images=None, images_aux=None, image_grid_thws=None, bbox_list=None, do_sample=False, temperature=0.0,
                stopping_criteria=None, top_p=None, top_k=None, **kwargs):
        """One ``prepare_inputs`` dict -> (SampleInputs, stop ids, (T, p, k) or None): the argument checks of the reference's call
        contract.  do_sample=False is greedy whatever the temperature, as in HF's generate."""
        samp = self._sampling_params(temperature, top_p, top_k, kwargs) if do_sample else None
        if inputs is None or inputs.dim() != 2 or inputs.shape[0] != 1:
            raise ValueError("generate expects `inputs` of shape [1, P] (the reference runs one sample per call)")
        if images is None or len(images) != 1:
            raise ValueError("generate expects exactly one image (the <image> placeholder of the prompt)")
        if images_aux is None:
            raise ValueError("images_aux is required (mm_use_region_index_token checkpoints always provide it)")
        grid = image_grid_thws[0].reshape(-1).tolist()
        boxes = bbox_list[0] if bbox_list else torch.zeros((0, 4))
        aux = images_aux[0]
        sample = self._P.SampleInputs(input_ids=inputs[0].tolist(), pixel_values=images[0], grid_hw=(int(grid[1]), int(grid[2])),
                                      image_aux=aux if aux.dim() == 3 else aux[0], boxes=boxes)
        stop = list(self.default_stop_ids)
        for crit in (stopping_criteria or []):
            for kw in getattr(crit, "keyword_ids", []):
                if kw.numel() == 1:                      # single-token keywords are tested on the device
                    stop.append(int(kw.item()))
                else:
                    # the reference matches the decoded text (mm_utils.py:158-181); a multi-token keyword cannot be tested by
                    # the device-side stop list, and silently ignoring it would change where generation ends
                    raise NotImplementedError(f"multi-token stop keyword {kw.tolist()} is not supported by the device-side stop test "
                                              "(every caller in the reference stops on the single token <|im_end|>)")
        return sample, stop, samp

    def _sampling(self, samps):
        """Per-sample (T, p, k) or None -> engine.Sampling (None when every sample is greedy).  One seed per sampled sample, drawn
        from torch's default CPU generator in sample order; a greedy sample in a sampled batch is top_k = 1 (the arg-max)."""
        if all(s is None for s in samps):
            return None
        E = import_module("vlm-fo1_b200.engine")
        T, P, K, seeds = [], [], [], []
        for s in samps:
            t, p, k = s if s is not None else (1.0, 1.0, 1)
            seeds.append(int(torch.empty((), dtype=torch.int64).random_().item()) if s is not None else 0)
            T.append(t); P.append(p); K.append(k)
        return E.Sampling(T, P, K, seeds)

    def _beams(self, do_sample, kwargs):
        """None (num_beams 1) or the engine.Beams of a beam-search call, from the call's kwargs, else generation_config.json, else
        HF's defaults.  Beam sampling is refused by _sampling_params; group, diverse and constrained beam search here."""
        gc = self.generation_config
        get = lambda name, default: kwargs[name] if kwargs.get(name) is not None else gc.get(name, default)
        N = get("num_beams", 1)
        N = 1 if N is None else int(N)
        if N <= 1 or do_sample:
            return None
        if (get("num_beam_groups", 1) or 1) > 1 or (get("diversity_penalty", 0.0) or 0.0) != 0.0:
            raise NotImplementedError("group / diverse beam search (num_beam_groups, diversity_penalty) is not supported by the fo1-b200 "
                                      "engine (it implements beam search)")
        if get("constraints", None) is not None or get("force_words_ids", None) is not None:
            raise NotImplementedError("constrained beam search (constraints, force_words_ids) is not supported by the fo1-b200 engine")
        n = self._num_return_sequences(kwargs)
        if n > N:
            raise ValueError(f"`num_return_sequences` ({n}) has to be smaller or equal to `num_beams` ({N}).")
        lp = get("length_penalty", 1.0)
        es = get("early_stopping", False)
        if es not in (True, False, "never"):
            raise ValueError(f"`early_stopping` must be a boolean or 'never', but is {es}.")
        E = import_module("vlm-fo1_b200.engine")
        eos = gc.get("eos_token_id", self.default_stop_ids)
        n_eos = len(eos) if isinstance(eos, (list, tuple)) else int(eos is not None)
        return E.Beams(num_beams=N, n_keep=max(2, 1 + n_eos) * N, length_penalty=float(1.0 if lp is None else lp), early_stopping=es,
                       num_return=n)

    def _beam_result(self, out, b, inputs, want, beams, b_local=0):
        """Prompt b of a beam-search engine output -> what HF's generate returns: LongTensor [num_return, P + T] (T: the longest
        returned hypothesis, pad after each one's end) or GenerateBeamDecoderOnlyOutput.  Beam indices are made relative to prompt
        b_local, as a call with that prompt alone returns them."""
        N, nr = beams.num_beams, beams.num_return
        rows = slice(b * nr, (b + 1) * nr)
        lens = out["lens"][rows]
        T = max(int(x) for x in lens)
        new = out["tokens"][rows, :T].to(torch.long)
        full = torch.cat([inputs[0].to(new.device).expand(nr, -1), new], 1)
        if want is None:
            return full
        from transformers.generation.utils import GenerateBeamDecoderOnlyOutput
        steps = int(out["beam_steps"][b])
        block = lambda key: tuple(out[key][t, b * N:(b + 1) * N] for t in range(steps))
        bi = out["beam_indices"][rows, :T]
        bi = torch.where(bi >= 0, bi - (b - b_local) * N, bi)
        return GenerateBeamDecoderOnlyOutput(sequences=full, sequences_scores=out["sequence_scores"][rows] if want[0] else None,
                                             scores=block("scores") if want[0] else None, logits=block("logits") if want[1] else None,
                                             beam_indices=bi, past_key_values=None)

    def _lookup(self, kwargs):
        """None or the engine.Lookup of a prompt-lookup call: ``prompt_lookup_num_tokens`` and ``max_matching_ngram_size`` from the
        call's kwargs, else generation_config.json, as HF reads them; a non-positive value raises HF's ValueError.  The corpus is the
        prompt's ids (the pipeline fills it in).  As in HF, ``num_return_sequences > 1`` with lookup raises ValueError, and with
        ``num_beams > 1`` the kwargs have no effect; a call with a ``streamer`` runs without lookup (same outputs).  Lookup runs on the per-kernel decode path: its tokens are bit-identical to the plain
        per-kernel call (FO1_NO_MEGA=1), and agree with the default persistent-kernel call wherever any two decode paths agree
        (DESIGN.md §2)."""
        gc = self.generation_config
        get = lambda name: kwargs[name] if kwargs.get(name) is not None else gc.get(name)
        K = get("prompt_lookup_num_tokens")
        if K is None:
            return None
        ng = get("max_matching_ngram_size")
        ng = 2 if ng is None else ng
        if int(K) <= 0 or int(ng) <= 0:
            raise ValueError("Invalid max_matching_ngram_size or num_output_tokens")
        E = import_module("vlm-fo1_b200.engine")
        return E.Lookup(num_tokens=int(K), max_ngram=int(ng))

    def _num_return_sequences(self, kwargs):
        n = kwargs.get("num_return_sequences")
        n = self.generation_config.get("num_return_sequences", 1) if n is None else n
        n = 1 if n is None else int(n)
        if n < 1:
            raise ValueError(f"`num_return_sequences` has to be a positive integer, but is {n}")
        return n

    def _results(self, out, inputs, want):
        """The n rows of an engine output as HF returns num_return_sequences: LongTensor [n, P + T_max] padded with the pad id, or the
        output dict with scores / logits as tuples of [n, V] (rows past a sequence's stop are unspecified)."""
        lens = [int(x) for x in out["lens"].cpu().tolist()]
        n, T = len(lens), max(lens)
        new = out["tokens"][:, :T].to(torch.long)                 # pad past each sequence's stop (the engine's pad_id)
        full = torch.cat([inputs.to(new.device).expand(n, -1), new], 1)
        if want is None:
            return full
        from transformers.generation.utils import GenerateDecoderOnlyOutput
        rows = lambda key: tuple(out[key][t] for t in range(T))
        return GenerateDecoderOnlyOutput(sequences=full, scores=rows("scores") if want[0] else None,
                                         logits=rows("logits") if want[1] else None, past_key_values=None)

    @torch.no_grad()
    def generate(self, inputs=None, images=None, images_aux=None, image_grid_thws=None, bbox_list=None, do_sample=False, temperature=0.0,
                 max_new_tokens=512, streamer=None, top_p=1.0, use_cache=True, stopping_criteria=None, pad_token_id=None, top_k=None, **kwargs):
        want = self._outputs(kwargs)
        beams = self._beams(do_sample, kwargs)
        lookup = self._lookup(kwargs)       # (with beams HF only warns and runs beam search; a streamed call runs without lookup)
        procs = self._processors(kwargs)
        n = self._num_return_sequences(kwargs)
        kwargs.pop("num_return_sequences", None)
        if procs is not None and (beams is not None or lookup is not None):
            raise NotImplementedError("logits processors with num_beams > 1 or prompt_lookup_num_tokens are not supported by the fo1-b200 "
                                      "engine (they run on its sampling and greedy paths)")
        E = import_module("vlm-fo1_b200.engine")
        pkw = lambda k: {"processors": E.Processors([procs] * k)} if procs is not None else {}
        if beams is not None:
            if streamer is not None:
                raise ValueError("`streamer` cannot be used with beam search (yet!). Make sure that `num_beams` is set to 1.")
            sample, stop, _ = self._sample(inputs, images, images_aux, image_grid_thws, bbox_list, do_sample, temperature, stopping_criteria,
                                           top_p, top_k, **kwargs)
            out = self.pipeline.generate([sample], int(max_new_tokens), sorted(set(stop)), pad_id=int(self._beam_pad(pad_token_id, stop)),
                                         early_exit_interval=8, want_scores=bool(want and want[0]), want_logits=bool(want and want[1]),
                                         beams=beams)
            return self._beam_result(out, 0, inputs, want, beams)
        if n > 1 and lookup is not None:
            raise ValueError(f"num_return_sequences has to be 1 when doing assisted generate, but is {n}.")
        if n > 1 and not do_sample:
            raise ValueError("Greedy methods without beam search do not support `num_return_sequences` different than 1 "
                             f"(got {n}).")
        if n > 1 and streamer is not None:
            raise ValueError("`streamer` cannot be used with `num_return_sequences` > 1: streamers accept one sequence")
        sample, stop, samp = self._sample(inputs, images, images_aux, image_grid_thws, bbox_list, do_sample, temperature, stopping_criteria,
                                          top_p, top_k, **kwargs)
        pad = pad_token_id if pad_token_id is not None else (stop[0] if stop else 0)
        if n > 1:
            # n copies of the sample share the whole prompt but its last row (the pipeline prefills it once); one seed each
            out = self.pipeline.generate([sample] * n, int(max_new_tokens), sorted(set(stop)), pad_id=int(pad), early_exit_interval=8,
                                         sampling=self._sampling([samp] * n), want_scores=bool(want and want[0]),
                                         want_logits=bool(want and want[1]), **pkw(n))
            return self._results(out, inputs[0], want)
        on_tokens = None
        if streamer is not None:
            # HF's order: the prompt once, then each generated token (the stop token included, pad not) as the device publishes
            # it, then end().  The decode loop stays device-resident: the engine reads the published columns from pinned host
            # memory without a per-token sync.  A streamer error stops the device and propagates, as in HF's generate.
            streamer.put(inputs.cpu())

            def on_tokens(lo, hi, toks, lens):
                for t in range(lo, min(hi, int(lens[0]))):
                    streamer.put(torch.tensor([int(toks[0, t - lo])], dtype=torch.long))
        out = self.pipeline.generate([sample], int(max_new_tokens), sorted(set(stop)), pad_id=int(pad), early_exit_interval=8,
                                     sampling=self._sampling([samp]), want_scores=bool(want and want[0]), want_logits=bool(want and want[1]),
                                     on_tokens=on_tokens, **({"lookup": lookup} if lookup is not None and streamer is None else {}), **pkw(1))
        res = self._result(out, 0, inputs, want)
        if streamer is not None:
            streamer.end()
        return res

    def _beam_pad(self, pad_token_id, stop):
        """HF's beam-search fill value: ``pad_token_id or eos_token_id[0]``."""
        eos = self.generation_config.get("eos_token_id", self.default_stop_ids)
        eos = list(eos) if isinstance(eos, (list, tuple)) else ([eos] if eos is not None else list(stop))
        return pad_token_id or (eos[0] if eos else 0)

    @torch.no_grad()
    def generate_batch(self, batch, max_new_tokens=None, output_logprobs=False):
        """``batch``: a list of the dicts ``prepare_inputs`` returns (one sample each, mm_utils.py:640-654).  All samples run as ONE
        packed batch through the engine (what the reference's evaluation loops do one image at a time, eval_coco.py:36-88).
        -> list of LongTensor [1, P_b + T_b], each exactly what ``generate(**batch[b])`` returns (the output dict where that dict
        asks for it).  ``output_logprobs``: each element is (that, fp32 [1, n_b]), the log-probability of each generated token
        computed on the device, with no vocabulary-wide rows."""
        if not batch:
            return []
        wants = [self._outputs(kw) for kw in batch]
        beams = [self._beams(kw.get("do_sample", False), kw) for kw in batch]
        procs = [self._processors(kw) for kw in batch]
        if any(p is not None for p in procs) and (any(b is not None for b in beams) or any(self._lookup(kw) is not None for kw in batch)):
            raise NotImplementedError("logits processors with num_beams > 1 or prompt_lookup_num_tokens are not supported by the fo1-b200 "
                                      "engine (they run on its sampling and greedy paths)")
        if any(b is not None for b in beams):
            return self._generate_batch_beams(batch, beams, wants, max_new_tokens, output_logprobs)
        if any(self._num_return_sequences(kw) != 1 for kw in batch):
            raise NotImplementedError("num_return_sequences > 1 in generate_batch: call generate for such a sample, or repeat it in the batch")
        keys = ("inputs", "images", "images_aux", "image_grid_thws", "bbox_list", "do_sample", "temperature", "stopping_criteria", "top_p",
                "top_k") + tuple(n for n, _ in _UNSUPPORTED_PROCESSORS)
        samples, stops, samps = zip(*(self._sample(**{k: v for k, v in kw.items() if k in keys}) for kw in batch))
        stop = sorted(set(x for s in stops for x in s))
        T = int(max_new_tokens if max_new_tokens is not None else max(int(kw.get("max_new_tokens", 512)) for kw in batch))
        pads = [kw.get("pad_token_id") for kw in batch]
        pad = pads[0] if pads[0] is not None else (stop[0] if stop else 0)
        sampling = self._sampling(samps)
        lookups = [self._lookup(kw) for kw in batch]
        if any(lk != lookups[0] for lk in lookups):
            raise NotImplementedError("generate_batch runs prompt lookup as one call: every sample must use the same "
                                      "prompt_lookup_num_tokens and max_matching_ngram_size (call generate for the others)")
        # a greedy sample in a sampled batch is scored on its raw logits, as HF's greedy search reports them
        raw = [int(s is None) for s in samps] if sampling is not None else None
        out = self.pipeline.generate(list(samples), T, stop, pad_id=int(pad), early_exit_interval=8, sampling=sampling,
                                     want_logprobs=bool(output_logprobs), want_scores=any(w is not None and w[0] for w in wants),
                                     want_logits=any(w is not None and w[1] for w in wants), raw_rows=raw,
                                     **({"lookup": lookups[0]} if lookups[0] is not None else {}),
                                     **({"processors": import_module("vlm-fo1_b200.engine").Processors(procs)}
                                        if any(p is not None for p in procs) else {}))
        out["lens"] = out["lens"].cpu().tolist()
        res = []
        for b, kw in enumerate(batch):
            r = self._result(out, b, kw["inputs"], wants[b])
            res.append((r, out["logprobs"][b:b + 1, :out["lens"][b]]) if output_logprobs else r)
        return res

    @torch.no_grad()
    def generate_iter(self, kwargs_iterable, batch_size=16, on_error=None):
        """In-flight batching: the dicts ``prepare_inputs`` returns (as ``generate_batch`` takes them) through ``batch_size`` decode
        slots; a finished sample hands its slot to the next one.  Yields (i, LongTensor [1, P_i + T_i]) in completion order, each
        honouring its own ``max_new_tokens`` as ``generate(**kw)`` does, and equal to that sample's row in a static batch of
        ``batch_size`` samples on the same decode path (at most 8 slots on the persistent kernel: ``generate(**kw)`` alone).  Seeds
        are drawn from torch's generator in sample order.  ``on_error(i, exception)``: a sample whose admission fails is reported
        there and skipped (without it the exception propagates).  Logits processors are honoured per sample.  Scores, streaming,
        beams, prompt lookup and num_return_sequences > 1 are refused with NotImplementedError."""
        batch = list(kwargs_iterable)
        if not batch:
            return
        for kw in batch:
            if self._outputs(kw) is not None:
                raise NotImplementedError("return_dict_in_generate is not supported by generate_iter (it returns token ids)")
            if kw.get("streamer") is not None:
                raise NotImplementedError("streamer is not supported by generate_iter")
            if self._beams(kw.get("do_sample", False), kw) is not None or int(kw.get("num_beams") or 1) > 1:
                raise NotImplementedError("num_beams > 1 is not supported by generate_iter")
            if self._lookup(kw) is not None:
                raise NotImplementedError("prompt_lookup_num_tokens is not supported by generate_iter")
            if self._num_return_sequences(kw) != 1:
                raise NotImplementedError("num_return_sequences > 1 is not supported by generate_iter")
        procs = [self._processors(kw) for kw in batch]
        keys = ("inputs", "images", "images_aux", "image_grid_thws", "bbox_list", "do_sample", "temperature", "stopping_criteria", "top_p",
                "top_k") + tuple(n for n, _ in _UNSUPPORTED_PROCESSORS)
        samples, stops, samps = zip(*(self._sample(**{k: v for k, v in kw.items() if k in keys}) for kw in batch))
        stop = sorted(set(x for s in stops for x in s))
        pads = [kw.get("pad_token_id") for kw in batch]
        pad = pads[0] if pads[0] is not None else (stop[0] if stop else 0)
        mnt = [int(kw.get("max_new_tokens", 512)) for kw in batch]
        for i, tokens, n in self.pipeline.generate_continuous(list(samples), int(batch_size), mnt, stop, pad_id=int(pad), early_exit_interval=8,
                                                             sampling=self._sampling(samps), on_error=on_error,
                                                             **({"processors": import_module("vlm-fo1_b200.engine").Processors(procs)}
                                                                if any(p is not None for p in procs) else {})):
            inputs = batch[i]["inputs"]
            yield i, torch.cat([inputs[0].to(tokens.device), tokens.to(torch.long)]).unsqueeze(0)

    # ---- teacher-forced scoring (the reference's forward(labels=...), omchat_qwen2_5_vl.py:466-532) ----
    def _score_sample(self, input_ids, images, images_aux, image_grid_thws, bbox_list, labels):
        """(SampleInputs, label list) of one forward-style call; labels None: nothing scored."""
        sample, _, _ = self._sample(input_ids, images, images_aux, image_grid_thws, bbox_list)
        if labels is None:
            lab = [-100] * len(sample.input_ids)
        else:
            labels = torch.as_tensor(labels)
            if labels.dim() == 2:
                if labels.shape[0] != 1:
                    raise ValueError("labels must be [1, P] like input_ids (the reference runs one sample per call)")
                labels = labels[0]
            lab = [int(x) for x in labels.tolist()]
            if len(lab) != len(sample.input_ids):
                raise ValueError(f"labels has {len(lab)} positions, input_ids {len(sample.input_ids)}")
        return sample, lab

    @torch.no_grad()
    def forward(self, input_ids=None, images=None, images_aux=None, image_grid_thws=None, bbox_list=None, labels=None, attention_mask=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None, **kwargs):
        """The reference's forward for one sample: -> transformers' Qwen2_5_VLCausalLMOutputWithPast with ``logits`` fp32 [1, L, V] at
        every spliced position (the engine's all_logits), ``loss`` HF's ForCausalLMLoss over ``labels`` (the mean over every
        non-ignored shifted label, NaN when none is; None without labels) from the device's per-token log-likelihoods,
        ``rope_deltas`` [1, 1] and ``past_key_values`` None.  No K/V cache in or out, attentions, hidden states or tuple returns."""
        if past_key_values is not None:
            raise NotImplementedError("forward with past_key_values is not supported by the fo1-b200 engine (its K/V cache stays inside it)")
        if inputs_embeds is not None:
            raise NotImplementedError("forward with inputs_embeds is not supported by the fo1-b200 engine (it splices input_ids itself)")
        for name, v in (("output_attentions", output_attentions), ("output_hidden_states", output_hidden_states)):
            if v:
                raise NotImplementedError(f"{name}=True is not supported by the fo1-b200 engine's forward (it returns loss and logits)")
        if return_dict is False:
            raise NotImplementedError("return_dict=False is not supported by the fo1-b200 engine's forward (it returns the output dataclass)")
        if attention_mask is not None and not bool(torch.as_tensor(attention_mask).bool().all()):
            raise NotImplementedError("a padded attention_mask is not supported by the fo1-b200 engine's forward (one unpadded sample)")
        sample, lab = self._score_sample(input_ids, images, images_aux, image_grid_thws, bbox_list, labels)
        out = self.pipeline.score([sample], [lab], want_all_logits=True)
        from transformers.models.qwen2_5_vl.modeling_qwen2_5_vl import Qwen2_5_VLCausalLMOutputWithPast
        loss = None
        if labels is not None:
            loss = (-out["seq_logprob"].sum() / out["seq_count"].sum().to(torch.float64)).to(torch.float32)
        return Qwen2_5_VLCausalLMOutputWithPast(loss=loss, logits=out["all_logits"].unsqueeze(0), past_key_values=None,
                                                rope_deltas=out["rope_delta"].to(torch.long).view(1, 1))

    __call__ = forward

    @torch.no_grad()
    def score_batch(self, batch, labels):
        """Scoring of many samples in ONE engine call without any logits matrix (what ``generate_batch`` is for ``generate``).
        ``batch``: the dicts ``prepare_inputs`` returns; ``labels[b]``: [1, P_b] or a list over sample b's input_ids (-100 ignored).
        Samples about the same image share the towers and their common prompt prefix.  -> per sample a dict: ``loss`` (fp32 scalar,
        forward's loss), ``logprobs`` fp32 [n_b] (the log-probability of each non-ignored shifted label, in order) and ``greedy``
        int32 [n_b] (1 where that label is the arg-max)."""
        if len(labels) != len(batch):
            raise ValueError("one label sequence per sample")
        keys = ("inputs", "images", "images_aux", "image_grid_thws", "bbox_list")
        pairs = [self._score_sample(*(kw.get(k) for k in keys), lab) for kw, lab in zip(batch, labels)]
        out = self.pipeline.score([p[0] for p in pairs], [p[1] for p in pairs], want_greedy=True)
        scored = torch.from_numpy(out["targets"] != -100)
        off = [0]
        for n in out["prompt_lens"]:
            off.append(off[-1] + n)
        res = []
        for b in range(len(batch)):
            sel = torch.nonzero(scored[off[b]:off[b + 1]]).view(-1).to(out["logprobs"].device) + off[b]
            loss = (-out["seq_logprob"][b] / out["seq_count"][b].to(torch.float64)).to(torch.float32)
            res.append(dict(loss=loss, logprobs=out["logprobs"][sel], greedy=out["greedy"][sel]))
        return res

    def _generate_batch_beams(self, batch, beams, wants, max_new_tokens, output_logprobs):
        """generate_batch of beam-search samples: one packed engine call when every sample asks for the same beam setting.  With
        ``output_logprobs`` each element carries fp32 [num_return, T], the returned tokens' log-probabilities gathered along their
        beam paths on the device (HF's compute_transition_scores(sequences, scores, beam_indices), 0 past each hypothesis' end)."""
        if any(b != beams[0] for b in beams):
            raise NotImplementedError("generate_batch runs beam search as one call: every sample must use the same num_beams, "
                                      "length_penalty, early_stopping and num_return_sequences (call generate for the others)")
        keys = ("inputs", "images", "images_aux", "image_grid_thws", "bbox_list", "do_sample", "temperature", "stopping_criteria", "top_p",
                "top_k") + tuple(n for n, _ in _UNSUPPORTED_PROCESSORS)
        samples, stops, _ = zip(*(self._sample(**{k: v for k, v in kw.items() if k in keys}) for kw in batch))
        stop = sorted(set(x for s in stops for x in s))
        T = int(max_new_tokens if max_new_tokens is not None else max(int(kw.get("max_new_tokens", 512)) for kw in batch))
        pad = self._beam_pad(batch[0].get("pad_token_id"), stop)
        out = self.pipeline.generate(list(samples), T, stop, pad_id=int(pad), early_exit_interval=8, want_logprobs=bool(output_logprobs),
                                     want_scores=any(w is not None and w[0] for w in wants),
                                     want_logits=any(w is not None and w[1] for w in wants), beams=beams[0])
        nr = beams[0].num_return
        res = []
        for b, kw in enumerate(batch):
            r = self._beam_result(out, b, kw["inputs"], wants[b], beams[0])
            if output_logprobs:
                width = int(out["lens"][b * nr:(b + 1) * nr].max())
                r = (r, out["logprobs"][b * nr:(b + 1) * nr, :width])
            res.append(r)
        return res
