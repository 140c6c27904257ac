"""Host-side mirror of the reference's multimodal forward for a BATCH of samples, over the engine:

    encode_images   (omchat_qwen2_5_vl.py:44-72)   -> Engine.vit_forward      (one packed launch sequence)
    encode_regions  (omchat_qwen2_5_vl.py:75-128)  -> Engine.davit_forward + fpn_forward + hfre_forward + region_project
    splice + M-RoPE (omchat_qwen2_5_vl.py:291-463) -> splice_plan (host ints) + Engine.build_embeds
    generate        (HF greedy loop)               -> Engine.generate (prefill + device-resident decode)
    score           (forward(labels=...))          -> Engine.loglik  (prefill + log-likelihood head)

One image per sample (what every caller in the reference does).  torch is the memory / stream plumbing."""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import hfre as HF
from .engine import Engine, Prefix, Processors, Sampling, SlotPool, splice_plan, splice_plan_batch


@dataclass
class SampleInputs:
    input_ids: Sequence[int]            # prompt ids with -200 (image) / -300 (region) placeholders (mm_utils.py:83-135)
    pixel_values: Optional[torch.Tensor]  # fp32 [gh*gw, 1176]  (Qwen2VLImageProcessor); None with image_u8
    grid_hw: Optional[Tuple[int, int]]
    image_aux: Optional[torch.Tensor]   # fp32 [3, H, W]      (CLIPImageProcessor, 'dynamic' mode); None with image_u8
    boxes: torch.Tensor                 # fp32 [N, 4] xyxy in aux-tensor pixels
    image_u8: Optional[torch.Tensor] = None   # uint8 [H, W, 3] RGB: pre-processed on the device by Fo1Pipeline.preprocess()


def _encoder_meta(s: SampleInputs):
    """Host facts that must agree before two samples' encoder inputs are compared by content."""
    if s.image_u8 is not None:
        return ("u8", tuple(s.image_u8.shape), tuple(s.boxes.shape))
    return ("px", tuple(s.grid_hw), tuple(s.pixel_values.shape), tuple(s.image_aux.shape), tuple(s.boxes.shape))


def _same_tensor(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a is b or (a.device == b.device and a.dtype == b.dtype and torch.equal(a, b))


def encoder_groups(samples: Sequence[SampleInputs]) -> List[int]:
    """rep[b]: the first sample whose encoder inputs (image and boxes) equal sample b's by content.  Host metadata first, then the boxes
    of the remaining candidates in one host copy, then their pixels: distinct images with distinct boxes cost at most that one copy."""
    B = len(samples)
    meta = [_encoder_meta(s) for s in samples]
    count: Dict[tuple, int] = {}
    for m in meta:
        count[m] = count.get(m, 0) + 1
    cand = [b for b in range(B) if count[meta[b]] > 1]
    rep = list(range(B))
    if not cand:
        return rep
    flat = [samples[b].boxes.reshape(-1).to(torch.float32) for b in cand]     # encode() reads the boxes as fp32
    on_dev = [i for i, x in enumerate(flat) if x.is_cuda]
    if on_dev:
        for i, h in zip(on_dev, torch.cat([flat[i] for i in on_dev]).cpu().split([flat[i].numel() for i in on_dev])):
            flat[i] = h
    boxes = dict(zip(cand, flat))
    for i, b in enumerate(cand):
        s = samples[b]
        for c in cand[:i]:
            if rep[c] != c or meta[c] != meta[b] or not torch.equal(boxes[c], boxes[b]):
                continue
            o = samples[c]
            pix = [(o.image_u8, s.image_u8)] if s.image_u8 is not None else [(o.pixel_values, s.pixel_values), (o.image_aux, s.image_aux)]
            if all(_same_tensor(x, y) for x, y in pix):
                rep[b] = c
                break
    return rep


def shared_prefix_groups(prompts: Sequence[Sequence[int]], rep: Sequence[int], image_rows: Sequence[int], lens: Sequence[int],
                         image_placeholder: int = -200) -> List[Tuple[List[int], int]]:
    """-> [(members, P)] for every set of >= 2 samples with equal encoder inputs (``rep``): P is the longest common prefix of their ids,
    placeholders included, counted in spliced rows (an image placeholder is ``image_rows[b]`` rows) and capped at min L_b - 1, so each
    member keeps one row of its own.  Sets with P == 0 are left out (they still share the towers)."""
    sets: Dict[int, List[int]] = {}
    for b, r in enumerate(rep):
        sets.setdefault(r, []).append(b)
    out = []
    for r, mem in sets.items():
        if len(mem) < 2:
            continue
        first = prompts[mem[0]]
        n = min(len(prompts[b]) for b in mem)
        k = 0
        while k < n and all(prompts[b][k] == first[k] for b in mem):
            k += 1
        rows = sum(image_rows[r] if t == image_placeholder else 1 for t in first[:k])
        P = min(rows, min(lens[b] for b in mem) - 1)
        if P >= 1:
            out.append((mem, P))
    return out


IGNORE_INDEX = -100


def splice_labels(input_ids: Sequence[int], labels: Sequence[int], image_rows: int, image_placeholder: int = -200,
                  region_placeholder: int = -300) -> List[int]:
    """The labels of a sample's spliced rows, by the reference's rule (omchat_qwen2_5_vl.py:318-368): a text position keeps its label,
    an image placeholder becomes ``image_rows`` rows labelled -100, a region placeholder one row labelled -100."""
    assert len(labels) == len(input_ids), "one label per input id"
    out: List[int] = []
    for t, lab in zip(input_ids, labels):
        if t == image_placeholder:
            out += [IGNORE_INDEX] * image_rows
        elif t == region_placeholder:
            out.append(IGNORE_INDEX)
        else:
            out.append(int(lab))
    return out


def shift_targets(spliced_labels: Sequence[int]) -> List[int]:
    """HF's ForCausalLMLoss shift within one sequence: row t predicts label t + 1; the last row predicts nothing (-100)."""
    return [int(x) for x in spliced_labels[1:]] + [IGNORE_INDEX]


def causal_lm_loss(seq_logprob: Sequence[float], seq_count: Sequence[int]) -> float:
    """ForCausalLMLoss (reduction 'mean' over every non-ignored shifted label of the batch) from per-sequence sums of the targets'
    log-probabilities and their counts: -sum / count, NaN when nothing is scored (torch's 0 / 0)."""
    n = int(sum(int(c) for c in seq_count))
    tot = float(sum(float(x) for x in seq_logprob))
    return -tot / n if n > 0 else float("nan")


def refill_need(n_slots: int, n_waiting: int) -> int:
    """Free slots at which a slot pool is refilled: a quarter of the pool, or the whole queue when it is shorter, so that the last
    requests are admitted as soon as there is room for them instead of waiting for a quarter of the pool to drain (0: empty queue)."""
    return min(max(1, n_slots // 4), n_waiting)


def run_slots(n_items: int, n_slots: int, admit: Callable[[List[int], List[int]], List[int]], decode: Callable[[int], int],
              poll: Callable[[], Tuple[Sequence[int], Sequence[int]]]) -> Iterator[Tuple[int, int, int]]:
    """The host loop of in-flight batching over a slot pool, items in queue order 0 .. n_items - 1, free slots lowest first.
    ``admit(items, slots)`` prefills the items into the slots and returns the items it admitted (a refused one is skipped and
    frees its slot); ``decode(exit_at)`` decodes until at most exit_at requests run; ``poll()`` -> (finished flag, length) per
    slot.  Yields (item, slot, length) in completion order (slot order within one segment); the slot's outputs are valid until the
    generator is resumed."""
    waiting = deque(range(n_items))
    free = list(range(n_slots))
    running: Dict[int, int] = {}
    while waiting or running:
        if waiting and len(free) >= refill_need(n_slots, len(waiting)):
            k = min(len(free), len(waiting))
            items, slots = [waiting.popleft() for _ in range(k)], free[:k]
            done = set(admit(items, slots))
            for it, b in zip(items, slots):
                if it in done:
                    running[b] = it
            free = sorted(set(free) - set(running))
            if not running:
                continue
        decode(n_slots - refill_need(n_slots, len(waiting)) if waiting else 0)
        fin, lens = poll()
        for b in sorted(running):
            if fin[b]:
                yield running.pop(b), b, int(lens[b])
                free.append(b)
        free.sort()


class Fo1Pipeline:
    def __init__(self, engine: Engine, vt_mode: str = "fpn", image_token_id: int = 151655, vision_start_token_id: int = 151652,
                 video_token_id: int = 151656, roi_size: int = 7, apply_pos_embed: bool = True):
        self.eng = engine
        self.vt_mode = vt_mode
        self.ids = dict(image_token_id=image_token_id, vision_start_token_id=vision_start_token_id, video_token_id=video_token_id)
        self.hcfg = HF.HfreConfig(region_dim=engine.cfg.region_dim, vt_mode=vt_mode, roi_size=roi_size, apply_pos_embed=apply_pos_embed)
        self.ws = HF.HfreWorkspace()
        self.profile_stages = False          # when set, CUDA events bracket every stage (read with stage_ms())
        self._marks = []
        self._keep_stages = None
        self._pre = None
        self.check_plan = True
        self._share_inputs = True            # tests clear it to get the unshared path as the reference of the shared one

    def _mark(self, name: str) -> None:
        if self.profile_stages:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._marks.append((name, e))

    def stage_ms(self) -> Dict[str, float]:
        """Milliseconds between consecutive stage marks of the last call (synchronises)."""
        torch.cuda.synchronize()
        out: Dict[str, float] = {}
        for (n0, e0), (n1, e1) in zip(self._marks[:-1], self._marks[1:]):
            out[n1] = out.get(n1, 0.0) + e0.elapsed_time(e1)
        return out

    # ---- device-side pre-processing (SURVEY.md section 8f rank 1) -----------------------------------------------
    def preprocess(self, samples: Sequence[SampleInputs]) -> List[SampleInputs]:
        """Samples that carry a uint8 image instead of the processors' tensors get them from the GPU (both towers;
        the aux tower in 'dynamic' mode, as the released checkpoint is configured)."""
        if all(s.image_u8 is None for s in samples):
            return list(samples)
        if self._pre is None:
            from .preprocess import DevicePreprocessor
            v = self.eng.cfg.vit
            self._pre = DevicePreprocessor(self.eng.device, v["patch_size"], v["spatial_merge_size"], v["temporal_patch_size"])
        out = []
        for s in samples:
            if s.image_u8 is None:
                out.append(s); continue
            img = s.image_u8.to(self.eng.device, non_blocking=True)
            px, grid = self._pre.primary(img)
            out.append(SampleInputs(s.input_ids, px, grid, self._pre.aux(img, 0), s.boxes))
        return out

    # ---- vision side -------------------------------------------------------------------------------------
    def encode(self, samples: Sequence[SampleInputs]):
        """-> (img_feats [sum merged tokens, hidden] bf16, per-sample row offsets, region tokens list of [N_b, hidden] bf16,
        region features fp32 list)."""
        eng, dev = self.eng, self.eng.device
        self._marks = []
        self._mark("start")
        samples = self.preprocess(samples)
        if any(s.image_u8 is not None for s in samples) or self._pre is not None:
            self._mark("preprocess")
        grids = [s.grid_hw for s in samples]
        feats, taps = eng.vit_forward([s.pixel_values for s in samples], grids)
        feats = eng.image_project(feats)                                             # mm_projector (:58-66); identity for the released checkpoint
        self._mark("vit")
        B = len(samples)
        H0, W0 = samples[0].image_aux.shape[-2:]
        same_aux = all(s.image_aux.shape[-2:] == (H0, W0) for s in samples)
        same_grid = all(g == grids[0] for g in grids)
        aux_b = vt_b = None                      # batch-contiguous level maps (the packed HFRE path)
        if same_aux:
            st = eng.davit_forward([s.image_aux for s in samples])
            aux_b = st
            aux = None
        else:
            aux = []
            for s in samples:
                st = eng.davit_forward([s.image_aux])
                aux.append([st[l][0] for l in range(4)])
        self._mark("davit")
        tok_off = np.cumsum([0] + [gh * gw for gh, gw in grids])
        hid = eng.cfg.vit["hidden_size"]
        vt = None
        if self.vt_mode == "fpn":
            if same_grid:
                gh, gw = grids[0]
                vt_b = eng.fpn_forward(taps[-1].view(B, gh, gw, hid))           # SimpleFPN on the LAST tap (:82-83)
            else:
                vt = []
                for b, (gh, gw) in enumerate(grids):
                    pyr = eng.fpn_forward(taps[-1][tok_off[b]:tok_off[b + 1]].view(1, gh, gw, hid))
                    vt.append([pyr[l][0] for l in range(4)])
        else:
            vt = [[taps[t][tok_off[b]:tok_off[b + 1]].view(grids[b][0], grids[b][1], hid) for t in range(len(taps))] for b in range(B)]
        self._mark("fpn")
        packed = aux_b is not None and vt_b is not None
        if not packed or self._keep_stages is not None:
            if aux is None:
                aux = [[aux_b[l][b] for l in range(4)] for b in range(B)]
            if vt is None:
                vt = [[vt_b[l][b] for l in range(4)] for b in range(B)]
        # boxes: the aux set in image pixels, the vt set rescaled to the ViT grid (:94-99); one packed array per set
        p = eng.cfg.vit["patch_size"]
        host_boxes = all(not s.boxes.is_cuda for s in samples)
        bl, sl = [], []
        for b, s in enumerate(samples):
            bx = s.boxes
            if bx.numel() == 0:
                bx = torch.tensor([[0.0, 10.0, 0.0, 10.0]], device=bx.device)        # the reference's dummy box (:90-91)
            Ha, Wa = s.image_aux.shape[-2:]
            gh, gw = grids[b]
            bl.append(bx)
            sl.append(np.tile(np.asarray([gw * p / Wa, gh * p / Ha, gw * p / Wa, gh * p / Ha], dtype=np.float32), (bx.shape[0], 1)))
        counts = [int(x.shape[0]) for x in bl]
        scale_rows = torch.from_numpy(np.concatenate(sl, 0))
        if host_boxes:     # fp32 multiply on the host: the same IEEE product the reference forms on the device; two copies instead of 4 B
            ba_h = torch.cat([x.to(torch.float32) for x in bl], 0)
            both = torch.stack([ba_h, ba_h * scale_rows], 0).pin_memory()
            both_d = both.to(dev, non_blocking=True)
            boxes_aux_p, boxes_vt_p = both_d[0], both_d[1]
        else:
            boxes_aux_p = torch.cat([x.to(dev, torch.float32) for x in bl], 0)
            boxes_vt_p = boxes_aux_p * scale_rows.to(dev, non_blocking=True)
        if packed:
            region_f32_p, region_bf16_p = HF.hfre_forward_packed(aux_b, vt_b, boxes_aux_p, boxes_vt_p, counts, self.hcfg, grids[0],
                                                                 want_bf16=True, workspace=self.ws)
        else:
            ba = list(torch.split(boxes_aux_p, counts, 0)); bv = list(torch.split(boxes_vt_p, counts, 0))
            rf, rb = HF.hfre_forward(aux, vt, ba, bv, self.hcfg, grids, want_bf16=True, workspace=self.ws)
            region_f32_p, region_bf16_p = torch.cat(rf, 0), torch.cat(rb, 0)
        self._mark("hfre")
        region_f32 = list(torch.split(region_f32_p, counts, 0))
        tokens = eng.region_project(region_bf16_p)
        self._mark("projector")
        region_tokens = list(torch.split(tokens, counts, 0))
        unit = eng.cfg.vit["spatial_merge_size"] ** 2
        img_off = np.cumsum([0] + [gh * gw // unit for gh, gw in grids])
        if self._keep_stages is not None:
            self._keep_stages.update(image_features=feats, taps=taps, davit=aux, fpn=vt if self.vt_mode == "fpn" else None,
                                     region_f32=region_f32, region_tokens=region_tokens)
        return feats, img_off, region_tokens, region_f32

    def encode_stages(self, samples: Sequence[SampleInputs]) -> dict:
        """encode() that also hands back every intermediate map for the stage-drift test: 'taps' (list over the tap layers of
        [sum gh*gw, hidden]), 'davit' / 'fpn' as [level][image] maps, 'image_features', 'region_f32', 'region_tokens'."""
        self._keep_stages = {}
        try:
            self.encode(samples)
            out = self._keep_stages
        finally:
            self._keep_stages = None
        B = len(samples)
        out["davit"] = [[out["davit"][b][l] for b in range(B)] for l in range(4)]
        if out["fpn"] is not None:
            out["fpn"] = [[out["fpn"][b][l] for b in range(B)] for l in range(4)]
        return out

    # ---- language side -----------------------------------------------------------------------------------
    def generate(self, samples: Sequence[SampleInputs], max_new_tokens: int, stop_ids: Sequence[int], pad_id: int = 151643,
                 early_exit_interval: int = 8, want_prefill_logits: bool = False, sampling=None, want_logprobs: bool = False,
                 want_scores: bool = False, want_logits: bool = False, raw_rows=None, on_tokens=None, beams=None, lookup=None,
                 processors=None):
        """``sampling``: None (greedy) or an engine.Sampling with one parameter set per sample.  ``want_logprobs`` / ``want_scores`` /
        ``want_logits`` / ``raw_rows``: per-token scores, as Engine.generate.  ``on_tokens``: the streaming callback of
        Engine.generate (columns of the whole batch, in sample order).  ``beams``: an engine.Beams, beam search for every sample
        (Engine.generate's outputs); the towers still run once per unique image, but each prompt is prefilled in full.  ``lookup``: an
        engine.Lookup, prompt-lookup decoding; without a corpus of its own, each sample's ``input_ids`` is its corpus (HF's).
        ``processors``: an engine.Processors, one ProcessorSet or None per sample; without prompts of its own, each sample's
        ``input_ids`` is its history's prompt (HF's input_ids)."""
        from dataclasses import replace
        if processors is not None and processors.prompts is None:
            processors = replace(processors, prompts=[list(s.input_ids) for s in samples])
        if lookup is not None and lookup.corpus is None:
            lookup = replace(lookup, corpus=[list(s.input_ids) for s in samples])
        eng, dev = self.eng, self.eng.device
        kw = dict(max_new_tokens=max_new_tokens, stop_ids=stop_ids, pad_id=pad_id, early_exit_interval=early_exit_interval,
                  want_prefill_logits=want_prefill_logits, sampling=sampling, want_logprobs=want_logprobs, want_scores=want_scores,
                  want_logits=want_logits, raw_rows=raw_rows, on_tokens=on_tokens, beams=beams, lookup=lookup, processors=processors)
        if self._share_inputs and len(samples) > 1:
            rep = encoder_groups(samples)
            if any(r != b for b, r in enumerate(rep)):
                return self._generate_shared(samples, rep, **kw)
        samples = self.preprocess(samples)           # uint8 images -> the towers' input tensors, on the device
        feats, img_off, region_tokens, _ = self.encode(samples)
        # splice + M-RoPE bookkeeping of the whole batch in one launch on the device (fo1_splice_plan_batch); the per-sample host
        # function fo1_splice_plan stays the bit-exact reference of it (tests/test_gpu_prompt.py)
        merge = eng.cfg.vit["spatial_merge_size"]
        plan = splice_plan_batch([s.input_ids for s in samples], [[s.grid_hw] for s in samples], [r.shape[0] for r in region_tokens], dev,
                                 merge=merge, **self.ids)
        lens = plan["lens"]
        embeds = eng.build_embeds(plan["kind"], plan["index"], feats, torch.cat(region_tokens, 0))
        pos = plan["position_ids"]
        if self.check_plan:                                      # opt-in: surface a malformed prompt as an exception (one D2H sync)
            st = plan["status"].cpu().tolist()
            if any(st):
                raise ValueError(f"fo1_splice_plan_batch: per-sample status {st} (placeholders and features disagree)")
        deltas = plan["rope_delta"]
        self._mark("splice")
        out = eng.generate(embeds, pos, lens, deltas, max_new_tokens, stop_ids, pad_id, want_prefill_logits=want_prefill_logits,
                           early_exit_interval=early_exit_interval, sampling=sampling, want_logprobs=want_logprobs, want_scores=want_scores,
                           want_logits=want_logits, raw_rows=raw_rows, on_tokens=on_tokens, beams=beams, lookup=lookup, processors=processors)
        self._mark("llm_prefill_decode")
        out["prompt_lens"] = lens
        return out

    def _generate_shared(self, samples, rep, max_new_tokens, stop_ids, pad_id, early_exit_interval, want_prefill_logits, sampling,
                         want_logprobs, want_scores, want_logits, raw_rows, on_tokens, beams, lookup, processors):
        """generate() of a batch in which some samples have equal encoder inputs: the towers run once per unique image, and each set's
        common prompt prefix is prefilled once (Engine.generate's ``prefix``).  Bit-identical to the unshared path."""
        eng, dev = self.eng, self.eng.device
        B = len(samples)
        own = [b for b in range(B) if rep[b] == b]
        slot = {b: i for i, b in enumerate(own)}
        uniq = self.preprocess([samples[b] for b in own])
        feats, _, region_tokens, _ = self.encode(uniq)
        merge = eng.cfg.vit["spatial_merge_size"]
        grids = [uniq[slot[rep[b]]].grid_hw for b in range(B)]
        prompts = [samples[b].input_ids for b in range(B)]
        plan = splice_plan_batch(prompts, [[g] for g in grids], [region_tokens[slot[rep[b]]].shape[0] for b in range(B)], dev, merge=merge,
                                 row_src=rep, **self.ids)
        lens = plan["lens"]
        if self.check_plan:
            st = plan["status"].cpu().tolist()
            if any(st):
                raise ValueError(f"fo1_splice_plan_batch: per-sample status {st} (placeholders and features disagree)")
        regions = torch.cat(region_tokens, 0)
        # beam search prefills each prompt once in full (its K/V goes to its N slots); only the towers are shared
        groups = shared_prefix_groups(prompts, rep, [gh * gw // (merge * merge) for gh, gw in grids], lens) if beams is None else []
        embeds, pos, prefix = self._prefix_inputs(plan, lens, groups, feats, regions)
        self._mark("splice")
        out = eng.generate(embeds, pos, lens, plan["rope_delta"], max_new_tokens, stop_ids, pad_id, want_prefill_logits=want_prefill_logits,
                           early_exit_interval=early_exit_interval, sampling=sampling, want_logprobs=want_logprobs, want_scores=want_scores,
                           want_logits=want_logits, raw_rows=raw_rows, on_tokens=on_tokens, prefix=prefix, beams=beams, lookup=lookup,
                           processors=processors)
        self._mark("llm_prefill_decode")
        out["prompt_lens"] = lens
        return out

    # ---- teacher-forced scoring -----------------------------------------------------------------------------
    def score(self, samples: Sequence[SampleInputs], labels: Sequence[Sequence[int]], want_greedy: bool = False,
              want_all_logits: bool = False, want_lse: bool = False) -> dict:
        """The log-likelihood of each sample's labels (HF layout over its ``input_ids``, -100 ignored) under the model, teacher
        forced, without decoding (Engine.loglik).  Labels are spliced as the reference splices them (splice_labels) and shifted within
        each sample (shift_targets).  Samples with equal encoder inputs share the towers, and their common prompt prefix is prefilled
        once, capped before the first scored row of every member: ranking K answers about one image is a score() of K samples that
        differ only in the answer.  Every output is bit-identical to scoring each sample alone.  Returns Engine.loglik's dict plus
        ``prompt_lens`` (spliced lengths) and ``targets`` (int32 numpy [sum L])."""
        eng, dev = self.eng, self.eng.device
        B = len(samples)
        assert len(labels) == B, "one label list per sample"
        rep = encoder_groups(samples) if self._share_inputs and B > 1 else list(range(B))
        own = [b for b in range(B) if rep[b] == b]
        slot = {b: i for i, b in enumerate(own)}
        uniq = self.preprocess([samples[b] for b in own])
        feats, _, region_tokens, _ = self.encode(uniq)
        merge = eng.cfg.vit["spatial_merge_size"]
        grids = [uniq[slot[rep[b]]].grid_hw for b in range(B)]
        prompts = [list(samples[b].input_ids) for b in range(B)]
        plan = splice_plan_batch(prompts, [[g] for g in grids], [region_tokens[slot[rep[b]]].shape[0] for b in range(B)], dev, merge=merge,
                                 row_src=rep, **self.ids)
        lens = plan["lens"]
        st = plan["status"].cpu().tolist()
        if any(st):
            raise ValueError(f"fo1_splice_plan_batch: per-sample status {st} (placeholders and features disagree)")
        image_rows = [gh * gw // (merge * merge) for gh, gw in grids]
        targets = []
        for b in range(B):
            sl = splice_labels(prompts[b], labels[b], image_rows[b])
            assert len(sl) == lens[b], f"sample {b}: {len(sl)} spliced labels for {lens[b]} rows"
            targets.append(shift_targets(sl))
        regions = torch.cat(region_tokens, 0)
        groups = shared_prefix_groups(prompts, rep, image_rows, lens) if self._share_inputs and not want_all_logits else []
        first = [next((t for t, x in enumerate(tg) if x != IGNORE_INDEX), len(tg)) for tg in targets]
        groups = [(mem, min(P, min(first[b] for b in mem))) for mem, P in groups]     # no scored row inside a prefix
        groups = [(mem, P) for mem, P in groups if P >= 1]
        embeds, pos, prefix = self._prefix_inputs(plan, lens, groups, feats, regions)
        self._mark("splice")
        tg = np.asarray([x for t in targets for x in t], dtype=np.int32)
        out = eng.loglik(embeds, pos, lens, tg, prefix=prefix, want_greedy=want_greedy, want_all_logits=want_all_logits, want_lse=want_lse)
        self._mark("llm_loglik")
        out["prompt_lens"] = lens
        out["targets"] = tg
        out["rope_delta"] = plan["rope_delta"]
        return out

    def _prefix_inputs(self, plan, lens, groups, feats, regions):
        """-> (embeds, position_ids, Prefix or None) of a spliced batch with the shared-prefix ``groups`` [(members, P)]: the groups'
        prefix rows once, then every sequence's own rows."""
        eng, dev = self.eng, self.eng.device
        if not groups:
            return eng.build_embeds(plan["kind"], plan["index"], feats, regions), plan["position_ids"], None
        B = len(lens)
        start = np.cumsum([0] + list(lens))
        seq_group, pre = [-1] * B, [0] * B
        sel = []
        for g, (mem, P) in enumerate(groups):
            sel.append(np.arange(start[mem[0]], start[mem[0]] + P))
            for b in mem:
                seq_group[b], pre[b] = g, P
        sel += [np.arange(start[b] + pre[b], start[b + 1]) for b in range(B)]
        idx = torch.from_numpy(np.concatenate(sel).astype(np.int64)).to(dev, non_blocking=True)
        n_pre = sum(P for _, P in groups)
        emb = eng.build_embeds(plan["kind"][idx].contiguous(), plan["index"][idx].contiguous(), feats, regions)
        pos_all = plan["position_ids"][:, idx]
        return emb[n_pre:], pos_all[:, n_pre:], Prefix([P for _, P in groups], emb[:n_pre], pos_all[:, :n_pre], seq_group)

    # ---- in-flight batching ---------------------------------------------------------------------------------
    def prompt_rows(self, s: SampleInputs, image_placeholder: int = -200) -> int:
        """Prompt rows of a sample after the splice: exact for processor outputs, and for a uint8 image the rows of the largest image the
        processors produce (2048 x 2048 px)."""
        v = self.eng.cfg.vit
        unit = v["spatial_merge_size"] ** 2
        n_ph = sum(1 for t in s.input_ids if t == image_placeholder)
        if s.grid_hw is not None:
            rows = s.grid_hw[0] * s.grid_hw[1] // unit
        else:
            side = 2048 // (v["patch_size"] * v["spatial_merge_size"])
            rows = side * side
        return len(s.input_ids) - n_ph + min(n_ph, 1) * rows

    def generate_continuous(self, samples: Sequence[SampleInputs], n_slots: int, max_new_tokens, stop_ids: Sequence[int],
                            pad_id: int = 151643, sampling: Optional[Sampling] = None, early_exit_interval: int = 8,
                            on_error: Optional[Callable[[int, BaseException], None]] = None,
                            processors: Optional[Processors] = None) -> Iterator[Tuple[int, torch.Tensor, int]]:
        """Every sample through a slot pool of ``n_slots`` slots (engine.SlotPool): a finished request hands its slot to the next
        waiting one.  ``max_new_tokens``: one int, or one per sample; ``sampling``: None (greedy) or one parameter set per sample.
        Yields (index, tokens int32 [n] on the device, n) in completion order.  Each request's tokens and length equal those of a
        static generate() of ``n_slots`` samples on the same decode path (at most 8 slots on the persistent kernel, or 16 on the
        per-kernel path of a 132-SM H100: those of generate() alone).  Admission groups are encoded together (equal images share the
        towers); a group that fails is retried request by request, and a request that still fails is passed to ``on_error(index,
        exception)`` and skipped (without ``on_error`` the exception propagates).  ``processors``: None or an engine.Processors with
        one ProcessorSet or None per sample (prompts: each sample's ``input_ids`` unless given)."""
        B = len(samples)
        if B == 0:
            return
        mnt = [int(max_new_tokens)] * B if isinstance(max_new_tokens, int) else [int(x) for x in max_new_tokens]
        assert len(mnt) == B and min(mnt) >= 1, "one max_new_tokens >= 1 per sample"
        assert sampling is None or len(sampling.temperature) == B, "one sampling parameter set per sample"
        T = max(mnt)
        cap = max(self.prompt_rows(s) + m for s, m in zip(samples, mnt))
        eng, dev = self.eng, self.eng.device
        merge = eng.cfg.vit["spatial_merge_size"]
        pool = SlotPool(eng, n_slots, cap, T, stop_ids, pad_id, sampled=sampling is not None, early_exit_interval=early_exit_interval)

        def admit_group(items, slots):
            group = self.preprocess([samples[i] for i in items])
            rep = encoder_groups(group) if self._share_inputs and len(group) > 1 else list(range(len(group)))
            own = [b for b in range(len(group)) if rep[b] == b]
            slot_of = {b: i for i, b in enumerate(own)}
            feats, _, region_tokens, _ = self.encode([group[b] for b in own])
            grids = [group[rep[b]].grid_hw for b in range(len(group))]
            plan = splice_plan_batch([s.input_ids for s in group], [[g] for g in grids],
                                     [region_tokens[slot_of[rep[b]]].shape[0] for b in range(len(group))], dev, merge=merge,
                                     row_src=rep, **self.ids)
            st = plan["status"].cpu().tolist()
            if any(st):
                raise ValueError(f"fo1_splice_plan_batch: per-sample status {st} (placeholders and features disagree)")
            embeds = eng.build_embeds(plan["kind"], plan["index"], feats, torch.cat(region_tokens, 0))
            sp = None
            if sampling is not None:
                sp = Sampling(*([list(f)[i] for i in items] for f in (sampling.temperature, sampling.top_p, sampling.top_k, sampling.seed)))
            pr = None
            if processors is not None:
                prompts = processors.prompts if processors.prompts is not None else [s.input_ids for s in samples]
                pr = Processors([processors.sets[i] for i in items], [list(prompts[i]) for i in items])
            pool.admit(slots, embeds, plan["position_ids"], plan["lens"], plan["rope_delta"], [mnt[i] for i in items], sampling=sp,
                       **({"processors": pr} if pr is not None else {}))

        def admit(items, slots):
            try:
                admit_group(items, slots)
                return items
            except Exception:
                if on_error is None:
                    raise
            done = []
            for it, b in zip(items, slots):        # the group failed: each request alone, the failing ones reported and skipped
                try:
                    admit_group([it], [b])
                    done.append(it)
                except Exception as exc:  # noqa: BLE001 -- handed to the caller's on_error
                    on_error(it, exc)
            return done

        def poll():
            return pool.finished.cpu().tolist(), pool.lens.cpu().tolist()

        try:
            for it, b, n in run_slots(B, n_slots, admit, pool.decode, poll):
                yield it, pool.tokens[b, :n].clone(), n
        finally:
            pool.close()
