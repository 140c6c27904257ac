"""Model handle over the C ABI: owns the fo1_model*, keeps the prepared weight tensors alive, and exposes
the stage entry points with torch tensors as memory handles."""
from __future__ import annotations

import ctypes as C
import threading
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import check, lib

_DT = {torch.bfloat16: _lib.FO1_BF16, torch.float32: _lib.FO1_F32}


class ModelConfigC(C.Structure):
    _fields_ = [
        ("vit_depth", C.c_int32), ("vit_hidden", C.c_int32), ("vit_heads", C.c_int32), ("vit_inter", C.c_int32),
        ("vit_inter_pad", C.c_int32), ("vit_out_hidden", C.c_int32), ("vit_patch", C.c_int32), ("vit_merge", C.c_int32),
        ("vit_temporal", C.c_int32), ("vit_in_ch", C.c_int32), ("vit_window", C.c_int32),
        ("vit_n_fullatt", C.c_int32), ("vit_fullatt", C.c_int32 * 8),
        ("davit_dims", C.c_int32 * 4), ("davit_depths", C.c_int32 * 4), ("davit_heads", C.c_int32 * 4),
        ("davit_groups", C.c_int32 * 4), ("davit_window", C.c_int32),
        ("fpn_out", C.c_int32), ("region_dim", C.c_int32), ("proj_aux_layers", C.c_int32), ("proj_img_layers", C.c_int32),
        ("llm_layers", C.c_int32), ("llm_hidden", C.c_int32), ("llm_heads", C.c_int32), ("llm_kv_heads", C.c_int32),
        ("llm_head_dim", C.c_int32), ("llm_inter", C.c_int32), ("llm_vocab", C.c_int32),
        ("mrope_section", C.c_int32 * 3), ("rope_theta", C.c_float), ("rms_eps", C.c_float), ("tie_embeddings", C.c_int32),
    ]


@dataclass
class EngineConfig:
    """Python-side mirror of fo1_model_config; defaults are the released 3B checkpoint's architecture
    (SURVEY.md section 8: ViT 32x1280, DaViT-large, SimpleFPN 512, Qwen2.5-3B)."""
    vit: dict = field(default_factory=lambda: dict(depth=32, hidden_size=1280, num_heads=16, intermediate_size=3420,
                                                   out_hidden_size=2048, patch_size=14, spatial_merge_size=2,
                                                   temporal_patch_size=2, in_channels=3, window_size=112,
                                                   fullatt_block_indexes=[7, 15, 23, 31]))
    davit: dict = field(default_factory=lambda: dict(depths=[1, 1, 9, 1], dim_embed=[256, 512, 1024, 2048],
                                                     num_heads=[8, 16, 32, 64], num_groups=[8, 16, 32, 64], window_size=12))
    fpn_out: int = 512
    region_dim: int = 5888
    proj_aux_layers: int = 2
    proj_img_layers: int = 0
    llm: dict = field(default_factory=lambda: dict(num_hidden_layers=36, hidden_size=2048, num_attention_heads=16,
                                                   num_key_value_heads=2, intermediate_size=11008, vocab_size=151936,
                                                   rope_theta=1000000.0, rms_norm_eps=1e-6, mrope_section=[16, 24, 24],
                                                   tie_word_embeddings=True))
    use_vit: bool = True
    use_davit: bool = True
    use_llm: bool = True

    def to_c(self) -> ModelConfigC:
        from .weights import vit_inter_pad
        c = ModelConfigC()
        if self.use_vit:
            v = self.vit
            c.vit_depth, c.vit_hidden, c.vit_heads = v["depth"], v["hidden_size"], v["num_heads"]
            c.vit_inter, c.vit_inter_pad = v["intermediate_size"], vit_inter_pad(v["intermediate_size"])
            c.vit_out_hidden, c.vit_patch, c.vit_merge = v["out_hidden_size"], v["patch_size"], v["spatial_merge_size"]
            c.vit_temporal, c.vit_in_ch, c.vit_window = v["temporal_patch_size"], v.get("in_channels", 3), v["window_size"]
            fa = list(v["fullatt_block_indexes"])
            c.vit_n_fullatt = len(fa)
            for i, x in enumerate(fa):
                c.vit_fullatt[i] = x
            c.fpn_out = self.fpn_out
        if self.use_davit:
            d = self.davit
            for i in range(4):
                c.davit_dims[i], c.davit_depths[i] = d["dim_embed"][i], d["depths"][i]
                c.davit_heads[i], c.davit_groups[i] = d["num_heads"][i], d["num_groups"][i]
            c.davit_window = d["window_size"]
        c.region_dim, c.proj_aux_layers, c.proj_img_layers = self.region_dim, self.proj_aux_layers, self.proj_img_layers
        l = self.llm
        c.llm_hidden = l["hidden_size"]
        if self.use_llm:
            c.llm_layers, c.llm_heads, c.llm_kv_heads = l["num_hidden_layers"], l["num_attention_heads"], l["num_key_value_heads"]
            c.llm_head_dim = l["hidden_size"] // l["num_attention_heads"]
            c.llm_inter, c.llm_vocab = l["intermediate_size"], l["vocab_size"]
            for i in range(3):
                c.mrope_section[i] = l["mrope_section"][i]
            c.rope_theta, c.rms_eps = l["rope_theta"], l["rms_norm_eps"]
            c.tie_embeddings = 1 if l.get("tie_word_embeddings", False) else 0
        return c


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Engine:
    def __init__(self, cfg: EngineConfig, device: Optional[torch.device] = None):
        self.cfg = cfg
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._c = cfg.to_c()
        self._h = C.c_void_p()
        L = lib()
        L.fo1_model_create.restype = C.c_int
        L.fo1_model_create.argtypes = [C.POINTER(ModelConfigC), C.POINTER(C.c_void_p)]
        L.fo1_model_destroy.restype = None
        L.fo1_model_destroy.argtypes = [C.c_void_p]
        L.fo1_model_set_weight.restype = C.c_int
        L.fo1_model_set_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
        L.fo1_model_finalize.restype = C.c_int
        L.fo1_model_finalize.argtypes = [C.c_void_p]
        for fn in ("fo1_vit_forward", "fo1_davit_forward", "fo1_fpn_forward", "fo1_region_project", "fo1_image_project"):
            getattr(L, fn).restype = C.c_int
        check(L.fo1_model_create(C.byref(self._c), C.byref(self._h)), "fo1_model_create")
        self.weights: Dict[str, torch.Tensor] = {}

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                lib().fo1_model_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def last_decode_path(self) -> int:
        """1: the last generate() ran the persistent decode kernel, 0: the per-kernel CUDA graph, -1: none yet."""
        return int(lib().fo1_last_decode_path(self._h))

    # ---- weights ----
    def set_weights(self, tensors: Dict[str, torch.Tensor]) -> None:
        L = lib()
        for name, t in tensors.items():
            assert t.is_cuda and t.is_contiguous(), name
            self.weights[name] = t
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(L.fo1_model_set_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()), _DT[t.dtype], t.dim(), shape),
                  f"fo1_model_set_weight({name})")

    def finalize(self) -> None:
        check(lib().fo1_model_finalize(self._h), "fo1_model_finalize")

    # ---- stages ----
    def vit_forward(self, pixel_values: Sequence[torch.Tensor], grids: Sequence[Tuple[int, int]]):
        """-> (img_feats [sum gh*gw/4, out_hidden] bf16, taps: list over tap layers of [sum gh*gw, hidden] bf16).
        Image b's slice of a tap is its channels-last map [gh, gw, hidden]."""
        v = self.cfg.vit
        B = len(pixel_values)
        px = [p.to(self.device, torch.float32).contiguous() for p in pixel_values]
        T = sum(gh * gw for gh, gw in grids)
        unit = v["spatial_merge_size"] ** 2
        feats = torch.empty((T // unit, v["out_hidden_size"]), dtype=torch.bfloat16, device=self.device)
        taps = [torch.empty((T, v["hidden_size"]), dtype=torch.bfloat16, device=self.device) for _ in v["fullatt_block_indexes"]]
        pp = (C.c_void_p * B)(*[p.data_ptr() for p in px])
        g = (C.c_int32 * (2 * B))(*[x for gw_ in grids for x in gw_])
        tp = (C.c_void_p * len(taps))(*[t.data_ptr() for t in taps])
        check(lib().fo1_vit_forward(self._h, pp, g, B, C.c_void_p(feats.data_ptr()), tp, _stream()), "fo1_vit_forward")
        return feats, taps

    def davit_forward(self, images: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """images: B x fp32 [3, H, W] (same size) -> 4 stage maps bf16 [B, H_s, W_s, C_s]."""
        B = len(images)
        im = [i.to(self.device, torch.float32).contiguous() for i in images]
        H, W = im[0].shape[-2:]
        assert all(i.shape[-2:] == (H, W) for i in im), "fo1_davit_forward batches images of one size"
        outs = []
        h, w = (H + 6 - 7) // 4 + 1, (W + 6 - 7) // 4 + 1
        for s in range(4):
            if s:
                h, w = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
            outs.append(torch.empty((B, h, w, self.cfg.davit["dim_embed"][s]), dtype=torch.bfloat16, device=self.device))
        ip = (C.c_void_p * B)(*[i.data_ptr() for i in im])
        op = (C.c_void_p * 4)(*[o.data_ptr() for o in outs])
        check(lib().fo1_davit_forward(self._h, ip, H, W, B, op, _stream()), "fo1_davit_forward")
        return outs

    def fpn_forward(self, tap: torch.Tensor) -> List[torch.Tensor]:
        """tap bf16 [B, gh, gw, hidden] -> 4 levels bf16 [B, gh*f, gw*f, fpn_out]."""
        B, gh, gw, _ = tap.shape
        tap = tap.contiguous()
        dims = [(gh * 4, gw * 4), (gh * 2, gw * 2), (gh, gw), (gh // 2, gw // 2)]
        outs = [torch.empty((B, h, w, self.cfg.fpn_out), dtype=torch.bfloat16, device=self.device) for h, w in dims]
        op = (C.c_void_p * 4)(*[o.data_ptr() for o in outs])
        check(lib().fo1_fpn_forward(self._h, C.c_void_p(tap.data_ptr()), gh, gw, B, op, _stream()), "fo1_fpn_forward")
        return outs

    def image_project(self, feats: torch.Tensor) -> torch.Tensor:
        """mm_projector on the merged image tokens (encode_images, omchat_qwen2_5_vl.py:58-66); identity when proj_img_layers == 0."""
        if self.cfg.proj_img_layers == 0:
            return feats
        feats = feats.contiguous()
        out = torch.empty((feats.shape[0], self.cfg.llm["hidden_size"]), dtype=torch.bfloat16, device=self.device)
        check(lib().fo1_image_project(self._h, C.c_void_p(feats.data_ptr()), feats.shape[0], C.c_void_p(out.data_ptr()), _stream()),
              "fo1_image_project")
        return out

    def region_project(self, feats: torch.Tensor) -> torch.Tensor:
        feats = feats.contiguous()
        out = torch.empty((feats.shape[0], self.cfg.llm["hidden_size"]), dtype=torch.bfloat16, device=self.device)
        check(lib().fo1_region_project(self._h, C.c_void_p(feats.data_ptr()), feats.shape[0], C.c_void_p(out.data_ptr()), _stream()),
              "fo1_region_project")
        return out


class SpliceCfgC(C.Structure):
    _fields_ = [("image_token_id", C.c_int32), ("video_token_id", C.c_int32), ("vision_start_token_id", C.c_int32),
                ("merge", C.c_int32), ("image_placeholder", C.c_int32), ("region_placeholder", C.c_int32)]


class GenerateDescC(C.Structure):
    _fields_ = [("n_seqs", C.c_int32), ("seq_lens", C.POINTER(C.c_int32)), ("inputs_embeds", C.c_void_p),
                ("position_ids", C.c_void_p), ("rope_deltas", C.POINTER(C.c_int32)), ("max_new_tokens", C.c_int32),
                ("stop_ids", C.POINTER(C.c_int32)), ("n_stop_ids", C.c_int32), ("pad_id", C.c_int32),
                ("out_tokens", C.c_void_p), ("out_lens", C.c_void_p), ("prefill_logits", C.c_void_p),
                ("all_logits", C.c_void_p), ("early_exit_interval", C.c_int32), ("steps_run", C.c_int32), ("rope_deltas_device", C.c_void_p),
                ("sampling", C.POINTER(_lib.SamplingDesc)), ("scores", C.POINTER(_lib.ScoreDesc)), ("stream", C.POINTER(_lib.StreamDesc)),
                ("prefix", C.POINTER(_lib.PrefixDesc)), ("processors", C.POINTER(_lib.ProcessorDesc)), ("lookup", C.POINTER(_lib.LookupDesc)),
                ("beam", C.POINTER(_lib.BeamDesc))]


def splice_plan(input_ids: Sequence[int], image_grids: Sequence[Tuple[int, int]], n_regions: int,
                image_token_id: int = 151655, video_token_id: int = 151656, vision_start_token_id: int = 151652,
                merge: int = 2, image_placeholder: int = -200, region_placeholder: int = -300):
    """Host-side integer work for one sample (fo1_splice_plan): -> dict(new_ids, kind, index, position_ids [3, L], rope_delta)."""
    import numpy as np
    L = lib()
    L.fo1_splice_plan.restype = C.c_int
    cfg = SpliceCfgC(image_token_id, video_token_id, vision_start_token_id, merge, image_placeholder, region_placeholder)
    ids = (C.c_int64 * len(input_ids))(*[int(t) for t in input_ids])
    grids = (C.c_int32 * max(2 * len(image_grids), 1))(*[int(x) for g in image_grids for x in g])
    cap = len(input_ids) + sum(gh * gw // (merge * merge) for gh, gw in image_grids) + 8
    new_ids = np.empty(cap, dtype=np.int64); kind = np.empty(cap, dtype=np.int32); index = np.empty(cap, dtype=np.int32)
    pos = np.empty((3, cap), dtype=np.int32)
    delta = C.c_int32(); n = C.c_int32()
    check(L.fo1_splice_plan(ids, len(input_ids), grids, len(image_grids), n_regions, C.byref(cfg),
                            new_ids.ctypes.data_as(C.POINTER(C.c_int64)), kind.ctypes.data_as(C.POINTER(C.c_int32)),
                            index.ctypes.data_as(C.POINTER(C.c_int32)), pos.ctypes.data_as(C.POINTER(C.c_int32)),
                            C.byref(delta), C.byref(n), cap), "fo1_splice_plan")
    k = n.value
    return dict(new_ids=new_ids[:k], kind=kind[:k], index=index[:k], position_ids=pos[:, :k].copy(), rope_delta=delta.value)


def _engine_build_embeds(self, kind: torch.Tensor, index: torch.Tensor, img_feats: Optional[torch.Tensor],
                         region_feats: Optional[torch.Tensor]) -> torch.Tensor:
    """inputs_embeds rows from the embedding table / image features / region features (device int32 kind, index)."""
    n = kind.numel()
    out = torch.empty((n, self.cfg.llm["hidden_size"]), dtype=torch.bfloat16, device=self.device)
    L = lib()
    L.fo1_llm_build_embeds.restype = C.c_int
    check(L.fo1_llm_build_embeds(self._h, C.c_void_p(kind.data_ptr()), C.c_void_p(index.data_ptr()), n,
                                 C.c_void_p(img_feats.data_ptr() if img_feats is not None else 0),
                                 C.c_void_p(region_feats.data_ptr() if region_feats is not None else 0),
                                 C.c_void_p(out.data_ptr()), _stream()), "fo1_llm_build_embeds")
    return out


@dataclass
class Sampling:
    """Per-sequence sampling parameters (fo1_sampling_desc): temperature > 0, top_p in (0, 1] (1 = off), top_k >= 0 (0 = off,
    1 = greedy), seed = the 64-bit Philox key of the sequence."""
    temperature: Sequence[float]
    top_p: Sequence[float]
    top_k: Sequence[int]
    seed: Sequence[int]


@dataclass
class Prefix:
    """Shared prompt prefixes of a generate call (fo1_prefix_desc): group g's sequences start with the same ``lens[g]`` rows, whose
    embeddings ``embeds`` bf16 [sum lens, hidden] and positions ``position_ids`` int32 [3, sum lens] are given once, groups back to
    back.  ``seq_group[b]``: sequence b's group, or -1."""
    lens: Sequence[int]
    embeds: torch.Tensor
    position_ids: torch.Tensor
    seq_group: Sequence[int]


@dataclass
class Beams:
    """Beam search of a generate call (fo1_beam_desc), one setting for every prompt: ``num_beams`` N in [2, 16]; ``n_keep`` the
    candidates kept per step, HF's max(2, 1 + number of eos ids) * N; ``length_penalty``; ``early_stopping`` True, False or
    "never"; ``num_return`` hypotheses per prompt (<= N)."""
    num_beams: int
    n_keep: int
    length_penalty: float = 1.0
    early_stopping: object = False
    num_return: int = 1

    def code(self) -> int:
        if self.early_stopping == "never":
            return 2
        if isinstance(self.early_stopping, bool):
            return int(self.early_stopping)
        raise ValueError(f"early_stopping must be True, False or 'never', not {self.early_stopping!r}")


@dataclass
class Lookup:
    """Prompt-lookup decoding of a generate call (fo1_lookup_desc): ``num_tokens`` drafts per step (HF's prompt_lookup_num_tokens; the
    device proposes at most 16), ``max_ngram`` (HF's max_matching_ngram_size) and ``corpus``, one id list per sequence (HF's prompt
    ``input_ids``; None: empty corpora, only the emitted tokens are searched)."""
    num_tokens: int
    max_ngram: int = 2
    corpus: Optional[Sequence[Sequence[int]]] = None


@dataclass(frozen=True)
class ProcessorSet:
    """One sequence's logits processors (include/fo1.h, fo1_processor_desc), HF's semantics and order.  0 / empty: off.
    ``eos_token_ids``: the ids MinLength and MinNewTokens mask (HF's eos_token_id, not the stop list).  ``sequence_bias``: ((ids,
    bias), ...) in HF's dict order; ``bad_words_ids``: (ids, ...) with HF's eos filtering already applied."""
    no_repeat_ngram_size: int = 0
    min_length: int = 0
    min_new_tokens: int = 0
    eos_token_ids: Tuple[int, ...] = ()
    suppress_tokens: Tuple[int, ...] = ()
    begin_suppress_tokens: Tuple[int, ...] = ()
    sequence_bias: Tuple[Tuple[Tuple[int, ...], float], ...] = ()
    bad_words_ids: Tuple[Tuple[int, ...], ...] = ()


@dataclass
class Processors:
    """Logits processors of a generate call: ``sets[b]``, sequence b's ProcessorSet or None (its rows are never edited), and
    ``prompts[b]``, its prompt ids as the caller passes them (placeholders included; None: the pipeline fills in each sample's
    ``input_ids``).  Equal sets are packed once."""
    sets: Sequence[Optional[ProcessorSet]]
    prompts: Optional[Sequence[Sequence[int]]] = None


def _processor_desc(pr: Processors, B: int):
    """(ProcessorDesc, keep-alive) of a call with B sequences; the sets deduplicated."""
    if len(pr.sets) != B or pr.prompts is None or len(pr.prompts) != B:
        raise ValueError(f"processors: {len(pr.sets)} sets / {None if pr.prompts is None else len(pr.prompts)} prompts for {B} sequences")
    uniq, seq_set = {}, []
    for s in pr.sets:
        seq_set.append(-1 if s is None else uniq.setdefault(s, len(uniq)))
    sets = list(uniq)
    ids, bias = [], []
    offs = {}
    for key, get in (("eos", lambda s: s.eos_token_ids), ("sup", lambda s: s.suppress_tokens), ("bsup", lambda s: s.begin_suppress_tokens)):
        offs[key] = [len(ids)]
        for s in sets:
            ids.extend(int(t) for t in get(s))
            offs[key].append(len(ids))
    # the sequence list: every set's bias sequences, then every set's bad words
    seq_offsets = [len(ids)]
    for key, get in (("bias", lambda s: s.sequence_bias), ("bad", lambda s: [(w, 0.0) for w in s.bad_words_ids])):
        offs[key] = [len(bias)]
        for s in sets:
            for w, v in get(s):
                ids.extend(int(t) for t in w)
                seq_offsets.append(len(ids))
                bias.append(float(v))
            offs[key].append(len(bias))
    flat = [int(t) for p in pr.prompts for t in p]
    poff = [0]
    for p in pr.prompts:
        poff.append(poff[-1] + len(p))
    i32 = lambda v: (C.c_int32 * max(len(v), 1))(*v)
    S = len(sets)
    keep = dict(seq_set=i32(seq_set), prompt=i32(flat), poff=i32(poff), ng=i32([s.no_repeat_ngram_size for s in sets]),
                ml=i32([s.min_length for s in sets]), mn=i32([s.min_new_tokens for s in sets]), eos=i32(offs["eos"]), sup=i32(offs["sup"]),
                bsup=i32(offs["bsup"]), bias_off=i32(offs["bias"]), bad_off=i32(offs["bad"]), seq_off=i32(seq_offsets),
                bias=(C.c_float * max(len(bias), 1))(*bias), ids=i32(ids))
    desc = _lib.ProcessorDesc(S, keep["seq_set"], keep["prompt"], keep["poff"], keep["ng"], keep["ml"], keep["mn"], keep["eos"], keep["sup"],
                              keep["bsup"], keep["bias_off"], keep["bad_off"], len(bias), keep["seq_off"], keep["bias"], len(ids), keep["ids"])
    return desc, keep


def logits_process(logits: torch.Tensor, processors: Processors, outputs: Optional[torch.Tensor], cols: Sequence[int]) -> None:
    """fo1_logits_process: the row routine alone.  ``logits`` fp32 [n, V] on the device, edited in place; row r is sequence r of
    ``processors`` at output column ``cols[r]`` with emitted tokens ``outputs[r, :cols[r]]`` (int32 [n, >= max cols], device)."""
    n, V = logits.shape
    desc, _keep = _processor_desc(processors, n)
    out = outputs.to(logits.device, torch.int32).contiguous() if outputs is not None else None
    check(lib().fo1_logits_process(logits.data_ptr(), logits.stride(0), n, V, C.byref(desc), out.data_ptr() if out is not None else None,
                                   out.stride(0) if out is not None else 0, (C.c_int32 * n)(*[int(c) for c in cols]), _stream()),
          "fo1_logits_process")


def _lookup_desc(lookup: Lookup, B: int, dev):
    """(LookupDesc, keep-alive, steps, accepted) of a call with B sequences."""
    corpus = lookup.corpus if lookup.corpus is not None else [[] for _ in range(B)]
    if len(corpus) != B:
        raise ValueError(f"lookup corpus: {len(corpus)} id lists for {B} sequences")
    flat = [int(t) for c in corpus for t in c]
    offs = [0]
    for c in corpus:
        offs.append(offs[-1] + len(c))
    ids = (C.c_int32 * max(len(flat), 1))(*flat)
    off = (C.c_int32 * (B + 1))(*offs)
    steps = torch.zeros((B,), dtype=torch.int32, device=dev)
    acc = torch.zeros((B,), dtype=torch.int32, device=dev)
    desc = _lib.LookupDesc(int(lookup.num_tokens), int(lookup.max_ngram), ids, off, steps.data_ptr(), acc.data_ptr())
    return desc, (ids, off), steps, acc


def lookup_drafts(corpus: torch.Tensor, lens: torch.Tensor, num_tokens: int, max_ngram: int, stop_ids: Sequence[int],
                  emitted: Optional[torch.Tensor] = None, max_new_tokens: int = 0):
    """fo1_lookup_drafts: the draft rule alone.  ``corpus`` int32 [B, ld] on the device, ``lens`` int32 [B] -> (drafts int32
    [B, num_tokens], n_draft int32 [B]).  ``emitted`` (int32 [B]) with ``max_new_tokens`` caps the drafts at max_new - emitted - 1."""
    B = corpus.shape[0]
    dev = corpus.device
    corpus, lens = corpus.to(torch.int32).contiguous(), lens.to(dev, torch.int32).contiguous()
    st = torch.tensor([int(x) for x in stop_ids] or [0], dtype=torch.int32, device=dev)
    drafts = torch.zeros((B, num_tokens), dtype=torch.int32, device=dev)
    nd = torch.zeros((B,), dtype=torch.int32, device=dev)
    em = emitted.to(dev, torch.int32).contiguous() if emitted is not None else None
    check(lib().fo1_lookup_drafts(corpus.data_ptr(), corpus.stride(0), lens.data_ptr(), B, int(num_tokens), int(max_ngram), st.data_ptr(),
                                  len(stop_ids), em.data_ptr() if em is not None else None, int(max_new_tokens), drafts.data_ptr(),
                                  nd.data_ptr(), _stream()), "fo1_lookup_drafts")
    return drafts, nd


def _engine_generate(self, inputs_embeds: torch.Tensor, position_ids: torch.Tensor, seq_lens: Sequence[int],
                     rope_deltas: Sequence[int], max_new_tokens: int, stop_ids: Sequence[int], pad_id: int,
                     want_prefill_logits: bool = False, want_all_logits: bool = False, early_exit_interval: int = 8,
                     sampling: Optional[Sampling] = None, want_logprobs: bool = False, want_scores: bool = False,
                     want_logits: bool = False, raw_rows: Optional[Sequence[int]] = None,
                     on_tokens: Optional[Callable[[int, int, "np.ndarray", "np.ndarray"], Optional[bool]]] = None,
                     prefix: Optional[Prefix] = None, beams: Optional[Beams] = None, lookup: Optional[Lookup] = None,
                     processors: Optional[Processors] = None):
    """Prefill + decode of a packed batch: greedy, or sampled per sequence when ``sampling`` is given.  position_ids int32
    [3, sum L].  Returns a dict of device tensors.

    Scoring (include/fo1.h, fo1_score_desc): ``want_logprobs`` adds ``logprobs`` fp32 [B, max_new] (the log-probability of each
    emitted token, 0 past ``lens``); ``want_scores`` / ``want_logits`` add ``scores`` / ``logits`` fp32 [max_new, B, V] (HF's
    output_scores / output_logits).  Each buffer is allocated only when asked for.  ``raw_rows`` (one 0 / 1 per sequence, with
    ``sampling``): 1 marks a greedy sequence (top_k 1, temperature 1) scored on its raw logits.  Tokens never depend on these.

    Streaming (include/fo1.h, fo1_stream_desc): ``on_tokens(lo, hi, tokens, lens)`` is called in the calling thread whenever the
    device has published new output columns: ``tokens`` int32 [B, hi - lo] (columns lo..hi-1, pad past a sequence's stop),
    ``lens`` int32 [B] (each sequence's length as of column hi).  Returning True stops every sequence after the next column the
    device records.  An exception from the callback (KeyboardInterrupt included) stops the device too, and is re-raised once it
    has stopped.  The outputs are bit-identical to the same call without ``on_tokens`` (up to where a stop was asked for).

    Shared prefixes (include/fo1.h, fo1_prefix_desc): with ``prefix``, ``seq_lens`` stay the full lengths and ``inputs_embeds`` /
    ``position_ids`` hold only each sequence's rows after its group's prefix.  Every output is bit-identical to the call on the
    full sequences; ``want_all_logits`` is refused.

    Beam search (include/fo1.h, fo1_beam_desc): with ``beams``, every prompt runs HF's beam search on its own N rows.  ``tokens``
    int32 [B * num_return, max_new] / ``lens`` [B * num_return] hold each prompt's best hypotheses, best first; added are
    ``sequence_scores`` fp32 [B * num_return], ``beam_indices`` int32 [B * num_return, max_new] (prompt * N + beam, -1 past the
    length) and ``beam_steps`` int32 [B] (the steps each prompt ran).  ``want_scores`` / ``want_logits`` give [max_new, B * N, V]
    log-prob / raw rows; ``want_logprobs`` [B * num_return, max_new] the returned tokens' log-probabilities.  ``raw_rows`` is unread.

    Prompt lookup (include/fo1.h, fo1_lookup_desc): with ``lookup``, each step drafts tokens from the sequence's corpus and verifies
    them in one step of B * (K + 1) rows on the per-kernel decode path.  Tokens, lengths, logprobs and the score rows up to each
    length are bit-identical to the same call on the per-kernel path without lookup (FO1_NO_MEGA=1); against the persistent
    kernel (B <= 32 by default) they agree as any two decode paths do (DESIGN.md §2).  ``steps_run`` counts verify steps; added
    are ``lookup_steps`` / ``lookup_accepted`` int32 [B] (verify steps each sequence took part in, drafts it accepted).

    Logits processors (include/fo1.h, fo1_processor_desc): with ``processors``, each sequence's rows are edited by its ProcessorSet
    before its token is chosen; a sequence without one is bit-identical to the call without processors.  ``logits`` stays raw,
    ``scores`` and ``logprobs`` follow the processed rows.

    Which options combine is the library's rule (include/fo1.h, fo1_llm_generate): a refused pair raises Fo1Error before anything
    is enqueued."""
    B = len(seq_lens)
    V = self.cfg.llm["vocab_size"]
    pre = [0] * B
    if prefix is not None:
        assert len(prefix.seq_group) == B, "one group index per sequence"
        pre = [int(prefix.lens[g]) if g >= 0 else 0 for g in prefix.seq_group]
    T = int(sum(seq_lens)) - sum(pre)
    assert inputs_embeds.shape == (T, self.cfg.llm["hidden_size"]) and inputs_embeds.dtype == torch.bfloat16
    inputs_embeds = inputs_embeds.contiguous()
    position_ids = position_ids.to(self.device, torch.int32).contiguous()
    assert position_ids.shape == (3, T)
    # beam search returns num_return hypotheses per prompt and scores each of its N beam rows
    R, S = (B * int(beams.num_return), B * int(beams.num_beams)) if beams is not None else (B, B)
    toks = torch.empty((R, max(max_new_tokens, 1)), dtype=torch.int32, device=self.device)
    lens = torch.zeros((R,), dtype=torch.int32, device=self.device)
    pl = torch.empty((B, V), dtype=torch.float32, device=self.device) if want_prefill_logits else None
    al = torch.empty((T, V), dtype=torch.float32, device=self.device) if want_all_logits else None
    lp = torch.empty((R, max_new_tokens), dtype=torch.float32, device=self.device) if want_logprobs else None
    sc = torch.empty((max_new_tokens, S, V), dtype=torch.float32, device=self.device) if want_scores else None
    lg = torch.empty((max_new_tokens, S, V), dtype=torch.float32, device=self.device) if want_logits else None
    d = GenerateDescC()
    d.n_seqs = B
    sl = (C.c_int32 * B)(*[int(x) for x in seq_lens])
    dev_deltas = rope_deltas if isinstance(rope_deltas, torch.Tensor) else None       # device int32 [B] from splice_plan_batch
    rd = (C.c_int32 * B)(*([0] * B if dev_deltas is not None else [int(x) for x in rope_deltas]))
    if dev_deltas is not None:
        assert dev_deltas.is_cuda and dev_deltas.dtype == torch.int32 and dev_deltas.numel() == B
        d.rope_deltas_device = dev_deltas.data_ptr()
    st = (C.c_int32 * max(len(stop_ids), 1))(*[int(x) for x in stop_ids])
    d.seq_lens, d.rope_deltas, d.stop_ids, d.n_stop_ids = sl, rd, st, len(stop_ids)
    d.inputs_embeds, d.position_ids = inputs_embeds.data_ptr(), position_ids.data_ptr()
    d.max_new_tokens, d.pad_id = max_new_tokens, pad_id
    d.out_tokens, d.out_lens = toks.data_ptr(), lens.data_ptr()
    d.prefill_logits = pl.data_ptr() if pl is not None else None
    d.all_logits = al.data_ptr() if al is not None else None
    d.early_exit_interval = early_exit_interval
    ptr = lambda t: t.data_ptr() if t is not None else None
    if sampling is not None:
        sd, _keep = _lib.sampling_desc(sampling.temperature, sampling.top_p, sampling.top_k, sampling.seed)
        assert len(sampling.temperature) == B, "one sampling parameter set per sequence"
        d.sampling = C.pointer(sd)
    extra = {}
    if beams is not None:
        seq_scores = torch.empty((R,), dtype=torch.float32, device=self.device)
        bidx = torch.empty((R, max(max_new_tokens, 1)), dtype=torch.int32, device=self.device)
        steps = torch.zeros((B,), dtype=torch.int32, device=self.device)
        bd = _lib.BeamDesc(int(beams.num_beams), int(beams.n_keep), float(beams.length_penalty), beams.code(), int(beams.num_return),
                           seq_scores.data_ptr(), bidx.data_ptr(), steps.data_ptr(), ptr(sc), ptr(lg), ptr(lp))
        d.beam = C.pointer(bd)
        extra.update(sequence_scores=seq_scores, beam_indices=bidx, beam_steps=steps)
    elif lp is not None or sc is not None or lg is not None:
        rr = (C.c_int32 * B)(*[int(x) for x in raw_rows]) if raw_rows is not None else None
        assert raw_rows is None or len(raw_rows) == B, "one raw_rows flag per sequence"
        scd = _lib.ScoreDesc(ptr(lp), ptr(sc), ptr(lg), rr)
        d.scores = C.pointer(scd)

    if prefix is not None:
        G = len(prefix.lens)
        pe = prefix.embeds.contiguous()
        pp = prefix.position_ids.to(self.device, torch.int32).contiguous()
        assert pe.dtype == torch.bfloat16 and pe.shape == (sum(int(x) for x in prefix.lens), self.cfg.llm["hidden_size"])
        assert pp.shape == (3, pe.shape[0])
        px = _lib.PrefixDesc(G, (C.c_int32 * max(G, 1))(*[int(x) for x in prefix.lens]), pe.data_ptr(), pp.data_ptr(),
                             (C.c_int32 * B)(*[int(g) for g in prefix.seq_group]))
        d.prefix = C.pointer(px)

    if processors is not None and any(x is not None for x in processors.sets):
        prd, _pr_keep = _processor_desc(processors, B)
        d.processors = C.pointer(prd)

    if lookup is not None:
        lk, _lk_keep, extra["lookup_steps"], extra["lookup_accepted"] = _lookup_desc(lookup, B, self.device)
        d.lookup = C.pointer(lk)

    L = lib()

    def launch(stream, st=None):
        d.stream = C.pointer(st) if st is not None else None
        check(L.fo1_llm_generate(self._h, C.byref(d), stream), "fo1_llm_generate")
    if on_tokens is None:
        launch(_stream())
    else:
        self._run_streamed(launch, B, max_new_tokens, on_tokens)
    out = dict(tokens=toks, lens=lens, prefill_logits=pl, all_logits=al, steps_run=d.steps_run, **extra)
    if want_logprobs:
        out["logprobs"] = lp
    if want_scores:
        out["scores"] = sc
    if want_logits:
        out["logits"] = lg
    return out


IGNORE_INDEX = -100


def _engine_loglik(self, inputs_embeds: torch.Tensor, position_ids: torch.Tensor, seq_lens: Sequence[int], targets,
                   prefix: Optional[Prefix] = None, want_greedy: bool = False, want_all_logits: bool = False, want_lse: bool = False):
    """Teacher-forced scoring of a packed batch (fo1_llm_loglik): the prefill of generate, then the log-likelihood of each scored
    row's target from the LM head, without a vocabulary-wide matrix.  ``targets``: int [sum L] over the rows of the full sequences
    (HF labels already shifted by one within each sequence), -100 = not scored; a host sequence or a tensor (copied to the host).
    ``prefix``: as generate's (``inputs_embeds`` / ``position_ids`` then hold each sequence's own rows only).  Returns a dict of device
    tensors: ``logprobs`` fp32 [sum L] (0 where not scored), ``seq_logprob`` fp64 [B], ``seq_count`` int32 [B]; with ``want_greedy``
    ``greedy`` int32 [sum L] (1: the target is the row's lowest-index maximum); with ``want_all_logits`` ``all_logits`` fp32 [sum L, V]
    (refused with a prefix); with ``want_lse`` ``lse`` / ``target_logits`` fp32 [n_scored] of the scored rows in row order."""
    import numpy as np
    B = len(seq_lens)
    pre = [0] * B
    if prefix is not None:
        assert len(prefix.seq_group) == B, "one group index per sequence"
        pre = [int(prefix.lens[g]) if g >= 0 else 0 for g in prefix.seq_group]
    rows = int(sum(int(x) for x in seq_lens))
    T = rows - sum(pre)
    assert inputs_embeds.shape == (T, self.cfg.llm["hidden_size"]) and inputs_embeds.dtype == torch.bfloat16
    inputs_embeds = inputs_embeds.contiguous()
    position_ids = position_ids.to(self.device, torch.int32).contiguous()
    assert position_ids.shape == (3, T)
    tg = np.ascontiguousarray(targets.cpu().numpy() if isinstance(targets, torch.Tensor) else np.asarray(targets), dtype=np.int32)
    assert tg.shape == (rows,), "one target per row of the full sequences"
    n_scored = int((tg != IGNORE_INDEX).sum())
    V = self.cfg.llm["vocab_size"]
    dev = self.device
    out = dict(logprobs=torch.empty(rows, dtype=torch.float32, device=dev), seq_logprob=torch.empty(B, dtype=torch.float64, device=dev),
               seq_count=torch.empty(B, dtype=torch.int32, device=dev))
    if want_greedy:
        out["greedy"] = torch.empty(rows, dtype=torch.int32, device=dev)
    if want_all_logits:
        out["all_logits"] = torch.empty((rows, V), dtype=torch.float32, device=dev)
    if want_lse:
        out["lse"] = torch.empty(max(n_scored, 1), dtype=torch.float32, device=dev)[:n_scored]
        out["target_logits"] = torch.empty(max(n_scored, 1), dtype=torch.float32, device=dev)[:n_scored]
    ptr = lambda k: out[k].data_ptr() if k in out else None
    d = _lib.LoglikDesc()
    d.n_seqs = B
    d.seq_lens = (C.c_int32 * B)(*[int(x) for x in seq_lens])
    d.inputs_embeds, d.position_ids = inputs_embeds.data_ptr(), position_ids.data_ptr()
    d.targets = tg.ctypes.data_as(C.POINTER(C.c_int32))
    d.logprobs, d.greedy, d.seq_logprob, d.seq_count = ptr("logprobs"), ptr("greedy"), ptr("seq_logprob"), ptr("seq_count")
    d.all_logits, d.lse, d.target_logits = ptr("all_logits"), ptr("lse"), ptr("target_logits")
    if prefix is not None:
        G = len(prefix.lens)
        pe = prefix.embeds.contiguous()
        pp = prefix.position_ids.to(dev, torch.int32).contiguous()
        assert pe.dtype == torch.bfloat16 and pe.shape == (sum(int(x) for x in prefix.lens), self.cfg.llm["hidden_size"])
        assert pp.shape == (3, pe.shape[0])
        px = _lib.PrefixDesc(G, (C.c_int32 * max(G, 1))(*[int(x) for x in prefix.lens]), pe.data_ptr(), pp.data_ptr(),
                             (C.c_int32 * B)(*[int(g) for g in prefix.seq_group]))
        d.prefix = C.pointer(px)
    check(lib().fo1_llm_loglik(self._h, C.byref(d), _stream()), "fo1_llm_loglik")
    return out


class SlotPool:
    """In-flight batching over the engine (include/fo1.h, fo1_slots_*): ``n_slots`` K/V cache slots of ``cap`` rows and their decode
    state live across calls.  ``admit`` prefills requests into free slots, ``decode(exit_at)`` decodes every slot until at most
    ``exit_at`` requests still run, and a finished slot's row of ``tokens`` int32 [n_slots, max_new_tokens] / ``lens`` /
    ``finished`` (device) stays valid until the slot is admitted again.  Each request's tokens and length equal those of a static
    Engine.generate of ``n_slots`` sequences on the same decode path.  While the pool is open, Engine.generate raises."""

    def __init__(self, engine: Engine, n_slots: int, cap: int, max_new_tokens: int, stop_ids: Sequence[int], pad_id: int,
                 sampled: bool = False, early_exit_interval: int = 8):
        dev = engine.device
        self.eng, self.n_slots, self.cap, self.max_new_tokens = engine, int(n_slots), int(cap), int(max_new_tokens)
        self.tokens = torch.empty((self.n_slots, self.max_new_tokens), dtype=torch.int32, device=dev)
        self.lens = torch.zeros((self.n_slots,), dtype=torch.int32, device=dev)
        self.finished = torch.ones((self.n_slots,), dtype=torch.int32, device=dev)
        st = (C.c_int32 * max(len(stop_ids), 1))(*[int(x) for x in stop_ids])
        d = _lib.SlotsDesc(self.n_slots, self.cap, self.max_new_tokens, st, len(stop_ids), int(pad_id), int(bool(sampled)),
                           int(early_exit_interval), self.tokens.data_ptr(), self.lens.data_ptr(), self.finished.data_ptr())
        check(lib().fo1_slots_open(engine._h, C.byref(d), _stream()), "fo1_slots_open")
        self.open = True

    def admit(self, slots: Sequence[int], inputs_embeds: torch.Tensor, position_ids: torch.Tensor, seq_lens: Sequence[int],
              rope_deltas: torch.Tensor, max_new_tokens: Sequence[int], sampling: Optional[Sampling] = None,
              processors: Optional[Processors] = None) -> None:
        """Prefill len(slots) requests (packed bf16 embeddings [sum L, hidden], int32 positions [3, sum L], device int32 rope deltas
        [n]) into ``slots`` and record their column 0; ``max_new_tokens``, ``sampling`` and ``processors`` per request."""
        n = len(slots)
        emb = inputs_embeds.contiguous()
        pos = position_ids.to(self.eng.device, torch.int32).contiguous()
        rd = rope_deltas.to(self.eng.device, torch.int32).contiguous()
        assert emb.dtype == torch.bfloat16 and emb.shape == (int(sum(seq_lens)), self.eng.cfg.llm["hidden_size"])
        assert pos.shape == (3, emb.shape[0]) and rd.numel() == n and len(seq_lens) == n and len(max_new_tokens) == n
        sd = keep = None
        if sampling is not None:
            sd, keep = _lib.sampling_desc(sampling.temperature, sampling.top_p, sampling.top_k, sampling.seed)
        a = _lib.SlotsAdmitDesc(n, (C.c_int32 * n)(*[int(x) for x in slots]), (C.c_int32 * n)(*[int(x) for x in seq_lens]), emb.data_ptr(),
                                pos.data_ptr(), rd.data_ptr(), (C.c_int32 * n)(*[int(x) for x in max_new_tokens]),
                                C.pointer(sd) if sd is not None else None)
        if processors is not None and any(x is not None for x in processors.sets):
            prd, keep2 = _processor_desc(processors, n)
            a.processors = C.pointer(prd)
        check(lib().fo1_slots_admit(self.eng._h, C.byref(a), _stream()), "fo1_slots_admit")

    def decode(self, exit_at: int) -> int:
        """Decode until at most ``exit_at`` requests run; -> the decode steps run (synchronises)."""
        steps = C.c_int32()
        check(lib().fo1_slots_decode(self.eng._h, int(exit_at), C.byref(steps), _stream()), "fo1_slots_decode")
        return steps.value

    def close(self) -> None:
        if self.open:
            self.open = False
            check(lib().fo1_slots_close(self.eng._h), "fo1_slots_close")

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def prefix_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, prefix_lens: Sequence[int], own_lens: Sequence[int],
                     q_heads: int, kv_heads: int, scale: float) -> torch.Tensor:
    """fo1_prefix_attention: own rows q bf16 [sum own, q_heads * 128] (pitch = row stride) against the caches bf16 [n, cap, kv_heads * 128]:
    own row i of sequence b attends cache keys 0 .. prefix_lens[b] + i of b.  -> bf16 [sum own, q_heads * 128]."""
    n, cap, kvd = k_cache.shape
    assert q.dtype == k_cache.dtype == v_cache.dtype == torch.bfloat16 and q.stride(1) == 1 and k_cache.is_contiguous() and v_cache.is_contiguous()
    out = torch.empty((q.shape[0], q_heads * 128), dtype=torch.bfloat16, device=q.device)
    d = _lib.PrefixAttnDesc(q.data_ptr(), q.stride(0), k_cache.data_ptr(), v_cache.data_ptr(), n, cap, (C.c_int32 * n)(*[int(x) for x in prefix_lens]),
                            (C.c_int32 * n)(*[int(x) for x in own_lens]), q_heads, kv_heads, 128, scale, out.data_ptr(), out.stride(0))
    check(lib().fo1_prefix_attention(C.byref(d), _stream()), "fo1_prefix_attention")
    return out


def sample_tokens(logits: torch.Tensor, temperature: Sequence[float], top_p: Sequence[float], top_k: Sequence[int], seed: Sequence[int],
                  step) -> torch.Tensor:
    """One sampled token per row of fp32 logits [n, V] on the device (fo1_sample_tokens).  ``step``: int (every row) or a device
    int32 tensor [n], the Philox counter of each row.  -> int32 [n] on the device."""
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    n, V = logits.shape
    if not isinstance(step, torch.Tensor):
        step = torch.full((n,), int(step), dtype=torch.int32, device=logits.device)
    step = step.to(logits.device, torch.int32).contiguous()
    out = torch.empty((n,), dtype=torch.int32, device=logits.device)
    L = lib()
    ws = torch.empty((max(int(L.fo1_sample_tokens_workspace_bytes(n)), 1),), dtype=torch.uint8, device=logits.device)
    sd, _keep = _lib.sampling_desc(temperature, top_p, top_k, seed)
    check(L.fo1_sample_tokens(C.c_void_p(logits.data_ptr()), logits.stride(0), n, V, C.byref(sd), C.c_void_p(step.data_ptr()),
                              C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), _stream()), "fo1_sample_tokens")
    return out


def score_rows(logits: torch.Tensor, tokens: torch.Tensor, temperature: Optional[Sequence[float]] = None,
               top_p: Optional[Sequence[float]] = None, top_k: Optional[Sequence[int]] = None, raw_rows: Optional[Sequence[int]] = None,
               want_scores: bool = False):
    """The scoring of a decode step for arbitrary tokens (fo1_score_rows): fp32 logits [n, V] on the device, tokens [n] ->
    (logprobs fp32 [n], scores fp32 [n, V] or None).  Without sampling parameters every row is scored raw; ``raw_rows`` marks
    single rows raw.  A token outside a row's kept set gets -inf."""
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    n, V = logits.shape
    tokens = tokens.to(logits.device, torch.int32).contiguous()
    assert tokens.numel() == n, "one token per row"
    lp = torch.empty((n,), dtype=torch.float32, device=logits.device)
    sc = torch.empty((n, V), dtype=torch.float32, device=logits.device) if want_scores else None
    sd = keep = None
    if temperature is not None:
        sd, keep = _lib.sampling_desc(temperature, top_p, top_k, [0] * n)
    rr = (C.c_int32 * n)(*[int(x) for x in raw_rows]) if raw_rows is not None else None
    check(lib().fo1_score_rows(C.c_void_p(logits.data_ptr()), logits.stride(0), n, V, C.byref(sd) if sd is not None else None, rr,
                               C.c_void_p(tokens.data_ptr()), C.c_void_p(lp.data_ptr()), C.c_void_p(sc.data_ptr()) if sc is not None else None,
                               V, _stream()), "fo1_score_rows")
    return lp, sc


_POLL_S = 2e-4      # host poll period of a streamed generate: a fraction of a decode step (about 3 ms at the 3B shape, B = 1)


def _engine_stream_buffers(self, B: int, T: int):
    """The pinned host buffers a streamed generate publishes into (fo1_stream_desc), allocated once and grown when a call needs
    more: -> (tokens int32 [>= B * T], lens int32 [>= B], control int32 [32]: progress at [0], cancel at [16], a cache line apart)."""
    buf = getattr(self, "_stream_buf", None)
    if buf is None or buf[0].numel() < B * T or buf[1].numel() < B:
        old = buf or (torch.empty(0), torch.empty(0), None)
        buf = (torch.empty(max(B * T, old[0].numel()), dtype=torch.int32, pin_memory=True),
               torch.empty(max(B, old[1].numel()), dtype=torch.int32, pin_memory=True),
               old[2] if old[2] is not None else torch.zeros(32, dtype=torch.int32, pin_memory=True))
        self._stream_buf = buf
    return buf


def _engine_run_streamed(self, launch, B: int, T: int, on_tokens) -> None:
    """Run ``launch(stream, StreamDesc)`` (one streamed fo1_llm_generate call) in a worker thread and deliver the published columns
    to ``on_tokens`` from this thread.  The worker enqueues on this thread's current stream, on the engine's device (the library
    does not set the device), and records an event after the call; the per-kernel path's host loop blocks in that call, so it
    must not run where the polling does.  Polling ends on `done`, on the worker's failure (its Fo1Error is raised), or once the
    event has completed (after one more drain), so a failed launch never leaves it spinning."""
    import numpy as np
    tok_t, lens_t, ctl_t = self._stream_buffers(B, max(T, 1))      # (a buffer is never empty: NULL is refused)
    tok = tok_t.numpy()[:B * T].reshape(B, T)
    lens, ctl = lens_t.numpy()[:B], ctl_t.numpy()
    ctl[0] = 0                       # progress (the call stores 0 too; this keeps a previous call's `done` from being read first)
    ctl[16] = 0                      # cancel
    prog, cancel = ctl_t.data_ptr(), ctl_t.data_ptr() + 16 * 4
    st = _lib.StreamDesc(tok_t.data_ptr(), lens_t.data_ptr(), prog, cancel)
    L = lib()
    stream = torch.cuda.current_stream(self.device)
    finished_ev = torch.cuda.Event()
    failure: List[BaseException] = []

    def work():
        try:
            with torch.cuda.device(self.device):
                launch(C.c_void_p(stream.cuda_stream), st)
                finished_ev.record(stream)
        except BaseException as e:  # noqa: BLE001 -- handed to the polling thread
            failure.append(e)

    worker = threading.Thread(target=work, name="fo1-generate-streamed", daemon=True)
    worker.start()
    seen = 0
    try:
        while True:
            finished = not worker.is_alive() and (bool(failure) or finished_ev.query())     # read BEFORE the last drain
            if failure:
                raise failure[0]
            p = int(L.fo1_stream_progress(prog))
            cols = p & (_lib.FO1_STREAM_DONE - 1)
            if cols > seen:
                lo, seen = seen, cols
                if on_tokens(lo, cols, tok[:, lo:cols].copy(), np.minimum(lens, cols).astype(np.int32)):
                    L.fo1_stream_cancel(cancel)
            if p & _lib.FO1_STREAM_DONE or finished:
                break
            time.sleep(_POLL_S)
    except BaseException:
        L.fo1_stream_cancel(cancel)     # the device stops within one step; wait for it, then re-raise
        worker.join()
        if not failure:
            stream.synchronize()
        raise
    worker.join()
    if failure:
        raise failure[0]


Engine.build_embeds = _engine_build_embeds
Engine.generate = _engine_generate
Engine.loglik = _engine_loglik
Engine._stream_buffers = _engine_stream_buffers
Engine._run_streamed = _engine_run_streamed
Engine.sample_tokens = staticmethod(sample_tokens)
Engine.lookup_drafts = staticmethod(lookup_drafts)
Engine.prefix_attention = staticmethod(prefix_attention)
Engine.score_rows = staticmethod(score_rows)


def splice_plan_batch(prompts: Sequence[Sequence[int]], image_grids: Sequence[Sequence[Tuple[int, int]]], n_regions: Sequence[int], device,
                      image_token_id: int = 151655, video_token_id: int = 151656, vision_start_token_id: int = 151652, merge: int = 2,
                      image_placeholder: int = -200, region_placeholder: int = -300, row_src: Optional[Sequence[int]] = None):
    """The splice + M-RoPE bookkeeping of a whole batch in ONE launch on the device (fo1_splice_plan_batch).  Per sample b:
    ``prompts[b]`` ids with placeholders, ``image_grids[b]`` its images' (gh, gw), ``n_regions[b]`` region rows.  Image rows /
    region rows of the batch are assumed packed back to back in sample order (what Fo1Pipeline.encode produces).  ``row_src``:
    sample b reads the image / region rows of sample row_src[b] <= b (same image and boxes); only the samples with row_src[b] == b
    have rows of their own, packed in their order.
    -> dict(kind, index, new_ids int32 [T]; position_ids int32 [3, T]; rope_delta int32 [B]) on the device, lens (host list)."""
    import numpy as np
    B = len(prompts)
    unit = merge * merge
    id_off = np.zeros(B + 1, np.int32); img_off = np.zeros(B + 1, np.int32); out_off = np.zeros(B + 1, np.int32)
    img_row = np.zeros(B, np.int32); reg_row = np.zeros(B, np.int32)
    rows_i = rows_r = 0
    for b in range(B):
        toks = sum(gh * gw // unit for gh, gw in image_grids[b])
        n_img_ph = sum(1 for t in prompts[b] if t == image_placeholder)
        id_off[b + 1] = id_off[b] + len(prompts[b]); img_off[b + 1] = img_off[b] + len(image_grids[b])
        # every image placeholder expands to its image's rows; more placeholders than images is reported per sample by the kernel
        exp = sum(gh * gw // unit for gh, gw in list(image_grids[b])[:n_img_ph])
        out_off[b + 1] = out_off[b] + len(prompts[b]) - min(n_img_ph, len(image_grids[b])) + exp
        src = b if row_src is None else int(row_src[b])
        if src != b:
            img_row[b] = img_row[src]; reg_row[b] = reg_row[src]
            continue
        img_row[b] = rows_i; reg_row[b] = rows_r
        rows_i += toks; rows_r += int(n_regions[b])
    T = int(out_off[B])
    host = np.concatenate([np.asarray([t for p in prompts for t in p], np.int32), id_off,
                           np.asarray([x for g in image_grids for hw in g for x in hw], np.int32).reshape(-1), img_off,
                           np.asarray(n_regions, np.int32), out_off, img_row, reg_row])
    d = torch.from_numpy(host).to(device, non_blocking=True)      # one H2D for every table
    cuts = np.cumsum([0, int(id_off[B]), B + 1, 2 * int(img_off[B]), B + 1, B, B + 1, B, B])
    v = [d[cuts[i]:cuts[i + 1]] for i in range(8)]
    out = torch.empty(6 * T + 2 * B, dtype=torch.int32, device=device)
    new_ids, kind, index, pos = out[:T], out[T:2 * T], out[2 * T:3 * T], out[3 * T:6 * T].view(3, T)
    delta, status = out[6 * T:6 * T + B], out[6 * T + B:]
    cfg = SpliceCfgC(image_token_id, video_token_id, vision_start_token_id, merge, image_placeholder, region_placeholder)
    L = lib()
    L.fo1_splice_plan_batch.restype = C.c_int
    L.fo1_splice_plan_batch.argtypes = [C.c_void_p] * 8 + [C.c_int32, C.c_int64, C.POINTER(SpliceCfgC)] + [C.c_void_p] * 7
    P = lambda t: C.c_void_p(t.data_ptr())
    check(L.fo1_splice_plan_batch(P(v[0]), P(v[1]), P(v[2]), P(v[3]), P(v[4]), P(v[5]), P(v[6]), P(v[7]), B, T, C.byref(cfg),
                                  P(new_ids), P(kind), P(index), P(pos), P(delta), P(status), _stream()), "fo1_splice_plan_batch")
    return dict(new_ids=new_ids, kind=kind, index=index, position_ids=pos, rope_delta=delta, status=status,
                lens=[int(out_off[b + 1] - out_off[b]) for b in range(B)])


def parse_predictions(tokens: torch.Tensor, lens: torch.Tensor, ground_ids: Tuple[int, int], objects_ids: Tuple[int, int],
                      region_ids: Sequence[int], newline_token_ids: Sequence[int] = (), vocab: int = 0, max_records: int = 256):
    """fo1_parse_predictions over a batch of decoded ids (device int32 [B, T], lens [B]) -> per sample list of
    (label first token, label end token, N or -1)."""
    import numpy as np
    B, T = tokens.shape
    dev = tokens.device
    rid = torch.tensor(list(region_ids), dtype=torch.int32, device=dev)
    bm = None
    if vocab > 0 and len(newline_token_ids):
        words = np.zeros((vocab + 31) // 32, np.uint32)
        for t in newline_token_ids:
            words[t >> 5] |= np.uint32(1 << (t & 31))
        bm = torch.from_numpy(words.view(np.int32)).to(dev)
    rec = torch.empty((B, max_records, 3), dtype=torch.int32, device=dev)
    cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
    L = lib()
    L.fo1_parse_predictions.restype = C.c_int
    L.fo1_parse_predictions.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    tokens = tokens.contiguous(); lens = lens.to(torch.int32).contiguous()
    check(L.fo1_parse_predictions(C.c_void_p(tokens.data_ptr()), tokens.stride(0), C.c_void_p(lens.data_ptr()), B, ground_ids[0], ground_ids[1],
                                  objects_ids[0], objects_ids[1], C.c_void_p(rid.data_ptr()), rid.numel(),
                                  C.c_void_p(bm.data_ptr()) if bm is not None else None, vocab, C.c_void_p(rec.data_ptr()), max_records,
                                  C.c_void_p(cnt.data_ptr()), _stream()), "fo1_parse_predictions")
    rec_h, cnt_h = rec.cpu().numpy(), cnt.cpu().numpy()
    return [[tuple(int(x) for x in rec_h[b, i]) for i in range(int(cnt_h[b]))] for b in range(B)]
