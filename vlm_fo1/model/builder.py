"""``load_pretrained_model`` with the reference's signature and return contract (vlm_fo1/model/builder.py:8-142):
``(tokenizer, model, (primary_image_processor, aux_image_processor))``.  Reads the checkpoint directory the same way
(config.json flags via getattr-with-default semantics, every ``*.safetensors`` shard, strict coverage of the two
towers' weights) and hands the tensors to the engine."""
from __future__ import annotations

import json
import os
from importlib import import_module
from types import SimpleNamespace

import torch

from vlm_fo1.model.fo1_model import Fo1ForCausalLM
from vlm_fo1.processors import AuxImageProcessor, PrimaryImageProcessor

DAVIT = {  # davit/configs.py:2-136
    "davit-base": dict(depths=[1, 1, 9, 1], dim_embed=[128, 256, 512, 1024], num_heads=[4, 8, 16, 32], num_groups=[4, 8, 16, 32], window_size=12),
    "davit-large": dict(depths=[1, 1, 9, 1], dim_embed=[256, 512, 1024, 2048], num_heads=[8, 16, 32, 64], num_groups=[8, 16, 32, 64], window_size=12),
}


def _strip(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def _mlp_depth(kind: str, identity_ok: bool) -> int:
    if kind == "identity" and identity_ok:
        return 0
    if kind == "linear":
        return 1
    if kind.startswith("mlp") and kind.endswith("x_gelu"):
        return int(kind[3:-6])
    raise ValueError(f"Unknown projector type: {kind}")                                   # multimodal_projector/builder.py:76,115


def load_pretrained_model(model_path, load_8bit=False, load_4bit=False, device="cuda"):
    if load_8bit or load_4bit:
        raise NotImplementedError("the fo1-b200 engine runs bf16 weights only")
    name = model_path.lower()
    if "vlm-fo1" not in name or not ("qwen2.5-vl" in name or "qwen2_5_vl" in name):
        # the reference dispatches on these substrings of the path (builder.py:35,39) and fails later otherwise
        raise ValueError(f"unsupported checkpoint path {model_path!r}: expected a 'vlm-fo1' + 'qwen2.5-vl' directory name")
    from safetensors.torch import load_file
    from transformers import AutoTokenizer
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    tokenizer = AutoTokenizer.from_pretrained(model_path, use_fast=False)
    raw = json.load(open(os.path.join(model_path, "config.json")))
    g = raw.get
    vc = raw["vision_config"]
    aux_name = str(g("mm_vision_tower_aux", "davit-large")).split("/")[-1].replace(".pth", "")
    if aux_name not in DAVIT:
        raise ValueError(f"Unknown aux vision tower: {aux_name}")                         # multimodal_encoder/builder.py:38
    use_fpn = bool(g("mm_use_simpleFPN_for_vt", False))
    if not g("mm_use_vision_tower_region_feature", False):
        raise ValueError("mm_use_vision_tower_region_feature=False is a dead configuration in the reference "
                         "(hybrid_finegrained_region_encoder.py:456 raises); not supported")
    # ---- the HFRE variant flags the reference reads in omchat_arch.py:17-31: honoured or refused, never ignored ----
    roi_size = int(g("mm_roi_output_size", 7))
    apply_pos = bool(g("mm_apply_position_embedding", True))
    pos_strategy = str(g("mm_pos_embedding_strategy", "bbox_based"))
    combination = str(g("mm_region_feature_combination", "concat"))
    unsupported = []
    if roi_size < 1 or roi_size > 16:
        unsupported.append(f"mm_roi_output_size={roi_size}")
    if apply_pos and pos_strategy != "bbox_based":
        unsupported.append(f"mm_pos_embedding_strategy={pos_strategy!r} (only 'bbox_based', hybrid_finegrained_region_encoder.py:436-467)")
    if combination != "concat":
        unsupported.append(f"mm_region_feature_combination={combination!r} (the mean / *_sep_pos paths hard-code ConvNeXt widths, :384-432)")
    for flag in ("mm_use_vt_region_feature_only", "mm_apply_region_layer_norm", "mm_use_separate_mlp_for_regions"):
        if g(flag, False):
            unsupported.append(f"{flag}=True")
    if unsupported:
        raise ValueError("checkpoint flags not supported by the fo1-b200 engine: " + "; ".join(unsupported))
    cfg = E.EngineConfig()
    cfg.vit = dict(depth=vc["depth"], hidden_size=vc["hidden_size"], num_heads=vc["num_heads"], intermediate_size=vc["intermediate_size"],
                   out_hidden_size=vc["out_hidden_size"], patch_size=vc.get("patch_size", 14), spatial_merge_size=vc.get("spatial_merge_size", 2),
                   temporal_patch_size=vc.get("temporal_patch_size", 2), in_channels=vc.get("in_chans", vc.get("in_channels", 3)),
                   window_size=vc.get("window_size", 112), fullatt_block_indexes=vc.get("fullatt_block_indexes", [7, 15, 23, 31]))
    cfg.davit = dict(DAVIT[aux_name])
    if "davit_depths" in raw:                     # fabricated reduced-depth checkpoints only
        cfg.davit["depths"] = list(raw["davit_depths"])
    cfg.fpn_out = 512 if use_fpn else 0
    cfg.region_dim = int(raw["mm_region_hidden_size"])
    cfg.proj_aux_layers = _mlp_depth(str(g("mm_projector_aux_type", "linear")), False)
    cfg.proj_img_layers = _mlp_depth(str(g("mm_projector_type", "linear")), True)
    cfg.llm = dict(num_hidden_layers=raw["num_hidden_layers"], hidden_size=raw["hidden_size"], num_attention_heads=raw["num_attention_heads"],
                   num_key_value_heads=raw["num_key_value_heads"], intermediate_size=raw["intermediate_size"], vocab_size=raw["vocab_size"],
                   rope_theta=raw.get("rope_theta", 1000000.0), rms_norm_eps=raw.get("rms_norm_eps", 1e-6),
                   mrope_section=raw["rope_scaling"]["mrope_section"], tie_word_embeddings=bool(g("tie_word_embeddings", False)))
    # ---- weights: every safetensors shard (builder.py:90-98) ----
    print(f"Loading weights from {model_path} ...")
    sd = {}
    for f in sorted(os.listdir(model_path)):
        if f.endswith(".safetensors"):
            sd.update(load_file(os.path.join(model_path, f), device="cpu"))
    vt = _strip(sd, "model.vision_tower.image_tower.")
    va = _strip(sd, "model.vision_tower_aux.image_tower.")
    if not vt or not va:
        print("No vision_tower weights found")
        raise Exception("No vision_tower weights found")                                  # builder.py:136-137
    sds = {"vit": vt, "davit": va, "proj_aux": _strip(sd, "model.mm_projector_aux.")}
    if use_fpn:
        sds["fpn"] = _strip(sd, "model.object_vp_extractor.simple_fpn.")
    if cfg.proj_img_layers:
        sds["proj_img"] = _strip(sd, "model.mm_projector.")
    llm = {k[len("model."):]: v for k, v in sd.items() if k.startswith("model.layers.") or k in ("model.embed_tokens.weight", "model.norm.weight")}
    if "lm_head.weight" in sd and not cfg.llm["tie_word_embeddings"]:
        llm["lm_head.weight"] = sd["lm_head.weight"]
    sds["llm"] = llm
    if device != "cuda":
        torch.cuda.set_device(torch.device(device))
    engine = CK.load_engine(cfg, sds, None)
    del sd, sds
    config = SimpleNamespace(**{k: v for k, v in raw.items() if not isinstance(v, dict)})
    config.mm_use_region_index_token = bool(g("mm_use_region_index_token", False))
    config.image_token_id = int(g("image_token_id", 151655)); config.video_token_id = int(g("video_token_id", 151656))
    config.vision_start_token_id = int(g("vision_start_token_id", 151652))
    gen_path = os.path.join(model_path, "generation_config.json")
    gen_cfg = json.load(open(gen_path)) if os.path.exists(gen_path) else {}
    eos = gen_cfg.get("eos_token_id", []) if os.path.exists(gen_path) else g("eos_token_id", [])
    stop_ids = [int(e) for e in (eos if isinstance(eos, list) else [eos]) if e is not None]
    # the sampling fields (top_k; the processors sampled decoding refuses) are read here and checked per call, never at load time
    model = Fo1ForCausalLM(engine, config, "fpn" if use_fpn else "concat", stop_ids, roi_size=roi_size, apply_pos_embed=apply_pos,
                           generation_config=gen_cfg)
    # the processors run on the engine's GPU (uint8 over PCIe; bit-identical to the host processors); FO1_HOST_PREPROCESS=1 keeps PIL / numpy
    pdev = None if os.environ.get("FO1_HOST_PREPROCESS") else engine.device
    primary = PrimaryImageProcessor(cfg.vit["patch_size"], cfg.vit["spatial_merge_size"], cfg.vit["temporal_patch_size"], 56 * 56, 2048 * 2048, device=pdev)
    aux = AuxImageProcessor(int(g("aux_image_size", 768)), str(g("aux_image_aspect_ratio", "squash")), device=pdev)
    return tokenizer, model, (primary, aux)
