"""Generate ``tests/golden/*.npz`` by running the REFERENCE's own modules -- TEST INFRASTRUCTURE ONLY.

Run in the build container (needs ``/root/reference``):  ``python oracle/gen_golden.py [stage ...]``
Stages: hfre fpn davit vit proj llm splice (default: all that are implemented).
The fixtures are small, committed, and replayed by ``tests/`` on machines without the reference.
Inputs are stored next to the outputs so the tests do not depend on RNG reproducibility.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
# make sure ``import vlm_fo1`` can only resolve to the reference, never to the repo's boundary mirror
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != REPO]
sys.path.insert(0, HERE)

import numpy as np
import torch

import ref_shim

GOLD = os.path.join(REPO, "tests", "golden")
os.makedirs(GOLD, exist_ok=True)


def bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def save(name: str, **arrays) -> None:
    out = {}
    for k, v in arrays.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        out[k] = np.asarray(v)
    # files stay below 1 MB: arrays are dealt, in order, into <name>.npz, <name>.part1.npz, ... (tests/golden_io.py merges them)
    parts, size = [{}], 0
    for k, v in out.items():
        if size + v.nbytes > 900_000 and parts[-1]:
            parts.append({}); size = 0
        parts[-1][k] = v; size += v.nbytes
    for i, part in enumerate(parts):
        path = os.path.join(GOLD, name + (".npz" if i == 0 else f".part{i}.npz"))
        np.savez_compressed(path, **part)
        print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


# ------------------------------------------------------------------------------------------ HFRE
def hfre_boxes(S: int, n_rand: int, gen: torch.Generator) -> torch.Tensor:
    """random interior boxes + the border / degenerate cases SURVEY.md appendix A lists."""
    w = torch.rand(n_rand, generator=gen) * (S / 2 - 4) + 4
    h = torch.rand(n_rand, generator=gen) * (S / 2 - 4) + 4
    x1 = torch.rand(n_rand, generator=gen) * (S - w)
    y1 = torch.rand(n_rand, generator=gen) * (S - h)
    rnd = torch.stack([x1, y1, x1 + w, y1 + h], dim=1)
    S_ = float(S)
    edge = torch.tensor([
        [0.0, 0.0, S_, S_],                     # whole image
        [0.0, 0.0, 1.0, 1.0],                   # < one cell, top-left corner
        [S_ - 0.1, S_ - 0.1, S_, S_],           # degenerate, bottom-right corner (max(size,1) pushes samples out)
        [2.0, S_ - 2.5, 9.0, S_ - 0.1],         # thin, on the bottom border
        [S_ - 0.8, 10.0, S_, 30.0],             # thin, on the right border
        [10.0, 10.0, 10.0, 10.0],               # zero-area
        [5.3, 7.7, 5.9, S_ - 3.0],              # very thin vertical
        [0.0, S_ / 2, S_, S_ / 2 + 0.5],        # very thin horizontal, full width
    ])
    return torch.cat([rnd, edge], dim=0).to(torch.float32)


def gen_hfre() -> None:
    hf, _ = ref_shim.load_hfre_only()
    gen = torch.Generator().manual_seed(1234)
    for tag, S, vt_S, chans, vt_c in (("small", 96, 98, (8, 16, 32, 64), 24), ("rect", 128, 126, (16, 16, 32, 32), 16)):
        # aux pyramid at strides 4/8/16/32 of an S x (S or 3S/4) image
        Sh, Sw = (S, S) if tag == "small" else (S, (S * 3) // 4)
        aux = [bf16_round(torch.randn(1, c, Sh // (4 << i), Sw // (4 << i), generator=gen)) for i, c in enumerate(chans)]
        boxes = hfre_boxes(min(Sh, Sw), 12, gen)
        gh, gw = vt_S // 14, (vt_S // 14 if tag == "small" else (vt_S // 14) - 2)
        sx, sy = (gw * 14) / Sw, (gh * 14) / Sh
        vt_boxes = boxes * torch.tensor([sx, sy, sx, sy])
        # variant A: four tap maps, concatenated by the module
        taps = [bf16_round(torch.randn(1, vt_c, gh, gw, generator=gen)) for _ in range(4)]
        D_a = sum(chans) + 4 * vt_c
        mod_a = hf.HFREModule(roi_output_size=7, region_feature_dim=D_a, apply_position_embedding=True,
                              pos_embedding_strategy="bbox_based", use_vision_tower_region_feature=True,
                              region_feature_combination="concat", vision_tower_region_feature_dim=4 * vt_c,
                              vision_tower_spatial_scale=1 / 14, use_simpleFPN_for_vt=False,
                              aux_vision_tower_spatial_scale=0.25)
        out_a = mod_a(aux_multi_level_features=[a.clone() for a in aux], aux_boxes=[boxes.clone()],
                      vt_multi_level_features=[t.clone() for t in taps], vt_boxes=[vt_boxes.clone()])
        # variant B: the module's SimpleFP is replaced by a fixed pyramid (the FPN itself is pinned
        # by the separate ``fpn`` fixture); everything after it is the reference's own code
        pyr = [bf16_round(torch.randn(1, vt_c, int(gh * f), int(gw * f), generator=gen)) for f in (4, 2, 1, 0.5)]
        D_b = sum(chans) + 4 * vt_c
        mod_b = hf.HFREModule(roi_output_size=7, region_feature_dim=D_b, apply_position_embedding=True,
                              pos_embedding_strategy="bbox_based", use_vision_tower_region_feature=True,
                              region_feature_combination="concat", vision_tower_region_feature_dim=4 * vt_c,
                              vision_tower_spatial_scale=1 / 14, use_simpleFPN_for_vt=False,
                              aux_vision_tower_spatial_scale=0.25)
        mod_b.use_simpleFPN_for_vt = True
        mod_b.simple_fpn = lambda x, _p=pyr: [p.clone() for p in _p]
        last_tap = taps[-1]
        out_b = mod_b(aux_multi_level_features=[a.clone() for a in aux], aux_boxes=[boxes.clone()],
                      vt_multi_level_features=last_tap.clone(), vt_boxes=[vt_boxes.clone()])
        # (aux-only, use_vision_tower_region_feature=False, raises UnboundLocalError in the reference
        #  at hybrid_finegrained_region_encoder.py:456 -- dead configuration, not pinned)
        save(f"hfre_{tag}", boxes=boxes, vt_boxes=vt_boxes, grid_hw=np.array([gh, gw]),
             **{f"aux{i}": a[0] for i, a in enumerate(aux)}, **{f"tap{i}": t[0] for i, t in enumerate(taps)},
             **{f"pyr{i}": p[0] for i, p in enumerate(pyr)},
             out_concat=out_a[0], out_fpn=out_b[0])


STAGES = {"hfre": gen_hfre}


# --------------------------------------------------------------------------- towers (reference modules)
def _bf16_params_(mod: torch.nn.Module) -> None:
    for prm in mod.parameters():
        prm.data = bf16_round(prm.data)


def _sd_bits(sd) -> dict:
    """state_dict -> {name: uint16 bf16 bit pattern} (values are already bf16-representable)."""
    return {"w::" + k: v.detach().to(torch.bfloat16).view(torch.int16).numpy() for k, v in sd.items()}


VIT_SMALL = dict(depth=4, hidden_size=64, num_heads=2, intermediate_size=88, out_hidden_size=48, patch_size=14,
                 spatial_merge_size=2, temporal_patch_size=2, in_channels=3, window_size=112, fullatt_block_indexes=[1, 3],
                 hidden_act="silu", in_chans=3, tokens_per_second=2)


def gen_vit() -> None:
    ref_shim.load_reference_package()
    from vlm_fo1.model.multimodal_encoder.qwen2_5_vl.configuration_qwen2_5_vl import Qwen2_5_VLVisionConfig
    from vlm_fo1.model.multimodal_encoder.qwen2_5_vl.modeling_qwen2_5_vl import Qwen2_5_VisionTransformerPretrainedModel
    from vlm_fo1.model.multimodal_encoder import qwen2_5_vl_encoder as enc
    torch.manual_seed(0)
    cfg = Qwen2_5_VLVisionConfig(**VIT_SMALL)
    enc.replace_qwen_vit_forward()
    model = Qwen2_5_VisionTransformerPretrainedModel._from_config(cfg, attn_implementation="eager").float().eval()
    for prm in model.parameters():  # the default init leaves norms at 1 / biases at 0: randomise so every term is exercised
        prm.data = torch.randn_like(prm) * (0.02 if prm.dim() > 1 else 0.3) + (1.0 if "norm" in "" else 0.0)
    for n, prm in model.named_parameters():
        if n.endswith("norm1.weight") or n.endswith("norm2.weight") or n.endswith("ln_q.weight"):
            prm.data = prm.data + 1.0
    _bf16_params_(model)
    model.init_vision_features_gather(enc.GATHER)
    out = {}
    int_tables = {}
    for tag, gh, gw in (("a", 6, 10), ("b", 8, 8)):
        px = bf16_round(torch.randn(gh * gw, 3 * 2 * 14 * 14))
        grid = torch.tensor([[1, gh, gw]])
        merged = model(px, grid_thw=grid)
        taps = enc.GATHER.extract_multi_level_features()[0]
        out[f"px_{tag}"] = px
        out[f"grid_{tag}"] = np.array([gh, gw])
        out[f"merged_{tag}"] = merged
        for i, t in enumerate(taps):
            out[f"tap{i}_{tag}"] = t[0].permute(1, 2, 0).contiguous()   # [gh, gw, C]
    # integer bookkeeping at the BASELINE grids (bit-exact targets)
    for gh, gw in ((6, 10), (8, 8), (32, 32), (46, 46), (64, 64), (28, 36), (96, 96), (2, 2), (4, 18)):
        wi, cu = model.get_window_index(torch.tensor([[1, gh, gw]]))
        cu = torch.unique_consecutive(torch.tensor(cu))
        int_tables[f"wi_{gh}x{gw}"] = wi.numpy().astype(np.int32)
        int_tables[f"cu_{gh}x{gw}"] = cu.numpy().astype(np.int32)
    save("vit_small", cfg_json=np.frombuffer(__import__("json").dumps(VIT_SMALL).encode(), dtype=np.uint8),
         **_sd_bits(model.state_dict()), **out, **int_tables)


DAVIT_SMALL = dict(depths=[1, 1, 2, 1], dim_embed=[32, 32, 64, 64], num_heads=[1, 1, 2, 2], num_groups=[1, 1, 2, 2],
                   patch_size=[7, 3, 3, 3], patch_stride=[4, 2, 2, 2], patch_padding=[3, 1, 1, 1],
                   patch_prenorm=[False, True, True, True], drop_path_rate=0.0, window_size=12)


def gen_davit() -> None:
    ref_shim.load_reference_package()
    from vlm_fo1.model.multimodal_encoder.davit.modeling_davit import DaViT
    from types import SimpleNamespace
    torch.manual_seed(1)
    model = DaViT.from_config(SimpleNamespace(**DAVIT_SMALL)).float().eval()
    for n, prm in model.named_parameters():
        if prm.dim() == 1:
            prm.data = torch.randn_like(prm) * 0.2 + (1.0 if n.endswith("norm.weight") else 0.0)
        else:
            prm.data = torch.randn_like(prm) * 0.05
    _bf16_params_(model)
    out = {}
    for tag, H, W in (("a", 72, 104), ("b", 96, 96)):
        img = bf16_round(torch.randn(1, 3, H, W))
        feats = model(img)["image_features"]
        out[f"img_{tag}"] = img[0]
        for i, f in enumerate(feats):
            out[f"stage{i}_{tag}"] = f[0].permute(1, 2, 0).contiguous()
    save("davit_small", cfg_json=np.frombuffer(__import__("json").dumps(DAVIT_SMALL).encode(), dtype=np.uint8),
         **_sd_bits(model.state_dict()), **out)


def gen_fpn() -> None:
    _, fpn = ref_shim.load_hfre_only()
    torch.manual_seed(2)
    model = fpn.SimpleFP(out_channels=32, norm="LN", square_pad=0, dim=64, stride=14).float().eval()
    for n, prm in model.named_parameters():
        if prm.dim() == 1:
            prm.data = torch.randn_like(prm) * 0.2 + (1.0 if "norm" in n or n.endswith("1.weight") else 0.0)
        else:
            prm.data = torch.randn_like(prm) * 0.08
    _bf16_params_(model)
    out = {}
    for tag, gh, gw in (("a", 6, 10), ("b", 8, 8)):
        tap = bf16_round(torch.randn(1, 64, gh, gw))
        levels = model(tap)
        out[f"tap_{tag}"] = tap[0].permute(1, 2, 0).contiguous()
        for i, f in enumerate(levels):
            out[f"level{i}_{tag}"] = f[0].permute(1, 2, 0).contiguous()
    save("fpn_small", **_sd_bits(model.state_dict()), **out)


STAGES.update({"vit": gen_vit, "davit": gen_davit, "fpn": gen_fpn})

# --------------------------------------------------------------------------- towers (reference modules)
def _bf16_params_(mod: torch.nn.Module) -> None:
    for prm in mod.parameters():
        prm.data = bf16_round(prm.data)


def _sd_bits(sd) -> dict:
    """state_dict -> {name: uint16 bf16 bit pattern} (values are already bf16-representable)."""
    return {"w::" + k: v.detach().to(torch.bfloat16).view(torch.int16).numpy() for k, v in sd.items()}


VIT_SMALL = dict(depth=4, hidden_size=64, num_heads=2, intermediate_size=88, out_hidden_size=48, patch_size=14,
                 spatial_merge_size=2, temporal_patch_size=2, in_channels=3, window_size=112, fullatt_block_indexes=[1, 3],
                 hidden_act="silu", in_chans=3, tokens_per_second=2)


def gen_vit() -> None:
    ref_shim.load_reference_package()
    from vlm_fo1.model.multimodal_encoder.qwen2_5_vl.configuration_qwen2_5_vl import Qwen2_5_VLVisionConfig
    from vlm_fo1.model.multimodal_encoder.qwen2_5_vl.modeling_qwen2_5_vl import Qwen2_5_VisionTransformerPretrainedModel
    from vlm_fo1.model.multimodal_encoder import qwen2_5_vl_encoder as enc
    torch.manual_seed(0)
    cfg = Qwen2_5_VLVisionConfig(**VIT_SMALL)
    enc.replace_qwen_vit_forward()
    model = Qwen2_5_VisionTransformerPretrainedModel._from_config(cfg, attn_implementation="eager").float().eval()
    for prm in model.parameters():  # the default init leaves norms at 1 / biases at 0: randomise so every term is exercised
        prm.data = torch.randn_like(prm) * (0.02 if prm.dim() > 1 else 0.3) + (1.0 if "norm" in "" else 0.0)
    for n, prm in model.named_parameters():
        if n.endswith("norm1.weight") or n.endswith("norm2.weight") or n.endswith("ln_q.weight"):
            prm.data = prm.data + 1.0
    _bf16_params_(model)
    model.init_vision_features_gather(enc.GATHER)
    out = {}
    int_tables = {}
    for tag, gh, gw in (("a", 6, 10), ("b", 8, 8)):
        px = bf16_round(torch.randn(gh * gw, 3 * 2 * 14 * 14))
        grid = torch.tensor([[1, gh, gw]])
        merged = model(px, grid_thw=grid)
        taps = enc.GATHER.extract_multi_level_features()[0]
        out[f"px_{tag}"] = px
        out[f"grid_{tag}"] = np.array([gh, gw])
        out[f"merged_{tag}"] = merged
        for i, t in enumerate(taps):
            out[f"tap{i}_{tag}"] = t[0].permute(1, 2, 0).contiguous()   # [gh, gw, C]
    # integer bookkeeping at the BASELINE grids (bit-exact targets)
    for gh, gw in ((6, 10), (8, 8), (32, 32), (46, 46), (64, 64), (28, 36), (96, 96), (2, 2), (4, 18)):
        wi, cu = model.get_window_index(torch.tensor([[1, gh, gw]]))
        cu = torch.unique_consecutive(torch.tensor(cu))
        int_tables[f"wi_{gh}x{gw}"] = wi.numpy().astype(np.int32)
        int_tables[f"cu_{gh}x{gw}"] = cu.numpy().astype(np.int32)
    save("vit_small", cfg_json=np.frombuffer(__import__("json").dumps(VIT_SMALL).encode(), dtype=np.uint8),
         **_sd_bits(model.state_dict()), **out, **int_tables)


DAVIT_SMALL = dict(depths=[1, 1, 2, 1], dim_embed=[32, 32, 64, 64], num_heads=[1, 1, 2, 2], num_groups=[1, 1, 2, 2],
                   patch_size=[7, 3, 3, 3], patch_stride=[4, 2, 2, 2], patch_padding=[3, 1, 1, 1],
                   patch_prenorm=[False, True, True, True], drop_path_rate=0.0, window_size=12)


def gen_davit() -> None:
    ref_shim.load_reference_package()
    from vlm_fo1.model.multimodal_encoder.davit.modeling_davit import DaViT
    from types import SimpleNamespace
    torch.manual_seed(1)
    model = DaViT.from_config(SimpleNamespace(**DAVIT_SMALL)).float().eval()
    for n, prm in model.named_parameters():
        if prm.dim() == 1:
            prm.data = torch.randn_like(prm) * 0.2 + (1.0 if n.endswith("norm.weight") else 0.0)
        else:
            prm.data = torch.randn_like(prm) * 0.05
    _bf16_params_(model)
    out = {}
    for tag, H, W in (("a", 72, 104), ("b", 96, 96)):
        img = bf16_round(torch.randn(1, 3, H, W))
        feats = model(img)["image_features"]
        out[f"img_{tag}"] = img[0]
        for i, f in enumerate(feats):
            out[f"stage{i}_{tag}"] = f[0].permute(1, 2, 0).contiguous()
    save("davit_small", cfg_json=np.frombuffer(__import__("json").dumps(DAVIT_SMALL).encode(), dtype=np.uint8),
         **_sd_bits(model.state_dict()), **out)


def gen_fpn() -> None:
    _, fpn = ref_shim.load_hfre_only()
    torch.manual_seed(2)
    model = fpn.SimpleFP(out_channels=32, norm="LN", square_pad=0, dim=64, stride=14).float().eval()
    for n, prm in model.named_parameters():
        if prm.dim() == 1:
            prm.data = torch.randn_like(prm) * 0.2 + (1.0 if "norm" in n or n.endswith("1.weight") else 0.0)
        else:
            prm.data = torch.randn_like(prm) * 0.08
    _bf16_params_(model)
    out = {}
    for tag, gh, gw in (("a", 6, 10), ("b", 8, 8)):
        tap = bf16_round(torch.randn(1, 64, gh, gw))
        levels = model(tap)
        out[f"tap_{tag}"] = tap[0].permute(1, 2, 0).contiguous()
        for i, f in enumerate(levels):
            out[f"level{i}_{tag}"] = f[0].permute(1, 2, 0).contiguous()
    save("fpn_small", **_sd_bits(model.state_dict()), **out)


STAGES.update({"vit": gen_vit, "davit": gen_davit, "fpn": gen_fpn})

LLM_SMALL = dict(num_hidden_layers=3, hidden_size=256, num_attention_heads=2, num_key_value_heads=1, intermediate_size=352,
                 vocab_size=512, rope_theta=1000000.0, rms_norm_eps=1e-6, mrope_section=[16, 24, 24], tie_word_embeddings=False)


def gen_llm() -> None:
    """Pins oracle/llm.py: (1) get_rope_index called unbound on the reference class; (2) a 3-layer stack of the
    reference's own Qwen2_5_VLDecoderLayer + Qwen2_5_VLRotaryEmbedding + Qwen2RMSNorm driven by the thin model loop
    (modeling_qwen2_5_vl.py:1188-1230) -- prefill with a causal mask, then two decode steps with a DynamicCache."""
    ref_shim.load_reference_package()
    from types import SimpleNamespace as NS
    from vlm_fo1.model.multimodal_encoder.qwen2_5_vl import modeling_qwen2_5_vl as M
    import json
    out = {}
    # ---- (1) rope index ----
    g = torch.Generator().manual_seed(5)
    self_ns = NS(config=NS(vision_config=NS(spatial_merge_size=2, tokens_per_second=2), image_token_id=151655, video_token_id=151656,
                           vision_start_token_id=151652))
    cases = []
    for ci, (grids, n_reg) in enumerate((([(8, 8)], 3), ([(6, 10)], 0), ([(4, 4), (8, 6)], 5), ([], 2), ([(64, 64)], 100))):
        ids = torch.randint(0, 151640, (6,), generator=g).tolist()
        for (gh, gw) in grids:
            ids += [151652] + [151655] * (gh * gw // 4) + [151653] + torch.randint(0, 151640, (2,), generator=g).tolist()
        for r in range(n_reg):
            ids += [int(torch.randint(0, 151640, (1,), generator=g)), -300]
        ids += torch.randint(0, 151640, (5,), generator=g).tolist() + [151645]
        grid_thw = torch.tensor([[1, gh, gw] for gh, gw in grids]) if grids else None
        if grid_thw is not None:
            pos, delta = M.Qwen2_5_VLForConditionalGeneration.get_rope_index(self_ns, torch.tensor([ids]), grid_thw, None, None, None)
            pos, delta = pos[:, 0], int(delta[0, 0])
        else:
            pos = torch.arange(len(ids)).view(1, -1).expand(3, -1); delta = 0
        out[f"rope_ids_{ci}"] = np.array(ids, dtype=np.int64)
        out[f"rope_grids_{ci}"] = np.array(grids, dtype=np.int32).reshape(-1, 2)
        out[f"rope_pos_{ci}"] = pos.numpy().astype(np.int64)
        out[f"rope_delta_{ci}"] = np.array(delta)
        cases.append(ci)
    # ---- (2) decoder stack from the reference's own layer modules ----
    torch.manual_seed(3)
    c = LLM_SMALL
    cfg = NS(hidden_size=c["hidden_size"], num_attention_heads=c["num_attention_heads"], num_key_value_heads=c["num_key_value_heads"],
             intermediate_size=c["intermediate_size"], hidden_act="silu", rms_norm_eps=c["rms_norm_eps"], attention_dropout=0.0,
             rope_scaling={"type": "default", "mrope_section": c["mrope_section"], "rope_type": "default"}, rope_theta=c["rope_theta"],
             max_position_embeddings=4096, use_sliding_window=False, sliding_window=None, max_window_layers=99,
             _attn_implementation="eager", head_dim=c["hidden_size"] // c["num_attention_heads"])
    layers = [M.Qwen2_5_VLDecoderLayer(cfg, i).float().eval() for i in range(c["num_hidden_layers"])]
    norm = M.Qwen2RMSNorm(c["hidden_size"], eps=c["rms_norm_eps"]).float()
    rot = M.Qwen2_5_VLRotaryEmbedding(config=cfg)
    embed = torch.nn.Embedding(c["vocab_size"], c["hidden_size"])
    head = torch.nn.Linear(c["hidden_size"], c["vocab_size"], bias=False)
    sd = {}
    for i, l in enumerate(layers):
        for n, prm in l.named_parameters():
            prm.data = bf16_round(torch.randn_like(prm) * (0.05 if prm.dim() > 1 else 0.2) + (1.0 if "layernorm" in n else 0.0))
            sd[f"layers.{i}.{n}"] = prm.data
    norm.weight.data = bf16_round(torch.randn(c["hidden_size"]) * 0.2 + 1.0); sd["norm.weight"] = norm.weight.data
    embed.weight.data = bf16_round(torch.randn_like(embed.weight) * 0.5); sd["embed_tokens.weight"] = embed.weight.data
    head.weight.data = bf16_round(torch.randn_like(head.weight) * 0.05); sd["lm_head.weight"] = head.weight.data
    from transformers.cache_utils import DynamicCache
    ids = out["rope_ids_0"]; pos = torch.from_numpy(out["rope_pos_0"]); delta = int(out["rope_delta_0"])
    L = len(ids)
    x = bf16_round(torch.randn(1, L, c["hidden_size"], generator=g))
    out["llm_embeds"] = x[0]
    cache = DynamicCache()

    def run(x, pos3, past):
        n = x.shape[1]
        cos_sin = rot(x, pos3[:, None, :])
        mask = torch.full((n, past + n), float("-inf")).triu(past + 1)[None, None]
        h = x
        for l in layers:
            h = l(h, attention_mask=mask, position_ids=pos3[:, None, :], past_key_value=cache, use_cache=True,
                  cache_position=torch.arange(past, past + n), position_embeddings=cos_sin)[0]
        return h

    h = run(x, pos, 0)
    logits = head(norm(h))[0]
    out["llm_prompt_logits"] = logits
    toks = []
    lg = logits[-1]
    step_logits = []
    for s in range(3):
        step_logits.append(lg)
        tok = int(lg.argmax()); toks.append(tok)
        p = L + s + delta
        h = run(embed(torch.tensor([[tok]])), torch.full((3, 1), p, dtype=torch.long), L + s)
        lg = head(norm(h))[0, -1]
    out["llm_step_logits"] = torch.stack(step_logits)
    out["llm_tokens"] = np.array(toks)
    save("llm_small", cfg_json=np.frombuffer(json.dumps(LLM_SMALL).encode(), dtype=np.uint8), n_rope_cases=np.array(len(cases)),
         **_sd_bits(sd), **out)


STAGES.update({"llm": gen_llm})


def gen_mm_utils() -> None:
    """Pins the boundary mirror vlm_fo1/mm_utils.py: the REFERENCE's own prepare_inputs / extract_predictions_* /
    adjust_bbox run on a fabricated byte-level tokenizer + this repo's processors (loaded by file path)."""
    import importlib.util, json, tempfile
    from types import SimpleNamespace as NS
    from PIL import Image
    if ref_shim.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shim.REFERENCE_ROOT)
    for k in [k for k in sys.modules if k == "vlm_fo1" or k.startswith("vlm_fo1.")]:
        del sys.modules[k]
    import vlm_fo1.mm_utils as RMU            # the reference's
    from vlm_fo1.task_templates import OD_template, OD_Counting_template
    assert RMU.__file__.startswith(ref_shim.REFERENCE_ROOT), RMU.__file__

    def load_by_path(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REPO, rel))
        m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m
    sys.path.insert(0, REPO)   # for `vlm-fo1_b200` only; `vlm_fo1` is already bound to the reference in sys.modules
    fo1 = __import__("importlib").import_module("vlm-fo1_b200.fabricate")
    PR = load_by_path("fo1_processors", "vlm_fo1/processors.py")
    d = os.path.join(tempfile.mkdtemp(), "VLM-FO1_Qwen2.5-VL-3B-v01"); os.makedirs(d)
    fo1.write_tokenizer(d)
    from transformers import AutoTokenizer
    tok = AutoTokenizer.from_pretrained(d, use_fast=False)
    procs = (PR.PrimaryImageProcessor(), PR.AuxImageProcessor(768, "dynamic"))
    model = NS(config=NS(mm_use_region_index_token=True))
    rng = np.random.default_rng(7)
    out = {}
    cases = []
    img_a = os.path.join(d, "a.png"); Image.fromarray(rng.integers(0, 256, (399, 500, 3), dtype=np.uint8)).save(img_a)
    img_b = os.path.join(d, "b.png"); Image.fromarray(rng.integers(0, 256, (2300, 1200, 3), dtype=np.uint8)).save(img_b)   # long edge > 2048
    boxes7 = [[161.0, 11.0, 292.0, 127.0], [268.0, 61.0, 428.0, 226.0], [12.0, 100.0, 140.0, 227.0], [205.0, 188.0, 332.0, 320.0],
              [326.0, 202.0, 478.0, 357.0], [136.0, 106.0, 269.0, 233.0], [25.0, 206.0, 200.0, 383.0]]
    boxes_out = [[-5.0, -3.0, 600.0, 500.0], [10.5, 20.25, 30.75, 41.0]]
    many = [[float(i), float(i), float(i + 20), float(i + 30)] for i in range(130)]
    specs = [("demo", img_a, boxes7, OD_template.format("orange"), None),
             ("clamp", img_a, boxes_out, OD_Counting_template.format("cats"), None),
             ("cap100", img_a, many, OD_template.format("things"), None),
             ("big", img_b, boxes7, OD_template.format("person"), None),
             # ("noboxes", ...): the reference itself crashes on a message without bbox_list (torch.tensor(None), mm_utils.py:396)
             ("system", img_a, boxes7[:2], OD_template.format("x"), "You are terse.")]
    for tag, img, boxes, text, system in specs:
        msgs = []
        if system:
            msgs.append({"role": "system", "content": system})
        m = {"role": "user", "content": [{"type": "image_url", "image_url": {"url": img}}, {"type": "text", "text": text}]}
        if boxes is not None:
            m["bbox_list"] = [list(b) for b in boxes]
        msgs.append(m)
        kw = RMU.prepare_inputs(d, model, procs, tok, msgs, device="cpu", max_tokens=64)
        out[f"{tag}_inputs"] = kw["inputs"].numpy()
        out[f"{tag}_grid"] = kw["image_grid_thws"][0].numpy()
        out[f"{tag}_aux_shape"] = np.array(kw["images_aux"][0].shape)
        out[f"{tag}_px_sum"] = np.array(float(kw["images"][0].double().sum()))
        out[f"{tag}_aux_sum"] = np.array(float(kw["images_aux"][0].double().sum()))
        out[f"{tag}_boxes"] = kw["bbox_list"][0].numpy() if kw["bbox_list"] else np.zeros((0, 4), np.float32)
        out[f"{tag}_stop"] = np.array([int(k.item()) for k in kw["stopping_criteria"][0].keyword_ids if k.numel() == 1])
        cases.append(dict(tag=tag, img=os.path.basename(img), boxes=boxes, text=text, system=system))
    pred = "<ground>orange</ground><objects><region1><region4><region1></objects> and <ground> cat </ground><objects><region0></objects><ground>orange</ground><objects><region6></objects>"
    idx = RMU.extract_predictions_to_indexes(pred)
    bxs = RMU.extract_predictions_to_bboxes(pred, boxes7)
    out["parse_json"] = np.frombuffer(json.dumps({"pred": pred, "indexes": {k: sorted(v) for k, v in idx.items()},
                                                  "bboxes": {k: sorted(v) for k, v in bxs.items()}}).encode(), dtype=np.uint8)
    out["cases_json"] = np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8)
    out["img_a"] = np.asarray(Image.open(img_a)); out["img_b_seed"] = np.array(7)
    save("mm_utils", **out)


STAGES.update({"mm_utils": gen_mm_utils})


def gen_processors() -> None:
    """Pins vlm_fo1/processors.py (the host-side pre-processing, SURVEY 8f rank 1):
    * aux tower: the REFERENCE's own CLIPImageProcessor (davit/image_processing_clip.py:222-367 with the img_cfg of
      davit/configs.py:139-152), loaded by file path, in both resize modes ('dynamic' = the released checkpoint, 'squash');
    * primary tower: the reference calls transformers' Qwen2VLImageProcessor (qwen2_5_vl_encoder.py:210-225, transformers
      4.50.1).  That release is not installed here; the INSTALLED transformers (version recorded in the fixture) provides
      the same class, whose resize may differ from the pinned release by <= 2 uint8 steps on a small fraction of pixels, so
      images that need no resize pin the patch order / normalisation exactly and resized ones pin the grid + values to 2 LSB.
    Outputs are stored as a strided sample + a float64 sum; the input images are re-drawn by the test (seed 11)."""
    import importlib.util
    import transformers
    from PIL import Image
    spec = importlib.util.spec_from_file_location("ref_clip_ip", os.path.join(ref_shim.REFERENCE_ROOT, "vlm_fo1/model/multimodal_encoder/davit/image_processing_clip.py"))
    RC = importlib.util.module_from_spec(spec); spec.loader.exec_module(RC)
    from transformers.models.qwen2_vl.image_processing_qwen2_vl import Qwen2VLImageProcessor
    base = {"do_resize": True, "size": {"height": 768, "width": 768}, "resample": 3, "do_center_crop": False, "do_rescale": True,
            "do_normalize": True, "image_mean": [0.485, 0.456, 0.406], "image_std": [0.229, 0.224, 0.225], "do_convert_rgb": True}
    rng = np.random.default_rng(11)
    out = {"transformers_version": np.array(transformers.__version__)}
    sizes = [(56, 84), (399, 500), (64, 33), (20, 20), (301, 1203)]
    out["sizes"] = np.array(sizes)
    prim = Qwen2VLImageProcessor(min_pixels=56 * 56, max_pixels=2048 * 2048)
    for i, hw in enumerate(sizes):
        arr = rng.integers(0, 256, hw + (3,), dtype=np.uint8)   # the test regenerates the images from the same seed / order
        img = Image.fromarray(arr)
        for mode in ("dynamic", "squash"):
            cfg = dict(base); cfg["resize_mode"] = mode
            if mode == "dynamic":
                cfg["do_resize"] = False
            r = RC.CLIPImageProcessor(**cfg).preprocess(img, return_tensors="pt")["pixel_values"][0].numpy()
            out[f"aux_{mode}{i}_shape"] = np.array(r.shape)
            out[f"aux_{mode}{i}_sample"] = r[:, ::7, ::5].copy()
            out[f"aux_{mode}{i}_sum"] = np.array(r.astype(np.float64).sum())
        q = prim.preprocess(img, return_tensors="pt")
        px = q["pixel_values"].numpy()
        out[f"prim{i}_grid"] = q["image_grid_thw"].numpy()
        out[f"prim{i}_shape"] = np.array(px.shape)
        out[f"prim{i}_sample"] = px[::3, ::11].copy()
        out[f"prim{i}_sum"] = np.array(px.astype(np.float64).sum())
    save("processors", **out)


STAGES.update({"processors": gen_processors})


def gen_prompt_data() -> None:
    """Pins the pure-data mirrors vlm_fo1/constants.py and vlm_fo1/task_templates.py: every public str / int of the
    REFERENCE's two modules, dumped to tests/golden/prompt_data.json."""
    import importlib.util, json
    out = {}
    for mod in ("constants", "task_templates"):
        spec = importlib.util.spec_from_file_location(f"ref_{mod}", os.path.join(ref_shim.REFERENCE_ROOT, "vlm_fo1", mod + ".py"))
        m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
        out[mod] = {k: v for k, v in vars(m).items() if not k.startswith("_") and isinstance(v, (str, int))}
    path = os.path.join(GOLD, "prompt_data.json")
    json.dump(out, open(path, "w"), indent=1, sort_keys=True)
    print(f"wrote {path}")


STAGES.update({"prompt_data": gen_prompt_data})


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    wanted = sys.argv[1:] or list(STAGES)
    for s in wanted:
        STAGES[s]()



