"""The FO1 hot path assembled from the REFERENCE'S OWN modules, on the CPU -- TEST / BASELINE INFRASTRUCTURE ONLY.

``bench.py --impl reference`` and the ``cpu_baseline`` leg time this (``kind: "reference"``).  The reference is a Python
tree without packaging metadata, so ``stage_copy()`` (called by ``__graft_entry__.build()``) copies its ``vlm_fo1`` package
(Python files only) into the git-ignored ``oracle/_ref/`` where a checkout of the reference is at hand (``FO1_REFERENCE_ROOT``).
The modules are imported from there with the three shims of ``oracle/ref_shim.py`` (SURVEY.md section 8c):

  ViT + taps      Qwen2_5_VisionTransformerPretrainedModel + replace_qwen_vit_forward + GATHER   (qwen2_5_vl_encoder.py:86-158, 37-80)
  aux tower       DaViT.from_config(davit-large)                                                  (modeling_davit.py:478-506)
  HFRE + FPN      HFREModule(use_simpleFPN_for_vt=True) incl. its SimpleFP                       (hybrid_finegrained_region_encoder.py:275-468)
  projector       build_vision_projector_aux (mlp2x_gelu)                                         (multimodal_projector/builder.py:78-115)
  decoder         36 x Qwen2_5_VLDecoderLayer + Qwen2_5_VLRotaryEmbedding + Qwen2RMSNorm + DynamicCache (modeling_qwen2_5_vl.py:1014-1095)

What cannot be constructed under the installed transformers (OmChatQwen25VLForCausalLM itself, SURVEY.md section 8c) is the
thin glue only: the splice, the model loop over the layers and the greedy loop, restated in oracle/llm.py / here from
omchat_qwen2_5_vl.py:291-463 and modeling_qwen2_5_vl.py:1188-1230, 1848-1860.  fp32, every host thread, attention
``sdpa`` (the reference hard-codes flash_attention_2, which is CUDA-only).  Weights are random: this arm is a timing
baseline; numerical pinning of the oracle against these same modules lives in oracle/gen_golden.py."""
from __future__ import annotations

import os
import time
from types import SimpleNamespace as NS
from typing import Dict, Optional, Sequence

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF_COPY = os.path.join(HERE, "_ref")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_COPY, "vlm_fo1", "model"))


def stage_copy() -> bool:
    """Copy the Python files of the reference's ``vlm_fo1`` package, and its demo caller ``inference.py`` (which
    tests/test_gpu_boundary.py executes unmodified against this repo's ``vlm_fo1`` mirror), from the reference checkout
    (``oracle/ref_shim.py``: REFERENCE_ROOT) into ``oracle/_ref/``.  Nothing from this copy is product code or tracked by git.
    Returns whether a copy is in place afterwards."""
    import shutil
    try:
        from . import ref_shim
    except ImportError:
        import ref_shim  # type: ignore
    src = os.path.join(ref_shim.REFERENCE_ROOT, "vlm_fo1")
    dst = os.path.join(REF_COPY, "vlm_fo1")
    if not os.path.isdir(src) or os.path.abspath(src) == os.path.abspath(dst):
        return available()
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    shutil.copytree(src, dst, ignore=lambda d, names: [n for n in names if not (n.endswith(".py") or os.path.isdir(os.path.join(d, n)))])
    shutil.copy(os.path.join(os.path.dirname(src), "inference.py"), os.path.join(REF_COPY, "inference.py"))
    return True


def _fill_(mod: torch.nn.Module) -> None:
    """cheap deterministic-enough values (a timing arm): no denormals, norms at 1"""
    g = torch.Generator().manual_seed(0)
    for n, p in mod.named_parameters():
        if p.dim() > 1:
            p.data.uniform_(-0.035, 0.035, generator=g)      # std 0.02
        elif "norm" in n and n.endswith("weight"):
            p.data.fill_(1.0)
        else:
            p.data.zero_()


def usable_cores(cap: int = 32) -> int:
    """Host threads worth using: the affinity mask and the cgroup CPU quota (a container that sees 128 logical CPUs but owns a fraction
    of them crawls when 128 OpenMP threads spin on it), capped where these small fp32 GEMMs stop scaling."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except AttributeError:
        pass
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(per))))
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read()); per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // per))
        except Exception:
            pass
    return max(1, min(n, cap))


class ReferencePath:
    """``sample``: None runs every block; ``dict(vit_blocks=8, llm_layers=4, davit_stage3=3)`` builds and runs a DEPTH SAMPLE -- one period
    of the ViT's block pattern (7 windowed + 1 full-attention block), a few decoder layers, DaViT's third stage at reduced depth -- and
    ``run`` scales the measured block times to the full depth (blocks of a stack cost the same; embeddings, mergers, FPN, HFRE, projector,
    LM head are always run in full).  The bench's bounded CPU sample (a full-depth image takes minutes on the host cores)."""

    def __init__(self, vit_cfg: dict, davit_name: str, llm_cfg: dict, region_dim: int = 5888, davit_depths=None, sample: Optional[dict] = None):
        import sys
        try:
            from . import ref_shim
        except ImportError:
            import ref_shim  # type: ignore
        # the repo's own ``vlm_fo1`` (the boundary mirror) must not shadow the reference's package
        for k in [k for k in sys.modules if k == "vlm_fo1" or k.startswith("vlm_fo1.")]:
            del sys.modules[k]
        ref_shim.REFERENCE_ROOT = REF_COPY
        sys.path = [REF_COPY] + [p for p in sys.path if os.path.abspath(p or ".") not in (REPO, REF_COPY)]
        ref_shim.load_reference_package()
        from vlm_fo1.model.multimodal_encoder.qwen2_5_vl.configuration_qwen2_5_vl import Qwen2_5_VLVisionConfig
        from vlm_fo1.model.multimodal_encoder.qwen2_5_vl import modeling_qwen2_5_vl as M
        from vlm_fo1.model.multimodal_encoder import qwen2_5_vl_encoder as enc
        from vlm_fo1.model.multimodal_encoder.davit.modeling_davit import DaViT
        from vlm_fo1.model.multimodal_encoder.davit.configs import model_configs
        from vlm_fo1.model.multimodal_visual_prompt_encoder.hybrid_finegrained_region_encoder import HFREModule
        from vlm_fo1.model.multimodal_projector.builder import build_vision_projector_aux
        self.M, self.enc = M, enc
        t0 = time.perf_counter()
        self.scale = dict(vit=1.0, llm=1.0, davit3=1.0)
        vit_cfg, llm_cfg = dict(vit_cfg), dict(llm_cfg)
        full_davit_depths = list(davit_depths) if davit_depths is not None else None
        if sample:
            fa = list(vit_cfg["fullatt_block_indexes"])
            period = fa[0] + 1 if fa else 0
            vb = int(sample.get("vit_blocks", 0))
            if vb and period and vb % period == 0 and vb < vit_cfg["depth"] and fa == [period * (i + 1) - 1 for i in range(len(fa))] \
                    and vit_cfg["depth"] % period == 0:
                self.scale["vit"] = vit_cfg["depth"] / vb
                vit_cfg["depth"] = vb
                vit_cfg["fullatt_block_indexes"] = [period * (i + 1) - 1 for i in range(vb // period)]
            ll = int(sample.get("llm_layers", 0))
            if ll and ll < llm_cfg["num_hidden_layers"]:
                self.scale["llm"] = llm_cfg["num_hidden_layers"] / ll
                llm_cfg["num_hidden_layers"] = ll
            d3 = int(sample.get("davit_stage3", 0))
            if d3 and full_davit_depths is not None and d3 < full_davit_depths[2]:
                self.scale["davit3"] = full_davit_depths[2] / d3
                davit_depths = list(full_davit_depths); davit_depths[2] = d3
        with torch.no_grad():
            vc = Qwen2_5_VLVisionConfig(depth=vit_cfg["depth"], hidden_size=vit_cfg["hidden_size"], num_heads=vit_cfg["num_heads"],
                                        intermediate_size=vit_cfg["intermediate_size"], out_hidden_size=vit_cfg["out_hidden_size"],
                                        patch_size=vit_cfg["patch_size"], spatial_merge_size=vit_cfg["spatial_merge_size"],
                                        temporal_patch_size=vit_cfg["temporal_patch_size"], window_size=vit_cfg["window_size"],
                                        fullatt_block_indexes=list(vit_cfg["fullatt_block_indexes"]), hidden_act="silu", in_chans=3)
            enc.replace_qwen_vit_forward()
            self.vit = M.Qwen2_5_VisionTransformerPretrainedModel._from_config(vc, attn_implementation="sdpa").float().eval()
            self.vit.init_vision_features_gather(enc.GATHER)
            dc = dict(model_configs[davit_name])
            if davit_depths is not None:
                dc["depths"] = list(davit_depths)
            dc["drop_path_rate"] = 0.0
            dc["enable_checkpoint"] = False
            self.davit = DaViT.from_config(NS(**dc)).float().eval()
            self.hfre = HFREModule(roi_output_size=7, region_feature_dim=region_dim, apply_position_embedding=True,
                                   pos_embedding_strategy="bbox_based", use_vt_region_feature_only=False,
                                   use_vision_tower_region_feature=True, region_feature_combination="concat",
                                   apply_region_layer_norm=False, vision_tower_region_feature_dim=2048,
                                   vision_tower_spatial_scale=1 / vit_cfg["patch_size"], use_simpleFPN_for_vt=True,
                                   aux_vision_tower_spatial_scale=0.25, aux_vision_tower_region_feature_dims=[256, 512, 1024, 2048]).float().eval()
            self.proj = build_vision_projector_aux(NS(mm_projector_aux_type="mlp2x_gelu", mm_region_hidden_size=region_dim,
                                                      hidden_size=llm_cfg["hidden_size"])).float().eval()
            c = llm_cfg
            self.lc = NS(hidden_size=c["hidden_size"], num_attention_heads=c["num_attention_heads"], num_key_value_heads=c["num_key_value_heads"],
                         intermediate_size=c["intermediate_size"], hidden_act="silu", rms_norm_eps=c["rms_norm_eps"], attention_dropout=0.0,
                         rope_scaling={"type": "default", "mrope_section": list(c["mrope_section"]), "rope_type": "default"},
                         rope_theta=c["rope_theta"], max_position_embeddings=32768, use_sliding_window=False, sliding_window=None,
                         max_window_layers=99, _attn_implementation="sdpa", head_dim=c["hidden_size"] // c["num_attention_heads"])
            try:
                self.layers = [M.Qwen2_5_VLDecoderLayer(self.lc, i).float().eval() for i in range(c["num_hidden_layers"])]
            except Exception:   # attention class table without an sdpa entry under this transformers: the eager class
                self.lc._attn_implementation = "eager"
                self.layers = [M.Qwen2_5_VLDecoderLayer(self.lc, i).float().eval() for i in range(c["num_hidden_layers"])]
            self.norm = M.Qwen2RMSNorm(c["hidden_size"], eps=c["rms_norm_eps"]).float()
            self.rot = M.Qwen2_5_VLRotaryEmbedding(config=self.lc)
            self.embed = torch.nn.Embedding(c["vocab_size"], c["hidden_size"])
            for m in (self.vit, self.davit, self.hfre, self.proj, self.embed, *self.layers):
                _fill_(m)
        self.llm_cfg, self.vit_cfg, self.region_dim = llm_cfg, vit_cfg, region_dim
        self.build_seconds = time.perf_counter() - t0
        self.attn = self.lc._attn_implementation

    # ---- the model loop of Qwen2_5_VLModel.forward (modeling_qwen2_5_vl.py:1188-1230) over the reference's layers ----
    def _decoder(self, x: torch.Tensor, pos3: torch.Tensor, past: int, cache) -> torch.Tensor:
        n = x.shape[1]
        cos_sin = self.rot(x, pos3[:, None, :])
        mask = torch.full((n, past + n), float("-inf")).triu(past + 1)[None, None]
        h = x
        for l in self.layers:
            h = l(h, attention_mask=mask, position_ids=pos3[:, None, :], past_key_value=cache, use_cache=True,
                  cache_position=torch.arange(past, past + n), position_embeddings=cos_sin)[0]
        return h

    @torch.no_grad()
    def run(self, *, input_ids: Sequence[int], pixel_values: torch.Tensor, grid_hw, image_aux: torch.Tensor, boxes: torch.Tensor,
            max_new_tokens: int, image_token_id: int = 151655, vision_start_token_id: int = 151652) -> Dict:
        try:
            from . import llm as OL
        except ImportError:
            import llm as OL  # type: ignore
        from transformers.cache_utils import DynamicCache
        t: Dict[str, float] = {}
        gh, gw = grid_hw
        t0 = time.perf_counter()
        merged = self.vit(pixel_values.float(), grid_thw=torch.tensor([[1, gh, gw]]))
        taps = self.enc.GATHER.extract_multi_level_features()[0]               # n_fullatt x [1, hidden, gh, gw]
        t["vit_s"] = (time.perf_counter() - t0) * self.scale["vit"]; t0 = time.perf_counter()
        st3 = {"t": 0.0}
        stage3 = self.davit.blocks[2]
        h1 = stage3.register_forward_pre_hook(lambda m, a: st3.__setitem__("t0", time.perf_counter()))
        h2 = stage3.register_forward_hook(lambda m, a, o: st3.__setitem__("t", time.perf_counter() - st3["t0"]))
        aux = self.davit(image_aux.float().unsqueeze(0))["image_features"]
        h1.remove(); h2.remove()
        t["davit_s"] = (time.perf_counter() - t0) + st3["t"] * (self.scale["davit3"] - 1.0); t0 = time.perf_counter()
        Ha, Wa = image_aux.shape[-2:]
        b = boxes.float() if boxes.numel() else torch.tensor([[0.0, 10.0, 0.0, 10.0]])
        p = self.vit_cfg["patch_size"]
        vt_boxes = b * torch.tensor([gw * p / Wa, gh * p / Ha, gw * p / Wa, gh * p / Ha])     # omchat_qwen2_5_vl.py:94-99
        region = self.hfre(aux_multi_level_features=aux, vt_multi_level_features=taps[-1], aux_boxes=[b], vt_boxes=[vt_boxes]).squeeze(0)
        t["fpn_hfre_s"] = time.perf_counter() - t0; t0 = time.perf_counter()
        region_tokens = self.proj(region)
        t["proj_s"] = time.perf_counter() - t0; t0 = time.perf_counter()
        new_ids, kind, index = OL.splice_plan(input_ids, [grid_hw], region_tokens.shape[0], image_token_id, self.vit_cfg["spatial_merge_size"])
        pos, delta = OL.rope_index(new_ids, [grid_hw], image_token_id, vision_start_token_id, self.vit_cfg["spatial_merge_size"])
        emb = self.embed.weight
        rows = [emb[ix] if k == 0 else (merged[ix] if k == 1 else region_tokens[ix]) for k, ix in zip(kind, index)]
        x = torch.stack(rows)[None]
        t["splice_s"] = time.perf_counter() - t0; t0 = time.perf_counter()
        cache = DynamicCache()
        L = x.shape[1]
        h = self._decoder(x, pos, 0, cache)
        t_layers = time.perf_counter() - t0; t0 = time.perf_counter()
        lg = (self.norm(h[:, -1:]) @ emb.t())[0, -1]                           # tied head, last position only
        t["llm_prefill_s"] = t_layers * self.scale["llm"] + (time.perf_counter() - t0); t0 = time.perf_counter()
        toks = []
        t_dec_layers = t_dec_head = 0.0
        for s in range(max_new_tokens):
            tok = int(lg.argmax()); toks.append(tok)
            if s == max_new_tokens - 1:
                break
            t0 = time.perf_counter()
            h = self._decoder(emb[tok][None, None, :], torch.full((3, 1), L + s + delta, dtype=torch.long), L + s, cache)
            t_dec_layers += time.perf_counter() - t0; t0 = time.perf_counter()
            lg = (self.norm(h) @ emb.t())[0, -1]
            t_dec_head += time.perf_counter() - t0
        t["llm_decode_s"] = t_dec_layers * self.scale["llm"] + t_dec_head
        t["total_s"] = sum(v for k, v in t.items() if k.endswith("_s"))
        return dict(tokens=toks, timings=t, prompt_len=L, scale=dict(self.scale))
