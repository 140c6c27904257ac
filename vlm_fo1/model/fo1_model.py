"""The object ``load_pretrained_model`` returns in place of the reference's ``OmChatQwen25VLForCausalLM``
(vlm_fo1/model/language_model/omchat_qwen2_5_vl.py:28-41): same ``.config`` attributes the callers read, same
``.generate(**kwargs)`` contract (mm_utils.py:640-654 builds the kwargs; returns LongTensor [1, P + T] whose first P
columns are ``inputs``), everything underneath delegated to the H100 engine."""
from __future__ import annotations

from importlib import import_module
from types import SimpleNamespace
from typing import List

import torch


class Fo1ForCausalLM:
    def __init__(self, engine, config: SimpleNamespace, vt_mode: str, stop_ids: List[int], roi_size: int = 7, apply_pos_embed: bool = True):
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

    # nn.Module-ish no-ops the callers invoke
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def get_model(self):
        return self

    def _sample(self, inputs=None, images=None, images_aux=None, image_grid_thws=None, bbox_list=None, do_sample=False, temperature=0.0,
                stopping_criteria=None, **kwargs):
        """One ``prepare_inputs`` dict -> (SampleInputs, stop ids): the argument checks of the reference's call contract."""
        if do_sample or (temperature or 0.0) != 0.0:
            raise NotImplementedError("the fo1-b200 engine decodes greedily (the reference's callers all pass temperature=0.0)")
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
        return sample, stop

    @torch.no_grad()
    def generate(self, inputs=None, images=None, images_aux=None, image_grid_thws=None, bbox_list=None, do_sample=False, temperature=0.0,
                 max_new_tokens=512, streamer=None, top_p=1.0, use_cache=True, stopping_criteria=None, pad_token_id=None, **kwargs):
        sample, stop = self._sample(inputs, images, images_aux, image_grid_thws, bbox_list, do_sample, temperature, stopping_criteria)
        pad = pad_token_id if pad_token_id is not None else (stop[0] if stop else 0)
        out = self.pipeline.generate([sample], int(max_new_tokens), sorted(set(stop)), pad_id=int(pad), early_exit_interval=8)
        n = int(out["lens"][0].item())
        new = out["tokens"][0, :n].to(torch.long)
        full = torch.cat([inputs[0].to(new.device), new]).unsqueeze(0)
        if streamer is not None:
            # the whole completion is handed over at once (the decode loop is device-resident: no per-token host sync);
            # a streamer error is the caller's to see, as in HF's generate
            streamer.put(inputs.cpu())
            streamer.put(new.cpu())
            streamer.end()
        return full

    @torch.no_grad()
    def generate_batch(self, batch, max_new_tokens=None):
        """``batch``: a list of the dicts ``prepare_inputs`` returns (one sample each, mm_utils.py:640-654).  All samples run as ONE
        packed batch through the engine (what the reference's evaluation loops do one image at a time, eval_coco.py:36-88).
        -> list of LongTensor [1, P_b + T_b], each exactly what ``generate(**batch[b])`` returns."""
        if not batch:
            return []
        samples, stops = zip(*(self._sample(**{k: v for k, v in kw.items() if k in (
            "inputs", "images", "images_aux", "image_grid_thws", "bbox_list", "do_sample", "temperature", "stopping_criteria")}) for kw in batch))
        stop = sorted(set(x for s in stops for x in s))
        T = int(max_new_tokens if max_new_tokens is not None else max(int(kw.get("max_new_tokens", 512)) for kw in batch))
        pads = [kw.get("pad_token_id") for kw in batch]
        pad = pads[0] if pads[0] is not None else (stop[0] if stop else 0)
        out = self.pipeline.generate(list(samples), T, stop, pad_id=int(pad), early_exit_interval=8)
        lens = out["lens"].cpu().tolist()
        res = []
        for b, kw in enumerate(batch):
            new = out["tokens"][b, :lens[b]].to(torch.long)
            res.append(torch.cat([kw["inputs"][0].to(new.device), new]).unsqueeze(0))
        return res
