"""-m gpu: the reference's caller sequence (inference.py:37-59) against this repo's ``vlm_fo1`` mirror and a fabricated
random-init checkpoint directory: load_pretrained_model -> prepare_inputs -> model.generate -> tokenizer.decode ->
extract_predictions_to_bboxes -> draw_bboxes_and_save, with the script's own defaults (device="cuda", max_tokens=4096,
torch.inference_mode).  The checkpoint is reduced-depth (real widths) so fabrication stays small; a full-depth directory
is produced the same way by ``vlm-fo1_b200/fabricate.py``."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu


def test_inference_py_call_sequence(tmp_path):
    from importlib import import_module
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); FB = import_module("vlm-fo1_b200.fabricate")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=2)
    model_path = FB.fabricate_checkpoint(str(tmp_path / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    img_path = str(tmp_path / "demo_image.jpg")
    Image.fromarray(np.random.default_rng(0).integers(0, 256, (399, 500, 3), dtype=np.uint8)).save(img_path)

    # ---- from here on: the statements of inference.py, unchanged apart from the two paths ----
    from detect_tools.upn import UPNWrapper  # noqa: F401
    from vlm_fo1.model.builder import load_pretrained_model
    from vlm_fo1.mm_utils import prepare_inputs, draw_bboxes_and_save, extract_predictions_to_bboxes
    from vlm_fo1.task_templates import OD_template
    bbox_list = [[161.0, 11.0, 292.0, 127.0], [268.0, 61.0, 428.0, 226.0], [12.0, 100.0, 140.0, 227.0], [205.0, 188.0, 332.0, 320.0],
                 [326.0, 202.0, 478.0, 357.0], [136.0, 106.0, 269.0, 233.0], [25.0, 206.0, 200.0, 383.0]]
    messages = [{"role": "user", "content": [{"type": "image_url", "image_url": {"url": img_path}},
                                             {"type": "text", "text": OD_template.format("orange")}], "bbox_list": bbox_list}]
    tokenizer, model, image_processors = load_pretrained_model(model_path)
    generation_kwargs = prepare_inputs(model_path, model, image_processors, tokenizer, messages,
                                       max_tokens=4096, top_p=0.05, temperature=0.0, do_sample=False)
    generation_kwargs["max_new_tokens"] = 24          # (the test bounds the length; a random-init model never emits <|im_end|>)
    with torch.inference_mode():
        output_ids = model.generate(**generation_kwargs)
        outputs = tokenizer.decode(output_ids[0, generation_kwargs["inputs"].shape[1]:]).strip()
    bboxes = extract_predictions_to_bboxes(outputs, bbox_list)
    out_path = str(tmp_path / "vlm_fo1_result.jpg")
    draw_bboxes_and_save(image=Image.open(img_path).convert("RGB"), fo1_bboxes=bboxes, output_path=out_path)
    # ---- contract checks ----
    P = generation_kwargs["inputs"].shape[1]
    assert output_ids.dim() == 2 and output_ids.shape[0] == 1 and P < output_ids.shape[1] <= P + 24
    assert torch.equal(output_ids[0, :P].cpu(), generation_kwargs["inputs"][0].cpu())      # callers slice at inputs.shape[1]
    assert isinstance(outputs, str) and isinstance(bboxes, dict) and os.path.exists(out_path)
    # determinism + stop handling through the same surface: stop on the 3rd generated id
    new = output_ids[0, P:].tolist()
    model.default_stop_ids = [new[2]]
    again = model.generate(**generation_kwargs)
    assert again[0, P:].tolist() == new[: new.index(new[2]) + 1]


def test_reference_inference_py_runs_unmodified(tmp_path, monkeypatch):
    """The reference's own ``inference.py`` FILE (staged byte-for-byte into oracle/_ref/ by __graft_entry__.build()), executed
    with runpy from a working directory laid out like the reference's (./resources/<checkpoint>, ./demo/demo_image.jpg) with
    this repo first on sys.path, so that its imports resolve to the repo's ``vlm_fo1`` / ``detect_tools`` mirror.  No statement
    of the script is re-typed here; max_tokens stays at the script's 4096 (a random-init model never emits <|im_end|>)."""
    import runpy
    import sys
    REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = os.path.join(REPO, "oracle", "_ref", "inference.py")
    if not os.path.exists(script):
        pytest.skip("oracle/_ref/inference.py not staged (build() copies it where a reference checkout exists)")
    from importlib import import_module
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); FB = import_module("vlm-fo1_b200.fabricate")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    FB.fabricate_checkpoint(str(tmp_path / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    os.makedirs(tmp_path / "demo")
    Image.fromarray(np.random.default_rng(0).integers(0, 256, (399, 500, 3), dtype=np.uint8)).save(str(tmp_path / "demo" / "demo_image.jpg"))
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(sys, "path", [REPO] + [p for p in sys.path if p != REPO])
    for k in [k for k in sys.modules if k == "vlm_fo1" or k.startswith("vlm_fo1.")]:
        if REPO not in (getattr(sys.modules[k], "__file__", "") or ""):
            del sys.modules[k]                     # a reference copy imported by another test must not shadow the mirror
    g = runpy.run_path(script, run_name="__main__")
    P = g["generation_kwargs"]["inputs"].shape[1]
    assert g["output_ids"].shape[0] == 1 and P < g["output_ids"].shape[1] <= P + 4096
    assert isinstance(g["outputs"], str) and isinstance(g["bboxes"], dict)
    assert os.path.exists(tmp_path / "demo" / "vlm_fo1_result.jpg")
