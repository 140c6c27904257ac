"""-m gpu: the batched evaluation drivers (evaluation/eval_coco.py, eval_countbench.py -- the reference's scripts with their
per-image loop batched) on a sample of the reference's own proposal files (tests/golden/eval_proposals_sample.json.gz: real box
counts, queries, image sizes; noise pixels stand in for the absent datasets) against a fabricated reduced-depth checkpoint.
Checks the file contract of the reference's scripts and that a batch returns exactly the ids the one-by-one calls return."""
import gzip
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    from importlib import import_module
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); FB = import_module("vlm-fo1_b200.fabricate")
    root = tmp_path_factory.mktemp("eval")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=2, fullatt_block_indexes=[0, 1])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=1)
    model_path = FB.fabricate_checkpoint(str(root / "resources" / "VLM-FO1_Qwen2.5-VL-3B-v01"), cfg, seed=0, device="cuda")
    fx = json.load(gzip.open(os.path.join(REPO, "tests", "golden", "eval_proposals_sample.json.gz"), "rt"))
    with open(root / "coco.jsonl", "w") as f:
        for d in fx["coco"]:
            f.write(json.dumps(d) + "\n")
    json.dump(fx["instances"], open(root / "instances.json", "w"))
    json.dump(fx["countbench"], open(root / "countbench.json", "w"))
    return root, model_path, fx


def test_eval_coco_batched_writes_the_reference_result_file(setup):
    root, model_path, fx = setup
    from evaluation.eval_coco import eval_coco
    ips = eval_coco(model_path, str(root / "coco.jsonl"), str(root / "instances.json"), str(root / "no_such_folder"), out_dir=str(root / "out"),
                    device="cuda:0", batch_size=4, limit=8, synthetic_images=str(root / "synth"), max_tokens=12)
    out = root / "out" / "VLM-FO1_Qwen2.5-VL-3B-v01" / "coco_predictions.json"
    assert out.exists() and ips > 0
    res = json.load(open(out))
    assert isinstance(res, list)                      # a random-init model grounds nothing: the list is (almost surely) empty
    for r in res:
        assert set(r) == {"image_id", "category_id", "bbox", "score"}


def test_eval_countbench_batched_runs(setup):
    root, model_path, fx = setup
    from evaluation.eval_countbench import count_from_answer, eval_countbench
    acc, ips = eval_countbench(str(root / "countbench.json"), str(root / "no_such_folder"), model_path, "cuda:0", batch_size=3, limit=6,
                               synthetic_images=str(root / "synth_cb"), max_tokens=8)
    assert 0.0 <= acc <= 1.0 and ips > 0
    assert count_from_answer("<region12><region3> there are 7 cats, not 9") == 7 and count_from_answer("none <region5>") == 0


def test_generate_batch_equals_one_by_one(setup):
    root, model_path, fx = setup
    from evaluation.common import ImageSource
    from vlm_fo1.mm_utils import prepare_inputs
    from vlm_fo1.model.builder import load_pretrained_model
    tokenizer, model, procs = load_pretrained_model(model_path, device="cuda:0")
    sizes = {im["file_name"]: (im["width"], im["height"]) for im in fx["instances"]["images"]}
    src = ImageSource(str(root / "none"), str(root / "synth2"))
    kws = []
    for d in fx["coco"][8:13]:
        msg = [{"role": "user", "content": [{"type": "image_url", "image_url": {"url": src.path(d["image"], sizes[d["image"]])}},
                                             {"type": "text", "text": d["conversations"][0]["value"]}], "bbox_list": d["bbox_list"]}]
        kws.append(prepare_inputs(model_path, model, procs, tokenizer, msg, device="cuda:0", max_tokens=10, top_p=0.05, temperature=0.0, do_sample=False))
    batch = model.generate_batch(kws)
    for i, (kw, got) in enumerate(zip(kws, batch)):
        one = model.generate(**kw)
        P = kw["inputs"].shape[1]
        assert one.shape[1] > P
        # the one-layer random checkpoint has nearly flat logits, so a last-bit difference anywhere upstream would flip a token
        assert one.shape == got.shape and torch.equal(one, got), (i, one[0, P:].tolist(), got[0, P:].tolist())
