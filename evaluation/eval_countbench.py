"""Batched counting evaluation -- the reference's ``evaluation/eval_countbench.py`` (eval_countbench.py:13-64) with its per-image
loop run through ``model.generate_iter`` with ``--batch_size`` decode slots (items prepared ``WINDOW`` batches at a time): same json (``question`` / ``answer`` / ``image`` / ``bboxes``), same
``prepare_inputs`` arguments, same answer extraction (strip ``<regionN>``, first integer not preceded by "region", else 0),
accuracy printed the same way.  ``--synthetic_images DIR`` as in eval_coco.py."""
import json
import os
import re
import sys

from tqdm import tqdm

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evaluation.common import WINDOW, ImageSource, Throughput, batches, size_from_boxes  # noqa: E402
from vlm_fo1.mm_utils import prepare_inputs  # noqa: E402
from vlm_fo1.model.builder import load_pretrained_model  # noqa: E402


def count_from_answer(outputs: str) -> int:
    """eval_countbench.py:47-52"""
    ans = re.sub(r'<region\d+>', '', outputs)
    numbers = re.findall(r'(?<!region)\d+', ans)
    return int(numbers[0]) if numbers else 0


def eval_countbench(data_path, image_path, model_id, device, batch_size=8, limit=None, synthetic_images=None, max_tokens=4096):
    tokenizer, model, image_processors = load_pretrained_model(model_id, device=device)
    with open(data_path, "r") as f:
        data = json.load(f)
    if limit:
        data = data[:limit]
    src = ImageSource(image_path, synthetic_images)
    gt_list, pred_list = [], []
    thr = Throughput()
    for chunk in tqdm(list(batches(data, WINDOW * batch_size))):
        kwargs_list = []
        for item in chunk:
            im = src.path(item['image'], size_from_boxes(item['bboxes']))
            messages = [{"role": "user",
                         "content": [{"type": "image_url", "image_url": {"url": im}}, {"type": "text", "text": item['question']}],
                         "bbox_list": item['bboxes']}]
            kwargs_list.append(prepare_inputs(model_id, model, image_processors, tokenizer, messages, device=device, max_tokens=max_tokens,
                                              top_p=0.05, temperature=0.0, do_sample=False))
            kwargs_list[-1]["streamer"] = None       # many images decode at once: nothing is streamed
        outputs_ids = dict(model.generate_iter(kwargs_list, batch_size=batch_size))
        for i, (item, kw) in enumerate(zip(chunk, kwargs_list)):
            output_ids = outputs_ids[i]
            outputs = tokenizer.decode(output_ids[0, kw['inputs'].shape[1]:]).strip()
            pred = count_from_answer(outputs)
            pred_list.append(pred)
            gt_list.append(item['answer'])
            if item['answer'] != pred:
                print(f"gt is {item['answer']}, but pred is {outputs}")
        thr.add(len(chunk))
    correct = sum(1 for p, g in zip(pred_list, gt_list) if p == g)
    total = len(pred_list)
    accuracy = correct / total if total > 0 else 0
    print(f"Accuracy: {accuracy:.4f}")
    return accuracy, thr.report(f"eval_countbench (batch {batch_size})")


if __name__ == "__main__":
    import argparse
    parser = argparse.ArgumentParser()
    parser.add_argument("--data_path", type=str, default="evaluation/processed_data/countbench_with_upn_score_0.3_0.8.json")
    parser.add_argument("--image_path", type=str, default="data/CountBenchQA/images")
    parser.add_argument("--model_id", type=str, default='resources/VLM-FO1_Qwen2.5-VL-3B-v01')
    parser.add_argument("--device", type=str, default='cuda:0')
    parser.add_argument("--batch_size", type=int, default=8)
    parser.add_argument("--limit", type=int, default=None)
    parser.add_argument("--max_tokens", type=int, default=4096)
    parser.add_argument("--synthetic_images", type=str, default=None)
    args = parser.parse_args()
    eval_countbench(args.data_path, args.image_path, args.model_id, args.device, args.batch_size, args.limit, args.synthetic_images, args.max_tokens)
