"""Batched COCO detection evaluation -- the reference's ``evaluation/eval_coco.py`` (eval_coco.py:12-103) with its per-image loop
(:36-88) run through ``model.generate_iter`` with ``--batch_size`` decode slots (a finished image hands its slot to the next one;
items are prepared ``WINDOW`` batches at a time): same inputs (the UPN proposal jsonl, the
COCO ``instances`` json for the category ids), same prompt per item (``conversations[0]['value']``), same
``prepare_inputs`` arguments (max_tokens=4096, top_p=0.05, temperature=0.0), same post-processing
(``extract_predictions_to_indexes`` -> one COCO result dict per (label, region index) whose label is a COCO category)
and the same ``<out_dir>/<model>/<file>_predictions.json``.  ``--synthetic_images DIR`` stands noise images of the recorded
sizes in for a missing image folder (throughput runs on the real box-count distribution)."""
import json
import os
import sys

from tqdm import tqdm

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from evaluation.common import WINDOW, ImageSource, Throughput, batches  # noqa: E402
from vlm_fo1.mm_utils import extract_predictions_to_indexes, prepare_inputs  # noqa: E402
from vlm_fo1.model.builder import load_pretrained_model  # noqa: E402


def eval_coco(model_id, eval_data_path, original_data_path, img_folder, out_dir=None, device='cuda:0', batch_size=16, limit=None,
              synthetic_images=None, max_tokens=4096):
    print(f"Evaluating {model_id} on {eval_data_path}...")
    tokenizer, model, image_processors = load_pretrained_model(model_id, device=device)

    output_path = os.path.join(out_dir, model_id.rstrip("/").split("/")[-1])
    os.makedirs(output_path, exist_ok=True)

    with open(eval_data_path, 'r') as f:
        data_list = [json.loads(line) for line in f]
    if limit:
        data_list = data_list[:limit]
    print(len(data_list))

    original_data = json.load(open(original_data_path, 'r'))
    catName_to_catId = {item['name']: item['id'] for item in original_data['categories']}
    sizes = {im['file_name']: (im['width'], im['height']) for im in original_data.get('images', [])}
    src = ImageSource(img_folder, synthetic_images)

    res_list = []
    filename = eval_data_path.split('/')[-1].replace('.jsonl', '')
    out_data_path = f'{output_path}/{filename}_predictions.json'
    thr = Throughput()

    for chunk in tqdm(list(batches(data_list, WINDOW * batch_size))):
        kwargs_list = []
        for data in chunk:
            image_path = src.path(data['image'], sizes.get(data['image'], (640, 480)))
            messages = [{"role": "user",
                         "content": [{"type": "image_url", "image_url": {"url": image_path}},
                                     {"type": "text", "text": data['conversations'][0]['value']}],
                         "bbox_list": data['bbox_list']}]
            kwargs_list.append(prepare_inputs(model_id, model, image_processors, tokenizer, messages, device=device, max_tokens=max_tokens,
                                              top_p=0.05, temperature=0.0, do_sample=False))
            kwargs_list[-1]["streamer"] = None       # many images decode at once: nothing is streamed
        # the reference skips a failing image (:63-65): a request whose admission fails is reported and left out
        outputs = dict(model.generate_iter(kwargs_list, batch_size=batch_size,
                                           on_error=lambda i, exc: print(f"Error: {chunk[i]['id']} ({exc!r})")))
        for i, (data, kw) in enumerate(zip(chunk, kwargs_list)):
            if i not in outputs:
                continue
            ans = tokenizer.decode(outputs[i][0, kw['inputs'].shape[1]:]).strip()
            print('ans:', ans)
            bbox_list, score_list = data['bbox_list'], data['score_list']
            for k, v in extract_predictions_to_indexes(ans).items():
                for box in v:
                    if k in catName_to_catId and 0 <= box < len(bbox_list):
                        current_bbox = bbox_list[box]
                        res_list.append({"image_id": data['id'], "category_id": catName_to_catId[k],
                                         "bbox": [current_bbox[0], current_bbox[1], current_bbox[2] - current_bbox[0], current_bbox[3] - current_bbox[1]],
                                         "score": score_list[box]})
        thr.add(len(chunk))

    print(f"predictions saved to: {out_data_path}")
    json.dump(res_list, open(out_data_path, 'w'))
    return thr.report(f"eval_coco (batch {batch_size})")


if __name__ == "__main__":
    import argparse
    parser = argparse.ArgumentParser()
    parser.add_argument("--model_id", type=str, default='resources/VLM-FO1_Qwen2.5-VL-3B-v01')
    parser.add_argument("--eval_data_path", type=str, default='evaluation/processed_data/cocoVal2017_with_upn_score_0.3_0.8.jsonl')
    parser.add_argument("--original_data_path", type=str, default='evaluation/processed_data/instances_val2017.json')
    parser.add_argument("--img_folder", type=str, default='data/coco/val2017')
    parser.add_argument("--out_dir", type=str, default='./evaluation')
    parser.add_argument("--device", type=str, default='cuda:0')
    parser.add_argument("--batch_size", type=int, default=16)
    parser.add_argument("--limit", type=int, default=None)
    parser.add_argument("--max_tokens", type=int, default=4096)
    parser.add_argument("--synthetic_images", type=str, default=None, help="directory for stand-in noise images when --img_folder lacks a file")
    args = parser.parse_args()
    eval_coco(args.model_id, args.eval_data_path, args.original_data_path, args.img_folder, args.out_dir, args.device, args.batch_size,
              args.limit, args.synthetic_images, args.max_tokens)
