"""Shared-prefix generation against the unshared path: K questions about one image, measured on the GPU.

One synthetic 896 px image with 64 boxes; K prompts that share the system turn, the image and the region tokens and differ in a
15-30 token question; 64 new greedy tokens; random-init FO1 at full depth (ViT 32, DaViT-large, Qwen2.5-3B 36 layers).  For each K the
shared path (the default) and the unshared one (the pipeline's private switch) alternate inside each repetition; median of the
repetitions.  Reported per path: call time, encode (towers + projector), the LLM call with 64 tokens and with 1 token (prefill and
the first token), and decode = their difference.  The tokens of the two paths must be identical.  Prints the card name and power
limit, then one JSON line per K.

    python scripts/prefix_bench.py [--reps 3] [--ks 1,8,32,80]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from importlib import import_module

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

ENCODE = ("preprocess", "vit", "davit", "fpn", "hfre", "projector")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figures stand without it, but say so
        return f"unknown ({e})"


def questions(base, K):
    P = import_module("vlm-fo1_b200.pipeline")
    cut = max(i for i, t in enumerate(base.input_ids) if t == -300) + 1
    out = []
    for q in range(K):
        g = torch.Generator().manual_seed(500 + q)
        ids = list(base.input_ids[:cut]) + [1000 + q] + torch.randint(0, 151643, (14 + q % 16,), generator=g).tolist()
        ids += [151645, 198, 151644, 77091, 198]
        out.append(P.SampleInputs(ids, base.pixel_values.clone(), base.grid_hw, base.image_aux.clone(), base.boxes.clone()))
    return out


def timed(pipe, samples, shared, T):
    pipe._share_inputs = shared
    pipe.profile_stages = True
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipe.generate(samples, T, stop_ids=[], early_exit_interval=0)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        st = pipe.stage_ms()
    finally:
        pipe._share_inputs = True
        pipe.profile_stages = False
    return ms, st, out["tokens"].cpu()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ks", default="1,8,32,80")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    P = import_module("vlm-fo1_b200.pipeline"); SY = import_module("vlm-fo1_b200.synthetic")
    assert torch.cuda.is_available(), "prefix_bench measures the GPU; there is no CPU path"
    print(f"card: {card()}", flush=True)
    cfg = E.EngineConfig()
    eng = CK.load_engine(cfg, CK.random_state_dicts(cfg, "cuda", 0))
    pipe = P.Fo1Pipeline(eng)
    s = SY.synthetic_sample(0, 896, 64)
    base = P.SampleInputs(s.input_ids, s.pixel_values.cuda(), s.grid_hw, s.image_aux.cuda(), s.boxes.cuda())
    for K in [int(k) for k in args.ks.split(",")]:
        samples = questions(base, K)
        for shared in (True, False):              # warm every shape
            timed(pipe, samples, shared, 64); timed(pipe, samples, shared, 1)
        rec = {True: [], False: []}
        toks = {}
        for _ in range(args.reps):
            for shared in (True, False):
                ms, st, tk = timed(pipe, samples, shared, 64)
                _, st1, _ = timed(pipe, samples, shared, 1)
                enc = sum(v for k, v in st.items() if k in ENCODE)
                rec[shared].append(dict(call_ms=ms, encode_ms=enc, splice_ms=st.get("splice", 0.0), llm64_ms=st["llm_prefill_decode"],
                                        llm1_ms=st1["llm_prefill_decode"]))
                toks[shared] = tk
        assert torch.equal(toks[True], toks[False]), f"K={K}: shared and unshared tokens differ"
        line = {"K": K, "card": card(), "tokens_identical": True}
        for shared, name in ((True, "shared"), (False, "unshared")):
            med = {k: float(np.median([r[k] for r in rec[shared]])) for k in rec[shared][0]}
            med["decode_ms"] = med["llm64_ms"] - med["llm1_ms"]
            line[name] = {k: round(v, 1) for k, v in med.items()}
        sh, un = line["shared"], line["unshared"]
        line["encode_plus_prefill_ratio"] = round((sh["encode_ms"] + sh["llm1_ms"]) / (un["encode_ms"] + un["llm1_ms"]), 3)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
