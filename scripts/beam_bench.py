"""Beam search against greedy decoding, measured on the GPU.

One synthetic 896 px image with 64 boxes; 64 new tokens with no stop id (every beam runs all 64 steps); random-init FO1 at full
depth (ViT 32, DaViT-large, Qwen2.5-3B 36 layers).  For N = 1 (greedy on the per-kernel path, the one beam search runs on) and
N = 2, 4, 8 beams, each repetition alternates beam search on the one prompt with greedy decoding of N copies of it (B = N rows,
per-kernel path); medians of the repetitions.  Reported per N:
  decode step  (LLM call with 64 tokens - LLM call with 1 token) / 63, beam search and greedy at B = N;
  beam kernels the per-step time of beam_rows / beam_select / beam_kv_reorder (torch.profiler CUDA activity of one extra call with
               eager launches and no PDL), and their share of the beam decode step;
  prefill      the 1-token LLM call of beam search against greedy at B = 1.
Prints the card name and power limit, then one JSON line per N.

    python scripts/beam_bench.py [--reps 3] [--ns 1,2,4,8]
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

T = 64
BEAM_KERNELS = ("beam_rows_kernel", "beam_select_kernel", "beam_kv_reorder_kernel")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figures stand without it, but say so
        return f"unknown ({e})"


def llm_ms(pipe, samples, tokens, beams):
    """the LLM stage (prefill + decode) of one pipeline call, per-kernel path"""
    pipe.profile_stages = True
    try:
        torch.cuda.synchronize()
        out = pipe.generate(samples, tokens, stop_ids=[], early_exit_interval=0, beams=beams)
        torch.cuda.synchronize()
        return pipe.stage_ms()["llm_prefill_decode"], out
    finally:
        pipe.profile_stages = False


def beam_kernel_us(pipe, sample, beams):
    """per-step device time of each beam kernel over one call with eager launches and no programmatic dependent launch (under PDL a
    kernel starts early and waits for its predecessor, so its span would include the predecessor's time)"""
    from torch.profiler import ProfilerActivity, profile
    os.environ["FO1_NO_GRAPH"] = os.environ["FO1_NO_PDL"] = "1"
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            pipe.generate([sample], T, stop_ids=[], early_exit_interval=0, beams=beams)
            torch.cuda.synchronize()
    finally:
        del os.environ["FO1_NO_GRAPH"], os.environ["FO1_NO_PDL"]
    tot = {k: 0.0 for k in BEAM_KERNELS}
    for ev in prof.events():
        for k in BEAM_KERNELS:
            if k in ev.name:
                tot[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    steps = {"beam_rows_kernel": T, "beam_select_kernel": T, "beam_kv_reorder_kernel": T - 1}
    return {k: tot[k] / steps[k] for k in BEAM_KERNELS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ns", default="1,2,4,8")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    P = import_module("vlm-fo1_b200.pipeline"); SY = import_module("vlm-fo1_b200.synthetic")
    assert torch.cuda.is_available(), "beam_bench measures the GPU; there is no CPU path"
    print(f"card: {card()}", flush=True)
    os.environ["FO1_NO_MEGA"] = "1"           # greedy on the per-kernel path, the path beam search runs on
    cfg = E.EngineConfig()
    eng = CK.load_engine(cfg, CK.random_state_dicts(cfg, "cuda", 0))
    pipe = P.Fo1Pipeline(eng)
    pipe._share_inputs = False                # greedy B = N decodes N independent full prompts (no shared prefix)
    s = SY.synthetic_sample(0, 896, 64)
    sample = P.SampleInputs(s.input_ids, s.pixel_values.cuda(), s.grid_hw, s.image_aux.cuda(), s.boxes.cuda())
    greedy1 = []
    for N in [int(n) for n in args.ns.split(",")]:
        beams = E.Beams(N, 2 * N, 1.0, False, 1) if N > 1 else None
        arms = {"beam": ([sample], beams), "greedy": ([sample] * N, None)}
        for name, (smp, bm) in arms.items():         # warm every shape
            llm_ms(pipe, smp, T, bm); llm_ms(pipe, smp, 1, bm)
        rec = {k: [] for k in arms}
        for _ in range(args.reps):
            for name, (smp, bm) in arms.items():
                t64, out = llm_ms(pipe, smp, T, bm)
                t1, _ = llm_ms(pipe, smp, 1, bm)
                rec[name].append(dict(step_ms=(t64 - t1) / (T - 1), prefill_ms=t1))
                assert eng.last_decode_path() in (0, -1)
        med = {k: {f: float(np.median([r[f] for r in v])) for f in v[0]} for k, v in rec.items()}
        line = {"N": N, "card": card(), "tokens": T,
                "beam_step_ms": round(med["beam"]["step_ms"], 3), "greedy_step_ms_at_B_eq_N": round(med["greedy"]["step_ms"], 3),
                "beam_prefill_ms": round(med["beam"]["prefill_ms"], 2)}
        if N == 1:
            greedy1.append(med["greedy"]["prefill_ms"])
        line["greedy_prefill_ms_at_B_eq_1"] = round(greedy1[0], 2) if greedy1 else None
        if N > 1:
            us = beam_kernel_us(pipe, sample, beams)
            line["beam_kernels_us_per_step"] = {k.replace("_kernel", ""): round(v, 1) for k, v in us.items()}
            sel_reorder = us["beam_select_kernel"] + us["beam_kv_reorder_kernel"]
            line["select_plus_reorder_share_of_step"] = round(sel_reorder / 1e3 / med["beam"]["step_ms"], 4)
            line["all_beam_kernels_share_of_step"] = round(sum(us.values()) / 1e3 / med["beam"]["step_ms"], 4)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
