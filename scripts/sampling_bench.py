"""Cost of sampled decoding against greedy decoding, measured on the GPU (bench.py's flagship workload is greedy).

Three measurements on the same seeded inputs, variants alternating inside each repetition:
  1. greedy vs sampled (T 0.7, top-p 0.9, top-k 50) decode at the c3 shape (1195-token prompts, 64 new tokens) for B = 1, 8, 32,
     through the persistent decode kernel (default) and the per-kernel graph (FO1_NO_MEGA=1).  Decode time = time of a 64-token
     generate minus time of a 1-token generate (the prefill and the first token).
  2. sampled decode with top-k 50 against top-k 0 (top-p 0.9 alone) at B = 32 on both paths.
  3. fo1_sample_tokens alone over [32][151936] fp32 logits (CUDA events, 50 launches).
Random-init Qwen2.5-3B decoder (36 layers, real widths).  Prints the card name and power limit, then one JSON line per figure.

    python scripts/sampling_bench.py [--reps 3] [--layers 36]
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

import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figures stand without it, but say so
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--batches", default="1,8,32")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint"); W = import_module("vlm-fo1_b200.weights")
    assert torch.cuda.is_available(), "sampling_bench measures the GPU; there is no CPU path"
    print(f"card: {card()}", flush=True)
    cfg = E.EngineConfig()
    cfg.use_vit = cfg.use_davit = False
    cfg.proj_aux_layers = 0
    cfg.llm = dict(cfg.llm, num_hidden_layers=args.layers)
    sd = CK.random_llm(cfg.llm, torch.Generator(device="cuda").manual_seed(5), "cuda")
    eng = E.Engine(cfg)
    eng.set_weights(W.prepare_llm(sd, cfg.llm, eng.device))
    eng.finalize()
    P, T = 1195, 64

    def inputs(B):
        g = torch.Generator().manual_seed(B)
        emb = (torch.randn(B * P, cfg.llm["hidden_size"], generator=g) * 0.05).bfloat16().cuda()
        pos = torch.arange(P, dtype=torch.int32).view(1, -1).expand(3, -1).repeat(1, B).contiguous()
        return emb, pos, [P] * B, [0] * B

    def samp(B, k):
        return E.Sampling([0.7] * B, [0.9] * B, [k] * B, [1000 + b for b in range(B)])

    def timed(B, x, n, sampling):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.generate(*x, n, stop_ids=[], pad_id=0, early_exit_interval=0, sampling=sampling)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def decode_ms(B, x, sampling):
        return timed(B, x, T, sampling) - timed(B, x, 1, sampling)

    results = []
    for no_mega in (False, True):
        if no_mega:
            os.environ["FO1_NO_MEGA"] = "1"
        else:
            os.environ.pop("FO1_NO_MEGA", None)
        path = "per-kernel" if no_mega else "mega"
        for B in [int(b) for b in args.batches.split(",")]:
            x = inputs(B)
            for s in (None, samp(B, 50)):        # warm every shape
                timed(B, x, T, s); timed(B, x, 1, s)
            timed(B, x, T, samp(B, 50))
            sampled_path = eng.last_decode_path()  # 1: the persistent kernel ran the sampled 64-token decode
            g_ms, s_ms = [], []
            for _ in range(args.reps):
                g_ms.append(decode_ms(B, x, None))
                s_ms.append(decode_ms(B, x, samp(B, 50)))
            r = dict(figure="greedy_vs_sampled_decode", path=path, B=B, new_tokens=T, greedy_ms=[round(v, 2) for v in g_ms],
                     sampled_ms=[round(v, 2) for v in s_ms], overhead_pct=round(100 * (min(s_ms) / min(g_ms) - 1), 2),
                     sampled_path=sampled_path)
            print(json.dumps(r), flush=True)
            results.append(r)
        B = 32
        x = inputs(B)
        timed(B, x, T, samp(B, 0)); timed(B, x, 1, samp(B, 0))
        k50, k0 = [], []
        for _ in range(args.reps):
            k50.append(decode_ms(B, x, samp(B, 50)))
            k0.append(decode_ms(B, x, samp(B, 0)))
        r = dict(figure="topk50_vs_topk0_decode", path=path, B=B, k50_ms=[round(v, 2) for v in k50], k0_ms=[round(v, 2) for v in k0])
        print(json.dumps(r), flush=True)
    os.environ.pop("FO1_NO_MEGA", None)
    # ---- the standalone kernel ----
    V = cfg.llm["vocab_size"]
    logits = torch.randn(32, V, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda") * 3
    for k, p in ((50, 0.9), (0, 0.9), (0, 1.0), (1, 1.0)):
        n = 32
        for _ in range(3):
            E.sample_tokens(logits, [0.7] * n, [p] * n, [k] * n, list(range(n)), step=0)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        steps = torch.zeros(n, dtype=torch.int32, device="cuda")
        ev0.record()
        for i in range(50):
            E.sample_tokens(logits, [0.7] * n, [p] * n, [k] * n, list(range(n)), step=steps)
        ev1.record()
        torch.cuda.synchronize()
        r = dict(figure="fo1_sample_tokens", rows=n, vocab=V, top_k=k, top_p=p, us_per_call=round(ev0.elapsed_time(ev1) / 50 * 1e3, 1))
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
