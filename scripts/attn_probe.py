"""Attention micro-benchmark (CUDA events, median of 10, L2 flushed): the shapes of one C3 step.
Prints one JSON object per shape; `python scripts/attn_probe.py ncu` runs each shape once (for an ncu capture)."""
import json, os, sys
import numpy as np
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from importlib import import_module
import fo1_b200  # noqa
ops = import_module("vlm-fo1_b200.ops")
NCU = len(sys.argv) > 1 and sys.argv[1] == "ncu"
PEAK = json.load(open(os.path.join(REPO, "MEASURED_PEAKS.json")))["bf16_tflops"] if os.path.exists(os.path.join(REPO, "MEASURED_PEAKS.json")) else 989.0   # H100 SXM data sheet, dense bf16
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def run(name, lens, qh, kvh, hd, causal):
    T = sum(lens)
    qkv = torch.randn(T, (qh + 2 * kvh) * hd, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, : qh * hd], qkv[:, qh * hd:(qh + kvh) * hd], qkv[:, (qh + kvh) * hd:]
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")
    out = torch.empty(T, qh * hd, device="cuda", dtype=torch.bfloat16)
    f = lambda: ops.attention_varlen(q, k, v, cu, max(lens), qh, kvh, hd, hd ** -0.5, causal=causal, out=out)
    fl = sum(4.0 * n * n * qh * hd * (0.5 if causal else 1.0) for n in lens)
    if NCU:
        f(); torch.cuda.synchronize(); return
    for _ in range(3):
        f()
    ts = []
    for _ in range(10):
        flush.zero_()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); f(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = float(np.median(ts))
    print(json.dumps({"shape": name, "T": T, "heads": qh, "hd": hd, "causal": causal, "ms": ms, "tflops": fl / ms / 1e9,
                      "frac_of_measured_burst": fl / ms / 1e9 / PEAK, "GBs_qkvo": (qkv.numel() + out.numel()) * 2 / ms / 1e6}), flush=True)


run("vit_full_8x4096", [4096] * 8, 16, 16, 80, False)
run("vit_full_32x4096", [4096] * 32, 16, 16, 80, False)
run("vit_window_32x4096", [64] * (64 * 32), 16, 16, 80, False)
run("llm_prefill_8x1195", [1195] * 8, 16, 2, 128, True)
run("llm_prefill_32x1195", [1195] * 32, 16, 2, 128, True)
run("davit_s2_32x25x144", [144] * (25 * 32), 32, 32, 32, False)
run("vit_full_8x9216", [9216] * 8, 16, 16, 80, False)
