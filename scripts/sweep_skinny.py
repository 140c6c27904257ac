"""Tile-width / split-K sweep of the decode (M = batch) GEMMs on one H100.  Each configuration streams a ROTATION of
distinct weight matrices (> L2 in total, like the 36 layers of a decode step) captured in one CUDA graph, so the
number is the steady-state back-to-back time per launch, not a cold single launch.
Writes bench_out/sweep_skinny_<tag>.json."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from importlib import import_module

import fo1_b200  # noqa: E402

ops = import_module("vlm-fo1_b200.ops")

SHAPES = {"qkv": (2560, 2048, False, True), "o": (2048, 2048, False, False), "gateup": (22016, 2048, True, False),
          "down": (2048, 11008, False, False)}
CANDS = {
    "qkv": [None, (32, 1), (32, 2), (64, 2), (64, 3), (64, 4), (64, 7), (128, 4), (128, 7), (128, 8), (128, 14), (256, 8), (256, 14), (256, 16)],
    "o": [None, (32, 2), (32, 4), (64, 4), (64, 8), (128, 8), (128, 9), (128, 16), (256, 16), (256, 18)],
    "gateup": [None, (64, 1), (128, 1), (192, 1), (256, 1), (64, 3), (128, 3), (128, 6), (128, 7), (256, 5), (256, 7), (256, 12), (64, 2)],
    "down": [None, (32, 2), (32, 4), (64, 4), (64, 9), (128, 8), (128, 9), (128, 18), (128, 27), (256, 16), (256, 18), (256, 36)],
}


def run(name, M):
    N, K, gated, has_bias = SHAPES[name]
    nW = max(8, int(700e6 / (N * K * 2)) + 1)
    ws = [(torch.randn(N, K, device="cuda") * 0.03).to(torch.bfloat16) for _ in range(nW)]
    a = (torch.randn(M, K, device="cuda") * 0.5).to(torch.bfloat16)
    bias = (torch.randn(N, device="cuda") * 0.1).to(torch.bfloat16) if has_bias else None
    n_out = N // 2 if gated else N
    out = torch.empty(M, n_out, device="cuda", dtype=torch.bfloat16)
    ref = None
    res = []
    for cand in CANDS[name]:
        tn, sk = cand or (0, 0)
        fn = lambda w: ops.gemm(a, w, bias=bias, act="silu" if gated else None, gated=gated, out=out, tile_n=tn, split_k=sk)
        try:
            fn(ws[0]); torch.cuda.synchronize()
            got = out.float().clone()
            if ref is None:
                ref = got
            err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-9)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for w in ws[:2]:
                    fn(w)
                s.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for w in ws:
                        fn(w)
            ts = []
            for _ in range(5):
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3 / nW)
            us = sorted(ts)[len(ts) // 2]
            byt = 2.0 * (N * K + M * K + M * n_out)
            r = {"name": name, "M": M, "N": N, "K": K, "cfg": "default" if cand is None else f"bn{cand[0]}_ks{cand[1]}", "us": round(us, 2),
                 "GBs": round(byt / us / 1e3, 1), "rel_err_vs_default": err}
        except Exception as ex:  # noqa
            r = {"name": name, "cfg": str(cand), "error": str(ex)[:200]}
        print(json.dumps(r), flush=True)
        res.append(r)
    return res


if __name__ == "__main__":
    tag = sys.argv[1] if len(sys.argv) > 1 else "a"
    M = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    names = sys.argv[3:] or list(SHAPES)
    allr = []
    for n in names:
        allr += run(n, M)
    os.makedirs(os.path.join(REPO, "bench_out"), exist_ok=True)
    json.dump(allr, open(os.path.join(REPO, "bench_out", f"sweep_skinny_{tag}.json"), "w"), indent=1)
