"""Candidate ranking on the GPU: K answers about one image scored by Fo1Pipeline.score against per-candidate generate with all_logits.

One synthetic 896 px image with 64 boxes and one question; K candidate answers of 2-12 tokens each (the labels cover the answer);
random-init FO1 at full depth (ViT 32, DaViT-large, Qwen2.5-3B 36 layers).  Two arms, alternated inside each repetition, median of
the repetitions:
  (a) score:    Fo1Pipeline.score over the K samples (towers once, the common prefix prefilled once, the log-likelihood head on the
                scored rows only);
  (b) generate: per candidate, the towers, the splice and Engine.generate with all_logits (max_new_tokens 1), then torch log_softmax /
                gather over the answer rows.
Reported per arm: call time (synchronised), peak device memory of the call (torch.cuda.max_memory_allocated), and the summed
log-probabilities of (a) against (b) (they differ by the two heads' summation orders only).  A separate torch.profiler pass over
(a) gives the log-likelihood GEMM's and merge kernel's device time.  Prints the card name and power limit, then one JSON line per K.

    python scripts/loglik_bench.py [--reps 3] [--ks 1,8,32,80]
"""
import argparse
import json
import os
import sys
import time
from importlib import import_module

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from prefix_bench import card  # noqa: E402


def candidates(base, K):
    P = import_module("vlm-fo1_b200.pipeline")
    cut = max(i for i, t in enumerate(base.input_ids) if t == -300) + 1
    g = torch.Generator().manual_seed(7)
    q = list(base.input_ids[:cut]) + torch.randint(0, 151643, (20,), generator=g).tolist() + [151645, 198, 151644, 77091, 198]
    samples, labels = [], []
    for k in range(K):
        n = 2 + k % 11
        ans = torch.randint(0, 151643, (n,), generator=g).tolist()
        samples.append(P.SampleInputs(q + ans, base.pixel_values.clone(), base.grid_hw, base.image_aux.clone(), base.boxes.clone()))
        labels.append([-100] * len(q) + ans)
    return samples, labels


def arm_score(pipe, samples, labels):
    out = pipe.score(samples, labels)
    return out["seq_logprob"].cpu().numpy()


def arm_generate(pipe, samples, labels):
    P = import_module("vlm-fo1_b200.pipeline")
    res = []
    eng = pipe.eng
    for s, lab in zip(samples, labels):
        feats, _, region_tokens, _ = pipe.encode([s])
        plan = P.splice_plan_batch([s.input_ids], [[s.grid_hw]], [region_tokens[0].shape[0]], eng.device,
                                   merge=eng.cfg.vit["spatial_merge_size"], **pipe.ids)
        emb = eng.build_embeds(plan["kind"], plan["index"], feats, torch.cat(region_tokens, 0))
        out = eng.generate(emb, plan["position_ids"], plan["lens"], plan["rope_delta"], 1, [], 0, want_all_logits=True, early_exit_interval=0)
        al = out["all_logits"]
        L = al.shape[0]
        tg = torch.tensor(P.shift_targets(P.splice_labels(s.input_ids, lab, L - len(s.input_ids) + 1)), device=al.device)
        keep = (tg != -100).nonzero().view(-1)
        lp = torch.log_softmax(al[keep], -1).gather(1, tg[keep][:, None])
        res.append(float(lp.double().sum()))
        del out, al
    return np.asarray(res)


def timed(fn, *a):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    r = fn(*a)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, r


def head_kernel_ms(pipe, samples, labels):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.score(samples, labels)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if "gemm_bf16_wgmma_kernel<128, 1, true>" in e.name or "loglik_merge" in e.name or "Lb1E" in e.name:
            tot[e.name] = tot.get(e.name, 0.0) + e.device_time_total / 1e3
    return {("gemm_loglik" if ("true" in k or "Lb1E" in k) else "merge"): round(v, 3) for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ks", default="1,8,32,80")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    P = import_module("vlm-fo1_b200.pipeline"); SY = import_module("vlm-fo1_b200.synthetic")
    assert torch.cuda.is_available(), "loglik_bench measures the GPU; there is no CPU path"
    print(f"card: {card()}", flush=True)
    cfg = E.EngineConfig()
    eng = CK.load_engine(cfg, CK.random_state_dicts(cfg, "cuda", 0))
    pipe = P.Fo1Pipeline(eng)
    s = SY.synthetic_sample(0, 896, 64)
    base = P.SampleInputs(s.input_ids, s.pixel_values.cuda(), s.grid_hw, s.image_aux.cuda(), s.boxes.cuda())
    for K in [int(k) for k in args.ks.split(",")]:
        samples, labels = candidates(base, K)
        arms = (("score", arm_score), ("generate", arm_generate))
        for _, fn in arms:                  # warm every shape
            fn(pipe, samples, labels)
        rec = {n: [] for n, _ in arms}
        vals = {}
        for _ in range(args.reps):
            for n, fn in arms:
                ms, mb, v = timed(fn, pipe, samples, labels)
                rec[n].append((ms, mb))
                vals[n] = v
        line = {"K": K, "card": card(), "max_abs_seq_logprob_diff": float(np.abs(vals["score"] - vals["generate"]).max())}
        for n, _ in arms:
            line[n] = {"call_ms": round(float(np.median([r[0] for r in rec[n]])), 1),
                       "peak_mib": round(float(np.median([r[1] for r in rec[n]])), 1)}
        line["speedup"] = round(line["generate"]["call_ms"] / line["score"]["call_ms"], 2)
        line["head_kernel_ms"] = head_kernel_ms(pipe, samples, labels)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
