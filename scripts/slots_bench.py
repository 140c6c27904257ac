"""In-flight batching (Fo1Pipeline.generate_continuous over a slot pool) against static batches (Fo1Pipeline.generate on chunks of B
requests, what generate_batch runs) on one GPU, random-init FO1 at full depth, N requests on S px noise images with K boxes, no stop
id, so each request's length is its own max_new_tokens:
  (a) every request 64 tokens;
  (b) ragged: max_new_tokens drawn log-uniformly from [8, 512] with a fixed seed.
At each B the two are alternated within every repetition; the median of the repetitions is reported with images/s, decode steps,
mean running rows per step and, for (b), the ideal ratio sum over chunks of the chunk's longest length / (sum of lengths / B): the
speed-up if decode steps were all the time and the slot pool never stalled.  Both runs' tokens must be equal (for the requests in
full chunks of B).  Prints one JSON line
per (workload, B) and the card's name and power limit read in the same run; for the slots also the number of decode segments and a
least-squares split of segment time into a per-step and a per-segment cost.  B > 32 runs the per-kernel decode path."""
import argparse
import json
import os
import subprocess
import sys
import time
from importlib import import_module

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--size", type=int, default=896)
    ap.add_argument("--boxes", type=int, default=64)
    ap.add_argument("--slots", type=str, default="8,16,32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    P = import_module("vlm-fo1_b200.pipeline"); SY = import_module("vlm-fo1_b200.synthetic")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = E.EngineConfig()
    sds = CK.random_state_dicts(cfg, dev, 0)
    eng = CK.load_engine(cfg, sds, dev)
    del sds
    torch.cuda.empty_cache()
    pipe = P.Fo1Pipeline(eng)
    N = args.requests
    samples = [P.SampleInputs(s.input_ids, s.pixel_values.to(dev), s.grid_hw, s.image_aux.to(dev), s.boxes.to(dev))
               for s in SY.synthetic_batch(0, N, args.size, args.boxes)]
    rng = np.random.default_rng(args.seed)
    ragged = [int(round(x)) for x in np.exp(rng.uniform(np.log(8), np.log(512), N))]
    workloads = {"a": [64] * N, "b": ragged}

    steps = [0]
    segments = []                   # (seconds, steps) of every decode segment of the last iterated run
    decode = E.SlotPool.decode

    def counted(self, exit_at):
        torch.cuda.synchronize()    # the admission's prefill is not part of the segment
        t0 = time.perf_counter()
        n = decode(self, exit_at)   # (ends in a synchronise)
        if n > 0:
            segments.append((time.perf_counter() - t0, n))
        steps[0] += n
        return n
    E.SlotPool.decode = counted

    def static(B, mnt):
        toks, st = {}, 0
        for c in range(0, N, B):
            idx = list(range(c, min(N, c + B)))
            T = max(mnt[i] for i in idx)
            out = pipe.generate([samples[i] for i in idx], T, stop_ids=[], early_exit_interval=0)
            st += T - 1
            for j, i in enumerate(idx):
                toks[i] = out["tokens"][j, :mnt[i]].clone()
        return toks, st

    def iterated(B, mnt):
        steps[0] = 0
        segments.clear()
        toks = {i: t for i, t, _ in pipe.generate_continuous(samples, B, mnt, stop_ids=[])}
        return toks, steps[0]

    def timed(fn, *a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn(*a)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def fit_segments():
        """(segments, ms per step, ms per segment): least squares of segment time = a * steps + b.  b is the fixed cost of a segment
        (the host checks, the first eager step, on the per-kernel path the capture and instantiation of its CUDA graph, the syncs)."""
        if len(segments) < 2:
            return len(segments), None, None
        A = np.array([[n, 1.0] for _, n in segments])
        a, b = np.linalg.lstsq(A, np.array([t for t, _ in segments]), rcond=None)[0]
        return len(segments), float(a) * 1e3, float(b) * 1e3

    slot_counts = [int(x) for x in args.slots.split(",")]
    for B in slot_counts:           # warm every shape the timed runs use
        static(B, [8] * N)
        iterated(B, [8] * N)
        print(f"# warmed B={B}", file=sys.stderr, flush=True)
    useful = {w: sum(m - 1 for m in mnt) for w, mnt in workloads.items()}
    for B in slot_counts:
        res = {w: {"static": [], "iter": []} for w in workloads}
        fits = {w: [] for w in workloads}
        for rep in range(args.reps):
            for w, mnt in workloads.items():
                ts, (tok_s, st_s) = timed(static, B, mnt)
                ti, (tok_i, st_i) = timed(iterated, B, mnt)
                # the contract: a request equals itself in a static batch of B requests, so a last chunk of fewer than B (another key
                # split, other GEMM shapes) is left out of the comparison
                assert all(torch.equal(tok_s[i], tok_i[i]) for i in range(N - N % B)), (w, B, "tokens differ")
                res[w]["static"].append((ts, st_s))
                res[w]["iter"].append((ti, st_i))
                fits[w].append(fit_segments())
                print(f"# B={B} rep={rep} ({w}): static {ts:.2f} s, slots {ti:.2f} s", file=sys.stderr, flush=True)
        for w, r in res.items():
            mnt = workloads[w]
            line = dict(workload=w, slots=B, requests=N, size=args.size, boxes=args.boxes, card=card, reps=args.reps, tokens_equal="full chunks" if N % B else True)
            for k in ("static", "iter"):
                t = float(np.median([x[0] for x in r[k]]))
                st = r[k][0][1]
                line[k] = dict(images_per_s=round(N / t, 3), seconds=round(t, 3), decode_steps=st,
                               mean_running_rows=round(useful[w] / max(st, 1), 2), seconds_all=[round(x[0], 3) for x in r[k]])
            n_seg, ms_step, ms_seg = fits[w][0]
            line["iter"]["segments"] = n_seg
            if ms_seg is not None:
                line["iter"]["segment_fit_ms"] = dict(per_step=round(ms_step, 3), per_segment=[round(f[2], 2) for f in fits[w]])
            line["speedup"] = round(line["iter"]["images_per_s"] / line["static"]["images_per_s"], 3)
            if w == "b":
                line["ideal_ratio"] = round(sum(max(mnt[c:c + B]) for c in range(0, N, B)) / (sum(mnt) / B), 3)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
