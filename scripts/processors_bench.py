"""Logits processors against plain decoding: random-init FO1 language model at full depth (3B widths), 1195-token prompts, 64 new
tokens, no stop id.  Cases alternate inside each repetition; the median of 3 is printed.

  {mega, pk} x {greedy, sampled} x {plain, proc}    at B = 1, 8 and 32
  proc: no_repeat_ngram_size=3, 20 bad-word bigrams and min_new_tokens=32 (two eos ids) on every sequence, the prompt ids as the
  history's prompt.  A greedy call with processors runs the persistent kernel's sampled loop with top_k 1 (as a scored greedy call
  does); sampled calls are T 0.7, top-p 0.9, top-k 50.

Per case: decode time (64-token call minus a 1-token call) and the time per step.  A second, separate pass runs each per-kernel
processed case once under torch.profiler with eager launches and no PDL and prints logits_process_kernel's time per launch
(one launch per step).
Usage: python scripts/processors_bench.py [--layers 36] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--prompt", type=int, default=1195)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--batches", default="1,8,32")
    a = ap.parse_args()
    from tests.test_gpu_decode_parity import _model, _mods, make_seq
    E, _, _ = _mods()
    V = 151936
    eng, _ = _model(vocab=V, layers=a.layers, seed=3)
    print(f"# {card()}; layers {a.layers}, prompt {a.prompt}, new {a.new}", flush=True)
    g = torch.Generator().manual_seed(0)
    bad = tuple(tuple(int(x) for x in torch.randint(0, V, (2,), generator=g)) for _ in range(20))
    ps = E.ProcessorSet(no_repeat_ngram_size=3, bad_words_ids=bad, min_new_tokens=32, eos_token_ids=(151643, 151645))
    for B in (int(x) for x in a.batches.split(",")):
        seqs = [make_seq(a.prompt, None, 50 + b, vocab=V) for b in range(B)]
        emb = torch.cat([s.emb for s in seqs]).cuda()
        pos = torch.cat([s.pos for s in seqs], 1).cuda()
        lens, deltas = [s.L for s in seqs], [s.delta for s in seqs]
        prompt_ids = [torch.randint(0, V, (a.prompt,), generator=g).tolist() for _ in range(B)]
        procs = E.Processors([ps] * B, prompt_ids)
        samp = E.Sampling([0.7] * B, [0.9] * B, [50] * B, list(range(B)))

        def call(T, mega, sampled, proc):
            if mega:
                os.environ.pop("FO1_NO_MEGA", None)
            else:
                os.environ["FO1_NO_MEGA"] = "1"
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = eng.generate(emb, pos, lens, deltas, T, stop_ids=[], pad_id=0, early_exit_interval=0, sampling=samp if sampled else None,
                               processors=procs if proc else None)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, out

        cases = {f"{'mega' if m else 'pk'}-{'sampled' if sm else 'greedy'}-{'proc' if p else 'plain'}": dict(mega=m, sampled=sm, proc=p)
                 for m in (True, False) for sm in (False, True) for p in (False, True)}
        res = {n: [] for n in cases}
        for n, kw in cases.items():      # warm-up
            call(a.new, **kw); call(1, **kw)
        for _ in range(a.reps):
            for n, kw in cases.items():
                full, out = call(a.new, **kw)
                path = eng.last_decode_path()
                pre, _ = call(1, **kw)
                res[n].append((full - pre, out["steps_run"], path))
        for n, r in res.items():
            r.sort()
            dec, steps, path = r[len(r) // 2]
            base = sorted(res[n.replace("-proc", "-plain")])[len(r) // 2][0]
            print(json.dumps(dict(B=B, case=n, path=path, decode_ms=round(dec * 1e3, 2), steps=steps, step_ms=round(dec * 1e3 / max(steps, 1), 3),
                                  vs_plain=round(dec / base - 1.0, 4))), flush=True)
        # ---- the profiler pass (separate: eager launches, no PDL, so that every kernel is a trace event of its own) ----
        os.environ["FO1_NO_GRAPH"] = "1"; os.environ["FO1_NO_PDL"] = "1"
        for n, kw in cases.items():
            if kw["mega"] or not kw["proc"]:
                continue
            call(a.new, **kw)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                _, out = call(a.new, **kw)
            launches, total = 0, 0.0
            for ev in prof.key_averages():
                if "logits_process_kernel" in ev.key:
                    launches += ev.count
                    total += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            print(json.dumps(dict(B=B, case=n, logits_process_launches=launches,
                                  logits_process_us_per_launch=round(total / max(launches, 1), 2))), flush=True)
        os.environ.pop("FO1_NO_GRAPH"); os.environ.pop("FO1_NO_PDL")


if __name__ == "__main__":
    main()
