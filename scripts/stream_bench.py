"""Cost of streamed decoding (Engine.generate(on_tokens=...), include/fo1.h fo1_stream_desc) on top of greedy and sampled decoding,
measured on the GPU, and how promptly the host sees the tokens.

At the c3 shape (1195-token prompts, 64 new tokens) for B = 1 and 8, through the persistent decode kernel (default) and the
per-kernel graph (FO1_NO_MEGA=1), four cases on the same seeded inputs, alternating inside each repetition:
  greedy; greedy + streaming; sampled (T 0.7, top-p 0.9, top-k 50); sampled + streaming.
Decode time = time of a 64-token generate minus time of a 1-token generate (the prefill and the first token); the median of the
repetitions is reported.  For the streamed cases also: the time from the call to the first on_tokens (prefill + column 0 + the
poll), and the median host-observed gap per column (time between on_tokens calls / columns they brought) against the device
step time (decode time / 63).  Random-init Qwen2.5-3B decoder (36 layers, real widths).  Prints the card name and power limit,
then one JSON line per (path, B).

    python scripts/stream_bench.py [--reps 3] [--layers 36] [--batches 1,8]
"""
import argparse
import json
import os
import statistics
import sys
import time
from importlib import import_module

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from scripts.sampling_bench import card  # noqa: E402

CASES = (("greedy", False, False), ("greedy_stream", False, True), ("sampled", True, False), ("sampled_stream", True, True))


class Clock:
    """on_tokens that stamps each call: (perf_counter, columns visible)."""

    def __init__(self):
        self.t0, self.stamps = time.perf_counter(), []

    def __call__(self, lo, hi, toks, lens):
        self.stamps.append((time.perf_counter(), hi))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--batches", default="1,8")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint"); W = import_module("vlm-fo1_b200.weights")
    assert torch.cuda.is_available(), "stream_bench measures the GPU; there is no CPU path"
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

    def timed(B, x, n, sampled, stream):
        s = E.Sampling([0.7] * B, [0.9] * B, [50] * B, [1000 + b for b in range(B)]) if sampled else None
        clock = Clock() if stream else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if clock is not None:
            clock.t0 = t0
        out = eng.generate(*x, n, stop_ids=[], pad_id=0, early_exit_interval=0, sampling=s, on_tokens=clock)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out, clock

    for no_mega in (False, True):
        if no_mega:
            os.environ["FO1_NO_MEGA"] = "1"
        else:
            os.environ.pop("FO1_NO_MEGA", None)
        path = "per-kernel" if no_mega else "mega"
        for B in [int(b) for b in args.batches.split(",")]:
            x = inputs(B)
            toks = {}
            for name, sampled, stream in CASES:          # warm every shape; streaming must not move a token
                timed(B, x, 1, sampled, stream)
                toks[name] = timed(B, x, T, sampled, stream)[1]["tokens"]
            decode_path = eng.last_decode_path()
            same = dict(greedy=torch.equal(toks["greedy"], toks["greedy_stream"]), sampled=torch.equal(toks["sampled"], toks["sampled_stream"]))
            ms = {name: [] for name, _, _ in CASES}
            first_ms = {name: [] for name, _, s in CASES if s}
            gap_ms = {name: [] for name, _, s in CASES if s}
            calls = {name: [] for name, _, s in CASES if s}
            for _ in range(args.reps):
                for name, sampled, stream in CASES:
                    full, _, clock = timed(B, x, T, sampled, stream)
                    ms[name].append(round(full - timed(B, x, 1, sampled, stream)[0], 2))
                    if stream:
                        st = clock.stamps
                        first_ms[name].append(round((st[0][0] - clock.t0) * 1e3, 2))
                        per_col = [(b[0] - a[0]) * 1e3 / (b[1] - a[1]) for a, b in zip(st, st[1:])]
                        gap_ms[name].append(round(statistics.median(per_col), 3) if per_col else None)
                        calls[name].append(len(st))
            med = {k: statistics.median(v) for k, v in ms.items()}
            r = dict(figure="streamed_decode", path=path, decode_path=decode_path, B=B, new_tokens=T, ms=ms,
                     median_ms={k: round(v, 2) for k, v in med.items()},
                     stream_pct=dict(greedy=round(100 * (med["greedy_stream"] / med["greedy"] - 1), 2),
                                     sampled=round(100 * (med["sampled_stream"] / med["sampled"] - 1), 2)),
                     spread_pct={k: round(100 * (max(v) - min(v)) / statistics.median(v), 2) for k, v in ms.items()},
                     device_step_ms=dict(greedy=round(med["greedy"] / (T - 1), 3), sampled=round(med["sampled"] / (T - 1), 3)),
                     first_on_tokens_ms=first_ms, host_gap_per_column_ms=gap_ms, on_tokens_calls=calls, tokens_unchanged=same)
            print(json.dumps(r), flush=True)
            del x, toks
            torch.cuda.empty_cache()
    os.environ.pop("FO1_NO_MEGA", None)


if __name__ == "__main__":
    main()
