"""Cost of per-token scoring (log-probabilities, HF output_scores / output_logits) on top of greedy and sampled decoding, measured
on the GPU.

At the c3 shape (1195-token prompts, 64 new tokens) for B = 1, 8, 32, through the persistent decode kernel (default) and the
per-kernel graph (FO1_NO_MEGA=1), five cases on the same seeded inputs, alternating inside each repetition:
  greedy; greedy + logprobs; greedy + scores + logits; sampled (T 0.7, top-p 0.9, top-k 50); sampled + logprobs.
Decode time = time of a 64-token generate minus time of a 1-token generate (the prefill and the first token).  Random-init
Qwen2.5-3B decoder (36 layers, real widths).  Prints the card name and power limit, then one JSON line per (path, B).

    python scripts/scores_bench.py [--reps 3] [--layers 36] [--batches 1,8,32]
"""
import argparse
import json
import os
import sys
import time
from importlib import import_module

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from scripts.sampling_bench import card  # noqa: E402

CASES = (("greedy", False, {}), ("greedy_logprobs", False, dict(want_logprobs=True)),
         ("greedy_scores_logits", False, dict(want_scores=True, want_logits=True)), ("sampled", True, {}),
         ("sampled_logprobs", True, dict(want_logprobs=True)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--batches", default="1,8,32")
    args = ap.parse_args()
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint"); W = import_module("vlm-fo1_b200.weights")
    assert torch.cuda.is_available(), "scores_bench measures the GPU; there is no CPU path"
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

    def timed(B, x, n, sampled, kw):
        s = E.Sampling([0.7] * B, [0.9] * B, [50] * B, [1000 + b for b in range(B)]) if sampled else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = eng.generate(*x, n, stop_ids=[], pad_id=0, early_exit_interval=0, sampling=s, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    def decode_ms(B, x, sampled, kw):
        return timed(B, x, T, sampled, kw)[0] - timed(B, x, 1, sampled, kw)[0]

    for no_mega in (False, True):
        if no_mega:
            os.environ["FO1_NO_MEGA"] = "1"
        else:
            os.environ.pop("FO1_NO_MEGA", None)
        path = "per-kernel" if no_mega else "mega"
        for B in [int(b) for b in args.batches.split(",")]:
            x = inputs(B)
            toks = {}
            for name, sampled, kw in CASES:          # warm every shape; scoring must not move a token
                timed(B, x, 1, sampled, kw)
                toks[name] = timed(B, x, T, sampled, kw)[1]["tokens"]
            decode_path = eng.last_decode_path()     # of a 64-token call (a 1-token call never enters the decode loop)
            same = dict(greedy=all(torch.equal(toks["greedy"], toks[n]) for n in ("greedy_logprobs", "greedy_scores_logits")),
                        sampled=torch.equal(toks["sampled"], toks["sampled_logprobs"]))
            ms = {name: [] for name, _, _ in CASES}
            for _ in range(args.reps):
                for name, sampled, kw in CASES:
                    ms[name].append(round(decode_ms(B, x, sampled, kw), 2))
            best = {k: min(v) for k, v in ms.items()}
            r = dict(figure="scored_decode", path=path, decode_path=decode_path, B=B, new_tokens=T, ms=ms,
                     logprobs_pct=dict(greedy=round(100 * (best["greedy_logprobs"] / best["greedy"] - 1), 2),
                                       sampled=round(100 * (best["sampled_logprobs"] / best["sampled"] - 1), 2)),
                     scores_logits_pct=round(100 * (best["greedy_scores_logits"] / best["greedy"] - 1), 2), tokens_unchanged=same)
            print(json.dumps(r), flush=True)
            del x, toks
            torch.cuda.empty_cache()
    os.environ.pop("FO1_NO_MEGA", None)


if __name__ == "__main__":
    main()
