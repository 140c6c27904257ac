"""Prompt-lookup decoding against plain decoding: random-init FO1 language model at full depth (3B widths), 1195-token prompts,
64 new tokens, no stop id.  Cases alternate inside each repetition; the median of 3 is printed.

  plain-mega    plain decoding on the persistent kernel
  plain-pk      plain decoding on the per-kernel path (FO1_NO_MEGA=1)
  lk-prompt-K   lookup, corpus = random prompt ids (only the output's own repeats give drafts)
  lk-own-K      lookup, corpus = the plain run's own output (high acceptance)
  lk-wrong-K    lookup, max_ngram 1, corpus = [t, z, ..., z] (K copies of a token z the output never contains) for every token t of
                the plain output: K wrong drafts every step

Per case: decode time (64-token call minus a 1-token call), loop steps (steps_run: the verify steps the host enqueued), the verify
steps each sequence took part in and the idle ones after its end (steps_run - lookup_steps), tokens emitted per verify step
((lookup_steps + lookup_accepted) / lookup_steps, from the device counters), and the time per loop step.  A second, separate pass
runs one call of each case under torch.profiler with eager launches and no PDL and prints the per-step time of the draft, row,
accept, attention and verify-attention kernels, and the K/V bytes the verify attention reads (every row re-reads its sequence's
cache).
Usage: python scripts/lookup_bench.py [--layers 36] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
KERNELS = ("lookup_drafts_kernel", "lookup_rows_kernel", "lookup_accept_kernel", "decode_attn_kernel<true>", "decode_attn_kernel<false>",
           "decode_attn_combine_kernel", "rope_kv_append_kernel<true>", "rope_kv_append_kernel<false>", "argmax_kernel")


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
    a = ap.parse_args()
    from tests.test_gpu_decode_parity import _model, _mods, make_seq
    E, _, _ = _mods()
    V = 151936
    eng, _ = _model(vocab=V, layers=a.layers, seed=3)
    kv_dim = eng.cfg.llm["num_key_value_heads"] * 128
    print(f"# {card()}; layers {a.layers}, prompt {a.prompt}, new {a.new}", flush=True)
    g = torch.Generator().manual_seed(0)
    for B in (1, 8):
        seqs = [make_seq(a.prompt, None, 50 + b, vocab=V) for b in range(B)]
        emb = torch.cat([s.emb for s in seqs]).cuda()
        pos = torch.cat([s.pos for s in seqs], 1).cuda()
        lens, deltas = [s.L for s in seqs], [s.delta for s in seqs]
        prompt_ids = [torch.randint(0, V, (a.prompt,), generator=g).tolist() for _ in range(B)]

        def call(T, lookup=None, mega=True):
            if mega:
                os.environ.pop("FO1_NO_MEGA", None)
            else:
                os.environ["FO1_NO_MEGA"] = "1"
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = eng.generate(emb, pos, lens, deltas, T, stop_ids=[], pad_id=0, early_exit_interval=8, lookup=lookup)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, out

        own = call(a.new, mega=False)[1]["tokens"].cpu().tolist()
        z = next(t for t in range(V) if all(t not in o for o in own))
        cases = {"plain-mega": dict(mega=True), "plain-pk": dict(mega=False)}
        for K in (4, 10):
            cases[f"lk-prompt-K{K}"] = dict(mega=False, lookup=E.Lookup(K, 2, prompt_ids))
            cases[f"lk-own-K{K}"] = dict(mega=False, lookup=E.Lookup(K, 2, own))
            wrong = [[x for t in sorted(set(o)) for x in [t] + [z] * K] for o in own]
            cases[f"lk-wrong-K{K}"] = dict(mega=False, lookup=E.Lookup(K, 1, wrong))
        res = {n: [] for n in cases}
        for n, kw in cases.items():      # warm-up
            call(a.new, **kw); call(1, **kw)
        for _ in range(a.reps):
            for n, kw in cases.items():
                full, out = call(a.new, **kw)
                pre, _ = call(1, **kw)
                assert out["tokens"].cpu().tolist() == own or kw["mega"], n      # lookup: the plain per-kernel tokens
                steps = out["steps_run"]
                if "lookup_steps" in out:
                    ls, acc = out["lookup_steps"].double(), out["lookup_accepted"].double()
                    seq_steps = int(ls.max())
                    per = float(((ls + acc) / ls.clamp(min=1)).mean())
                    acc_mean = float(acc.mean())
                else:
                    seq_steps, per, acc_mean = steps, 1.0, 0.0
                res[n].append((full - pre, steps, seq_steps, per, acc_mean))
        for n, r in res.items():
            r.sort()
            dec, steps, seq_steps, per, acc_mean = r[len(r) // 2]
            print(json.dumps(dict(B=B, case=n, decode_ms=round(dec * 1e3, 2), loop_steps=steps, verify_steps=seq_steps,
                                  idle_steps=steps - seq_steps, accepted=round(acc_mean, 2), tokens_per_step=round(per, 3),
                                  step_ms=round(dec * 1e3 / max(steps, 1), 3))), flush=True)
        # ---- the profiler pass (separate: eager launches, no PDL, so that every kernel is a trace event of its own) ----
        os.environ["FO1_NO_GRAPH"] = "1"; os.environ["FO1_NO_PDL"] = "1"
        for n, kw in cases.items():
            if kw["mega"]:
                continue
            call(a.new, **kw)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                _, out = call(a.new, **kw)
            steps = max(out["steps_run"], 1)
            t = {k: 0.0 for k in KERNELS}
            for ev in prof.key_averages():
                for k in KERNELS:
                    if k + "(" in ev.key or ev.key.endswith(k):
                        t[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            per_step = {k: round(v / steps / 1e3, 4) for k, v in t.items() if v > 0}     # ms per loop step
            line = dict(B=B, case=n, profiled_steps=steps, kernel_ms_per_step=per_step)
            lk = kw.get("lookup")
            if lk is not None:      # K/V bytes the verify attention reads per step: every row re-reads keys 0 .. its own index
                R, L0 = B * (min(lk.num_tokens, 16) + 1), a.prompt + a.new // 2
                kv_bytes = a.layers * R * L0 * kv_dim * 2 * 2
                line["verify_attn_kv_gb_per_step"] = round(kv_bytes / 1e9, 3)
                line["plain_attn_kv_gb_per_step"] = round(a.layers * B * L0 * kv_dim * 2 * 2 / 1e9, 3)
            print(json.dumps(line), flush=True)
        os.environ.pop("FO1_NO_GRAPH"); os.environ.pop("FO1_NO_PDL")


if __name__ == "__main__":
    main()
