"""Old against new for the decoder: a seeded set of Engine.generate calls whose every output is saved, so that two builds of the
engine (before and after a change to the decoder) can be required to agree bit for bit.

The set: greedy, sampled, scored and streamed calls at B = 1, 8, 17 and 33, on both decode paths (the default, and the per-kernel
path with FO1_NO_MEGA=1); a shared-prefix batch (one group and loners); beam search with N = 4; prompt lookup with K = 4; logits
processors (sets that differ per sequence, some sequences without one) on greedy, sampled, scored and streamed calls at B = 8 and 17
on both decode paths, and with the shared prefix.  Every call asks for the prefill logits.  Random-init decoder (Qwen2.5-3B widths, 4 layers, 20000-token vocabulary) on the GPU.

    python scripts/ab_generate.py --out run.pt             # run the set, save every output
    python scripts/ab_generate.py --compare old.pt new.pt  # torch.equal on every output of every call
"""
import argparse
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

VOCAB, T = 20000, 12


class Streamed:
    """on_tokens recorder: the streamed columns assembled into [B, T], and the last lens."""

    def __init__(self, B):
        self.tokens = torch.full((B, T), -1, dtype=torch.int32)
        self.lens = None

    def __call__(self, lo, hi, tokens, lens):
        self.tokens[:, lo:hi] = torch.from_numpy(tokens.copy())
        self.lens = torch.from_numpy(lens.copy())


def _batch(make_seq, B, seed):
    seqs = [make_seq(30 + 9 * (b % 7), None, seed + b, vocab=VOCAB) for b in range(B)]
    return (torch.cat([s.emb for s in seqs]).cuda(), torch.cat([s.pos for s in seqs], 1).cuda(), [s.L for s in seqs],
            [s.delta for s in seqs])


def _processors(E, B, seed):
    """Processor sets for B sequences, cycling through four: a bias strong enough that the n-gram ban has to act, lists and min lengths
    that hold back the stop ids, and None (a row that is never edited).  The prompts start with an image placeholder."""
    S = E.ProcessorSet
    sets = [S(no_repeat_ngram_size=2, sequence_bias=(((5,), 30.0),), min_new_tokens=3, eos_token_ids=(7, 11)),
            None,
            S(sequence_bias=(((9,), 2.5), ((9, 5), -1.0)), bad_words_ids=((13,), (4, 6)), suppress_tokens=(17,), begin_suppress_tokens=(19,)),
            S(min_length=40, eos_token_ids=(7,), no_repeat_ngram_size=3)]
    g = torch.Generator().manual_seed(seed)
    prompts = [[-200] + torch.randint(0, VOCAB, (10 + b,), generator=g).tolist() for b in range(B)]
    return E.Processors([sets[b % len(sets)] for b in range(B)], prompts)


def run(out_path):
    from tests.test_gpu_decode_parity import _model, _mods, make_seq
    E, _, _ = _mods()
    eng, _ = _model(vocab=VOCAB, layers=4, seed=5)
    results = {}

    def call(name, no_mega, *args, stream=False, **kw):
        if no_mega:
            os.environ["FO1_NO_MEGA"] = "1"
        else:
            os.environ.pop("FO1_NO_MEGA", None)
        rec = Streamed(len(args[2])) if stream else None
        out = eng.generate(*args, T, stop_ids=kw.pop("stop_ids", [7, 11]), pad_id=3, early_exit_interval=4, want_prefill_logits=True,
                           on_tokens=rec, **kw)
        torch.cuda.synchronize()
        res = {k: v.cpu() for k, v in out.items() if isinstance(v, torch.Tensor)}
        if rec is not None:
            res["streamed_tokens"], res["streamed_lens"] = rec.tokens, rec.lens
        res["decode_path"] = torch.tensor([eng.last_decode_path()])
        results[name] = res
        print(name, sorted(res), flush=True)
        return out

    for B in (1, 8, 17, 33):
        x = _batch(make_seq, B, 100 * B)
        samp = E.Sampling([0.8] * B, [0.9] * B, [40] * B, [1000 + b for b in range(B)])
        for no_mega in (False, True):
            p = "pk" if no_mega else "default"
            call(f"greedy/B{B}/{p}", no_mega, *x)
            call(f"sampled/B{B}/{p}", no_mega, *x, sampling=samp)
            call(f"scored/B{B}/{p}", no_mega, *x, sampling=samp, want_logprobs=True, want_scores=True, want_logits=True)
            call(f"scored-greedy/B{B}/{p}", no_mega, *x, want_logprobs=True, want_scores=True, want_logits=True)
            call(f"streamed/B{B}/{p}", no_mega, *x, sampling=samp, stream=True)
        if B <= 8:
            call(f"all-logits/B{B}", False, *x, want_all_logits=True)

    # shared prefix: sequences 0..5 share a 40-row prefix, 6 and 7 stand alone
    Bp, P = 8, 40
    s0 = make_seq(P + 12, None, 7, vocab=VOCAB)
    own = [make_seq(P + 12 + b, None, 300 + b, vocab=VOCAB) for b in range(Bp)]
    groups = [0] * 6 + [-1, -1]
    emb = torch.cat([o.emb[P:] if g == 0 else o.emb for o, g in zip(own, groups)]).cuda()
    pos = torch.cat([o.pos[:, P:] if g == 0 else o.pos for o, g in zip(own, groups)], 1).cuda()
    lens = [o.L for o in own]
    prefix = E.Prefix(lens=[P], embeds=s0.emb[:P].cuda(), position_ids=s0.pos[:, :P].cuda(), seq_group=groups)
    xp = (emb, pos, lens, [o.delta for o in own])
    sampp = E.Sampling([0.8] * Bp, [0.9] * Bp, [40] * Bp, [2000 + b for b in range(Bp)])
    for no_mega in (False, True):
        p = "pk" if no_mega else "default"
        call(f"prefix-greedy/{p}", no_mega, *xp, prefix=prefix)
        call(f"prefix-scored/{p}", no_mega, *xp, prefix=prefix, sampling=sampp, want_logprobs=True, want_scores=True, want_logits=True)
        call(f"prefix-streamed/{p}", no_mega, *xp, prefix=prefix, stream=True)

    # logits processors: greedy, sampled, scored and streamed, on both decode paths, and with the shared prefix
    for B in (8, 17):
        x = _batch(make_seq, B, 9000 + B)
        procs = _processors(E, B, 40 + B)
        samp = E.Sampling([0.8] * B, [0.9] * B, [40] * B, [4000 + b for b in range(B)])
        for no_mega in (False, True):
            p = "pk" if no_mega else "default"
            call(f"processed-greedy/B{B}/{p}", no_mega, *x, processors=procs)
            call(f"processed-sampled/B{B}/{p}", no_mega, *x, sampling=samp, processors=procs)
            call(f"processed-scored/B{B}/{p}", no_mega, *x, sampling=samp, want_logprobs=True, want_scores=True, want_logits=True,
                 processors=procs)
            call(f"processed-scored-greedy/B{B}/{p}", no_mega, *x, want_logprobs=True, want_scores=True, want_logits=True, processors=procs)
            call(f"processed-streamed/B{B}/{p}", no_mega, *x, sampling=samp, stream=True, processors=procs)
    procs_p = _processors(E, Bp, 60)
    for no_mega in (False, True):
        p = "pk" if no_mega else "default"
        call(f"prefix-processed/{p}", no_mega, *xp, prefix=prefix, sampling=sampp, want_logprobs=True, want_scores=True, want_logits=True,
             processors=procs_p)

    # beam search, N = 4
    for B in (1, 8):
        x = _batch(make_seq, B, 5000 + B)
        beams = E.Beams(4, 12, 1.0, False, 2)      # n_keep: HF's max(2, 1 + 2 stop ids) * N
        call(f"beam/B{B}", False, *x, beams=beams, want_logprobs=True, want_scores=True, want_logits=True)

    # prompt lookup, K = 4: corpus = the plain greedy output (accepting drafts) and random ids (mostly rejected)
    g = torch.Generator().manual_seed(9)
    for B in (1, 8, 17):
        x = _batch(make_seq, B, 7000 + B)
        plain = call(f"lookup-plain/B{B}", True, *x, stop_ids=[])
        own_corpus = plain["tokens"].cpu().tolist()
        rand_corpus = [torch.randint(0, VOCAB, (50,), generator=g).tolist() for _ in range(B)]
        samp = E.Sampling([0.8] * B, [0.9] * B, [40] * B, [3000 + b for b in range(B)])
        call(f"lookup-own/B{B}", True, *x, stop_ids=[], lookup=E.Lookup(4, 2, own_corpus))
        call(f"lookup-rand/B{B}", True, *x, lookup=E.Lookup(4, 2, rand_corpus))
        call(f"lookup-sampled/B{B}", True, *x, sampling=samp, lookup=E.Lookup(4, 2, own_corpus))
        call(f"lookup-scored/B{B}", True, *x, sampling=samp, want_logprobs=True, want_scores=True, want_logits=True,
             lookup=E.Lookup(4, 2, own_corpus))
    call("lookup-prefix", True, *xp, prefix=prefix, lookup=E.Lookup(4, 2, [[1, 2, 3]] * Bp))
    torch.save(results, out_path)
    print(f"{len(results)} calls -> {out_path}")


def compare(a_path, b_path):
    a, b = torch.load(a_path), torch.load(b_path)
    bad = []
    if sorted(a) != sorted(b):
        bad.append(f"call sets differ: {sorted(set(a) ^ set(b))}")
    n = 0
    for name in sorted(set(a) & set(b)):
        if sorted(a[name]) != sorted(b[name]):
            bad.append(f"{name}: outputs differ: {sorted(set(a[name]) ^ set(b[name]))}")
        for k in sorted(set(a[name]) & set(b[name])):
            n += 1
            if not torch.equal(a[name][k], b[name][k]):
                bad.append(f"{name}: {k}")
    print(f"{len(set(a) & set(b))} calls, {n} outputs compared, {len(bad)} differ")
    for line in bad:
        print("  DIFF", line)
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    run(args.out)
