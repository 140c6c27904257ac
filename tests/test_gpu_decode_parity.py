"""-m gpu: the per-step fp32 logits of BOTH decode paths (the persistent kernel, csrc/decode_mega.cu, and the per-kernel graph)
against the CPU decoder (oracle/llm.py), teacher-forced on each sequence's own tokens, on weights whose RMSNorm gains are not 1
and whose q / k / v biases are not 0.

Why those weights: the persistent kernel reads decode copies with the norm gains folded in (qkv_dec = W_qkv diag(g1), gu_dec,
head_dec = lm_head diag(g_final); weights.py::prepare_llm) and adds qkv_b itself.  With checkpoint.random_llm's unit gains and
zero biases a wrong fold, a read of the unfolded copy or a dropped bias add all compute the same numbers, so this file sets the
gains to 1 + 0.2 N(0, 1) and the biases to 0.2 N(0, 1) (bf16-rounded; the recipe of oracle/gen_golden.py's llm_small fixture).

Prompts carry M-RoPE positions from the splice plan: each sequence has its own image grid (or none), hence its own, negative,
rope delta, and its own seeded embeddings.  Every generate call runs scored (DEC_SCORED: the logits row of every column) and
once more unscored; tokens and lengths must be bit-equal, which ties the greedy instantiation to the rows checked here.

Checks for every sequence and every column t < out_lens (column 0 is the prefill's row), with the oracle run twice -- bf16
storage points (precision.act_bf16) and plain fp32:
  (A) rerr(engine, fp32) <= 1.25 x rerr(bf16 oracle, fp32) + 5e-4 over the sequence's stacked rows (test_gpu_parity_stages);
  (B) per row nerr(engine, bf16 oracle) <= 1e-3 + k x 2^-8, k = 3 on the per-kernel path and 4 on the persistent kernel
      (TOL_B below says why);
  argmax: the engine's token is the oracle's arg-max wherever the oracle's top-1 / top-2 margin exceeds 6 sigma of the measured
      logit error;
  path: fo1_last_decode_path() is the path the case is meant to run.
Negative controls (CPU only): the fp32 oracle with every gain reset to 1, with the biases zeroed, and with the decode position one
too far must each fall outside (A) or (B) against the same engine rows -- the bound can see the defects this file is about.
Measured values of every case are written as parity_decode_<case>.json (test_gpu_parity_stages._record)."""
from dataclasses import dataclass

import pytest
import torch

from tests.golden_io import nerr, rerr
from tests.test_gpu_parity_stages import _record

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -8
# (B), k single-ulp flips at the largest logit.  The per-kernel path stores bf16 where the oracle does: k = 3, as the prompt logits
# of test_llm_layers_real_width_c4_prompt.  The persistent kernel rounds elsewhere: its folded weights W diag(g) are bf16 (one
# rounding the reference does not have, in qkv, gate / up and the head) and it never stores the normed activations (two roundings
# the reference has), so its rounding errors are less correlated with the bf16 oracle's: k = 4.  Measured: oracle/llm.py's decoder
# restated with exactly those storage points sits 0.79 .. 1.07 x tol(3) from the bf16 oracle on short prompts at an (A) ratio of
# 0.67 .. 0.71; the kernel sits up to 1.19 x tol(3) from it (the worst of 640 rows, H100) at an (A) ratio of 0.68 .. 0.73.
TOL_B = {0: 1e-3 + 3 * ULP, 1: 1e-3 + 4 * ULP}     # by decode path (fo1_last_decode_path)
T_COLS = 20                    # output columns: short caches cross 16-key tile boundaries while decoding
CTRL_SEQS = 3                  # sequences per case the negative controls are computed for (the first, a middle and the last)


def _mods():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine"), import_module("vlm-fo1_b200.checkpoint"), import_module("vlm-fo1_b200.weights")


def randomise_gains_and_biases(sd, seed):
    """random_llm's state dict with every RMSNorm gain set to 1 + 0.2 N(0, 1) and every q / k / v bias to 0.2 N(0, 1), bf16."""
    g = torch.Generator().manual_seed(seed)
    for k in sorted(sd):
        if k.endswith("layernorm.weight") or k == "norm.weight":
            sd[k] = (1.0 + 0.2 * torch.randn(sd[k].shape, generator=g)).to(sd[k].device, torch.bfloat16)
        elif k.endswith(("q_proj.bias", "k_proj.bias", "v_proj.bias")):
            sd[k] = (0.2 * torch.randn(sd[k].shape, generator=g)).to(sd[k].device, torch.bfloat16)
    return sd


def _model(H=2048, heads=16, kv_heads=2, inter=11008, vocab=20000, layers=2, seed=31):
    E, CK, W = _mods()
    cfg = E.EngineConfig()
    cfg.use_vit = cfg.use_davit = False
    cfg.proj_aux_layers = 0
    cfg.llm = dict(cfg.llm, hidden_size=H, num_attention_heads=heads, num_key_value_heads=kv_heads, intermediate_size=inter,
                   vocab_size=vocab, num_hidden_layers=layers)
    sd = randomise_gains_and_biases(CK.random_llm(cfg.llm, torch.Generator(device="cuda").manual_seed(seed), "cuda"), seed + 1)
    eng = E.Engine(cfg)
    eng.set_weights(W.prepare_llm(sd, cfg.llm, eng.device))
    eng.finalize()
    return eng, Oracle({k: v.float().cpu() for k, v in sd.items()}, cfg.llm)


# ------------------------------------------------------------------------------------------------------------ prompts
@dataclass
class Seq:
    key: tuple
    emb: torch.Tensor          # bf16 [L, H] (CPU)
    pos: torch.Tensor          # int32 [3, L]
    delta: int

    @property
    def L(self):
        return self.emb.shape[0]


def make_seq(L, grid, seed, H=2048, vocab=20000):
    """A spliced prompt of L rows: text, then (grid given) <vision_start> + the image's gh*gw/4 tokens, then text; positions and
    rope delta from the engine's splice plan, embeddings N(0, 0.05^2) seeded by `seed`."""
    E, _, _ = _mods()
    g = torch.Generator().manual_seed(seed)
    text = lambda n: torch.randint(0, vocab - 16, (n,), generator=g).tolist()
    vstart, img_tok = vocab - 2, vocab - 1
    if grid is None:
        ids = text(L)
    else:
        n_img = grid[0] * grid[1] // 4
        assert L >= n_img + 1, (L, grid)
        pre = (L - n_img - 1) // 3
        ids = text(pre) + [vstart, -200] + text(L - n_img - 1 - pre)
    plan = E.splice_plan(ids, [grid] if grid else [], 0, image_token_id=img_tok, vision_start_token_id=vstart)
    assert len(plan["kind"]) == L
    emb = (torch.randn(L, H, generator=g) * 0.05).bfloat16()
    return Seq((L, grid, seed), emb, torch.from_numpy(plan["position_ids"]).to(torch.int32), int(plan["rope_delta"]))


# ------------------------------------------------------------------------------------------------------------ oracle
class Oracle:
    """oracle.llm.Decoder teacher-forced on the engine's tokens.  Each (model variant, sequence, precision)'s prompt pass -- the
    K/V lists and the last position's logits -- is computed once and kept, so a sequence reused by another case only re-runs
    its decode steps."""

    def __init__(self, sd, cfg):
        self.cfg = cfg
        self.sds = {"base": sd}
        self.cache = {}

    def _sd(self, variant):
        if variant not in self.sds:
            base = self.sds["base"]
            if variant == "unit_gains":
                self.sds[variant] = {k: (torch.ones_like(v) if k.endswith("layernorm.weight") or k == "norm.weight" else v) for k, v in base.items()}
            elif variant == "zero_bias":
                self.sds[variant] = {k: (torch.zeros_like(v) if k.endswith("_proj.bias") else v) for k, v in base.items()}
            else:
                raise KeyError(variant)
        return self.sds[variant]

    def rows(self, seq, toks, bf16, variant="base", pos_shift=0):
        """Logits [1 + len(toks), V]: the prompt's last position, then one decode step per forced token (the token of column s at
        position L + s + delta + pos_shift)."""
        from oracle import llm as OL, precision
        sd = self._sd(variant)
        key = (variant, seq.key, bool(bf16))
        with precision.act_bf16(bf16), torch.no_grad():
            if key not in self.cache:
                dec = OL.Decoder(sd, self.cfg)
                h = dec.forward(seq.emb.float(), seq.pos.long())
                self.cache[key] = (list(dec.kv), dec.logits(h[-1:])[0])
            kv, first = self.cache[key]
            dec = OL.Decoder(sd, self.cfg)
            dec.kv = list(kv)
            emb = sd["embed_tokens.weight"]
            out = [first]
            for s, tok in enumerate(toks):
                p = seq.L + s + seq.delta + pos_shift
                h = dec.forward(emb[int(tok)][None, :], torch.full((3, 1), p, dtype=torch.long))
                out.append(dec.logits(h)[0])
        return torch.stack(out)


# ------------------------------------------------------------------------------------------------------------ engine + checks
def run_engine(eng, seqs, T, stop_ids=(), path=None):
    """Scored and unscored generate over the packed batch -> (tokens [B, T], lens [B], logits [T, B, V]) on the CPU."""
    emb = torch.cat([s.emb for s in seqs]).cuda()
    pos = torch.cat([s.pos for s in seqs], dim=1).contiguous()
    lens, deltas = [s.L for s in seqs], [s.delta for s in seqs]
    kw = dict(stop_ids=list(stop_ids), pad_id=0, early_exit_interval=4)
    out = eng.generate(emb, pos, lens, deltas, T, want_logits=True, want_prefill_logits=True, **kw)
    torch.cuda.synchronize()
    if path is not None:
        assert eng.last_decode_path() == path
    plain = eng.generate(emb, pos, lens, deltas, T, **kw)
    torch.cuda.synchronize()
    if path is not None:
        assert eng.last_decode_path() == path
    assert torch.equal(out["tokens"], plain["tokens"]) and torch.equal(out["lens"], plain["lens"])
    assert torch.equal(out["logits"][0], out["prefill_logits"])
    return out["tokens"].cpu(), out["lens"].cpu(), out["logits"].cpu()


def a_bound(ref_bf16, ref_f32):
    return 1.25 * rerr(ref_bf16, ref_f32) + 5e-4


def check_case(name, orc, seqs, toks, lens, logits, path, controls=True):
    """(A), (B) and the arg-max check for every sequence; the negative controls on CTRL_SEQS of them.  Records, then asserts."""
    B = len(seqs)
    tol_b = TOL_B[path]
    per_seq, ctrl = [], {"unit_gains": [], "zero_bias": [], "pos_plus_1": []}
    failures = []
    ctrl_idx = sorted({0, B // 2, B - 1})[:CTRL_SEQS] if controls else []
    compared = 0
    for b, seq in enumerate(seqs):
        n = int(lens[b])
        forced = toks[b, :n - 1].tolist()
        got = logits[:n, b]
        ref = orc.rows(seq, forced, True)
        f32 = orc.rows(seq, forced, False)
        ra = rerr(got, f32) / a_bound(ref, f32)
        rb = max(nerr(got[t], ref[t]) for t in range(n)) / tol_b
        sigma = float((got - ref).pow(2).mean().sqrt())
        top2 = ref.topk(2, dim=-1)
        dec = [t for t in range(n) if float(top2.values[t, 0] - top2.values[t, 1]) > 6.0 * sigma]
        bad = [t for t in dec if int(toks[b, t]) != int(top2.indices[t, 0])]
        compared += len(dec)
        per_seq.append(dict(b=b, L=seq.L, delta=seq.delta, cols=n, A_ratio=ra, B_ratio=rb, sigma=sigma, decidable=len(dec),
                            argmax_mismatch=bad))
        if ra > 1.0 or rb > 1.0 or bad:
            failures.append(per_seq[-1])
        if b in ctrl_idx:
            den = a_bound(ref, f32)
            for cname, kw in (("unit_gains", dict(variant="unit_gains")), ("zero_bias", dict(variant="zero_bias")),
                              ("pos_plus_1", dict(pos_shift=1))):
                c = orc.rows(seq, forced, False, **kw)
                # the control stands in for the reference: (A) with it as the fp32 yardstick, (B) with it in place of the bf16 oracle
                ca = rerr(got, c) / den
                cb = max(nerr(got[t], c[t]) for t in range(n)) / tol_b
                ctrl[cname].append(dict(b=b, A_ratio=ca, B_ratio=cb, miss=max(ca, cb)))
    rec = dict(case=name, B=B, path=path, tol_B=tol_b, columns=int(toks.shape[1]), worst_A_ratio=max(p["A_ratio"] for p in per_seq),
               worst_B_ratio=max(p["B_ratio"] for p in per_seq), decidable_argmax=compared,
               control_min_miss={k: min(x["miss"] for x in v) for k, v in ctrl.items() if v}, controls=ctrl, per_seq=per_seq)
    _record(f"decode_{name}", rec)
    assert not failures, (name, failures)
    for cname, v in ctrl.items():
        for x in v:
            assert x["miss"] > 1.0, (name, cname, x)
    return rec


# ------------------------------------------------------------------------------------------------------------ cases
@pytest.fixture(scope="module")
def model():
    return _model()


def _pool():
    """The sequences of cases a-g (3B widths, vocabulary 20000).  Grids: 46x46 (529 image tokens) down to 4x4; None = text only."""
    grids = [None, (20, 32), (8, 12), None, (12, 12), (6, 6), None, (14, 14), (4, 4), (10, 8), None, (16, 6), (8, 8), None, (6, 10), (2, 4)]
    long = make_seq(3000, (46, 46), 1000)
    b_lens = [1, 15, 16, 17, 127, 128, 129, 255, 300]
    b_grids = [None, None, (4, 4), (6, 6), (8, 12), (12, 12), None, (20, 32), (14, 14)]
    b = [make_seq(L, gr, 1100 + i) for i, (L, gr) in enumerate(zip(b_lens, b_grids))]
    c_lens = [37 + 23 * i for i in range(16)]                                  # 37 .. 382
    fits = lambda gr, L: gr if gr is not None and gr[0] * gr[1] // 4 < L else None
    c = [make_seq(L, fits(grids[i], L), 1200 + i) for i, L in enumerate(c_lens)]
    d_extra = make_seq(211, (10, 14), 1300)
    e_lens = [1 + (29 * i) % 97 for i in range(32)]                            # short, ragged: 1 .. 97
    e = [make_seq(L, fits([None, (4, 6), (2, 4)][i % 3], L), 1400 + i) for i, L in enumerate(e_lens)]
    return dict(a=[long], b=b, c=c, d=c + [d_extra], e=e, f=e + [c[0]], g=b)


# order: B grows 9 -> 33 with the cache capacity small, then B = 1 with the largest cache, then B = 9 again with a small one --
# stale arena, K/V or attention-counter state from the previous call would show as a mismatch
CASES = [("b", 1), ("c", 1), ("d", 1), ("e", 1), ("f", 0), ("a", 1), ("g", 0)]


@pytest.fixture(scope="module")
def pool():
    return _pool()


@pytest.mark.parametrize("case,path", CASES, ids=[c for c, _ in CASES])
def test_decode_step_logits_match_oracle(model, pool, case, path, monkeypatch):
    eng, orc = model
    monkeypatch.setenv("FO1_MEGA_MAX_B", "32")
    if case == "g":
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    seqs = pool[case]
    stop = ()
    if case == "e":
        # up to three stop ids from the sequences' own tokens, chosen so that at most half of the batch ends early and the
        # rest runs on (its rows after the others' stop are checked like any other)
        free, _, _ = run_engine(eng, seqs, T_COLS, path=path)
        rows = [free[i, :T_COLS - 1].tolist() for i in range(len(seqs))]
        ended, stop = set(), []
        for tok in free[:, 4:8].flatten().tolist():
            hit = {i for i, r in enumerate(rows) if tok in r}
            if tok not in stop and len(ended | hit) <= len(seqs) // 2:
                stop.append(tok); ended |= hit
            if len(stop) == 3:
                break
        assert ended, free
    toks, lens, logits = run_engine(eng, seqs, T_COLS, stop, path=path)
    if case == "e":
        assert int(lens.min()) < T_COLS and int(lens.max()) == T_COLS, lens.tolist()
    else:
        assert lens.tolist() == [T_COLS] * len(seqs)
    check_case(case, orc, seqs, toks, lens, logits, path)


def test_decode_step_logits_real_vocabulary():
    """h: the LM head at its real width (vocabulary 151936), B = 2 (8 key splits per (sequence, kv head)), 8 columns."""
    eng, orc = _model(vocab=151936, seed=41)
    seqs = [make_seq(700, (46, 46), 2000, vocab=151936), make_seq(90, None, 2001, vocab=151936)]
    toks, lens, logits = run_engine(eng, seqs, 8, path=1)
    check_case("h", orc, seqs, toks, lens, logits, 1)


# ------------------------------------------------------------------------------------------------------------ decode-path choice
@pytest.mark.parametrize("shape", [
    pytest.param(dict(H=256, heads=2, kv_heads=1, inter=384, vocab=1024), id="hidden256_inter384_vocab1024"),
    pytest.param(dict(vocab=20008), id="3b_widths_vocab20008"),
])
def test_unsupported_shape_decodes_on_per_kernel_path(shape):
    """A model shape the persistent kernel does not run (hidden / 64 < 8 warps; a vocabulary that is not a multiple of 16) still
    gets its decode copies from prepare_llm; generate must take the per-kernel path, with logits that pass the same checks."""
    eng, orc = _model(seed=51, **shape)
    H, V = shape.get("H", 2048), shape["vocab"]
    seqs = [make_seq(L, gr, 3000 + i, H=H, vocab=V) for i, (L, gr) in enumerate([(150, (8, 12)), (33, None), (64, (4, 4))])]
    toks, lens, logits = run_engine(eng, seqs, 12, path=0)
    check_case(f"shape_{shape.get('H', 2048)}_{V}", orc, seqs, toks, lens, logits, 0, controls=False)
