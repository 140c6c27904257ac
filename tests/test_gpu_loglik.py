"""-m gpu: teacher-forced scoring (include/fo1.h, fo1_llm_loglik), every check against the same call with all_logits.

  1. the log-likelihood head: target logits and greedy flags torch.equal what all_logits holds, lse within a per-element bound of the
     fp64 logsumexp of the all_logits row (derived below from where the kernel rounds), at V = 151,936 and V = 20,008 (not a multiple
     of the 128-column tile) and M = 1 .. 2,000 scored rows, with targets at column 0, V - 1, either side of a tile edge and on tied
     maxima; negative controls that the checks must reject;
  2. batch invariance: a sequence's outputs alone, in batches of 8 and 33, and with its prefix shared or not;
  3. the HF surface: forward's logits and loss, its refusals, score_batch, and the round trip with generate."""
from importlib import import_module

import numpy as np
import pytest
import torch

from tests.test_gpu_batch_invariance import _sample, pipe  # noqa: F401 (pipe: fixture)
from tests.test_gpu_sampling import fab  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
TILE = 128              # the head's partial granule (kLoglikTile)


def _llm_engine(V, seed=0, H=256):
    """A one-layer LLM-only engine of vocabulary V with an untied LM head built to exercise the kernel: logits of std ~8, two rows
    far above the rest (so exp without the max subtraction overflows), and two identical hot rows in different tiles (tied maxima)."""
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint")
    cfg = E.EngineConfig()
    cfg.use_vit = cfg.use_davit = False
    cfg.proj_aux_layers = 0
    cfg.llm = dict(cfg.llm, num_hidden_layers=1, hidden_size=H, num_attention_heads=H // 128, num_key_value_heads=1,
                   intermediate_size=512, vocab_size=V, tie_word_embeddings=False)
    sds = CK.random_state_dicts(cfg, "cuda", seed)
    g = torch.Generator(device="cuda").manual_seed(100 + seed)
    w = torch.randn(V, H, device="cuda", generator=g) * 0.5
    hot = torch.randn(H, device="cuda", generator=g) * 4.0
    w[7] = hot; w[129] = hot                        # tied maxima across a tile edge: column 7 is the lowest index
    w[V - 1] = torch.randn(H, device="cuda", generator=g) * 4.0
    sds["llm"]["lm_head.weight"] = w.to(torch.bfloat16)
    return CK.load_engine(cfg, sds), cfg


def _inputs(eng, lens, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = eng.cfg.llm["hidden_size"]
    T = sum(lens)
    emb = (torch.randn(T, H, device="cuda", generator=g)).to(torch.bfloat16)
    pos = torch.cat([torch.arange(L, dtype=torch.int32) for L in lens]).repeat(3, 1).cuda()
    return emb, pos


def _targets(lens, M, V, seed):
    """M scored rows (never a sequence's last), random targets with the edge columns mixed in."""
    rng = np.random.default_rng(seed)
    cand = []
    off = 0
    for L in lens:
        cand += list(range(off, off + L - 1))
        off += L
    rows = np.sort(rng.choice(cand, size=M, replace=False))
    tg = np.full(sum(lens), -100, np.int32)
    tg[rows] = rng.integers(0, V, size=M)
    edges = [0, V - 1, TILE - 1, TILE, 7, 129, (V // TILE) * TILE - 1, (V // TILE) * TILE]
    for i, c in enumerate(edges):
        if i < M:
            tg[rows[(i * 7919) % M]] = min(c, V - 1)
    return tg, rows


def lse_bound(x, chunk=64):
    """lse_bound_rows over chunks of rows (the fp64 temporaries are several [rows, V] matrices)."""
    parts = [lse_bound_rows(x[i:i + chunk]) for i in range(0, x.shape[0], chunk)]
    return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])


def lse_bound_rows(x):
    """Per-row bound on |lse - logsumexp64(x)| for fp32 logit rows x [R, V] (float64 in, exact fp32 values), from the kernel's code:
      tile t (128 columns) of the epilogue: s_t = sum of expf(x - m_t), each thread 32 terms in a chain then 2 butterfly adds;
        expf is within 2 ulp (4u relative), and x - m_t is rounded (relative error |x - m_t| u in the exponential);
      merge: s_t * expf(m_t - M) (1 rounding + 4u + |m_t - M| u), lanes sum ceil(n_t / 32) terms then 5 butterfly adds;
      lse = M + logf(S): logf within 1 ulp (2u relative of log S), the add rounds once (u |lse|).
    Summed as first-order relative errors of positive terms, times a safety factor of 1.5."""
    R, V = x.shape
    n_t = -(-V // TILE)
    xp = torch.full((R, n_t * TILE), float("-inf"), dtype=torch.float64, device=x.device)
    xp[:, :V] = x
    mt = xp.view(R, n_t, TILE).max(-1).values
    M = mt.max(-1).values
    w = torch.exp(xp - M[:, None])                                              # e^(x - M), 0 on the padding
    d_in = (xp - mt.repeat_interleave(TILE, 1)).abs().nan_to_num(0.0)
    d_t = (mt - M[:, None]).abs().repeat_interleave(TILE, 1)
    S = w.sum(-1)
    rel = (w * ((4 + 34 + 1 + 4) * U + (d_in + d_t) * U)).sum(-1) / S + (n_t // 32 + 1 + 5) * U
    lse = M + torch.log(S)
    return 1.5 * (rel * (1 + rel) + 2 * U * torch.log(S).abs() + U * lse.abs()), lse


CASES = [(151936, 1), (151936, 7), (151936, 300), (151936, 2000), (20008, 1), (20008, 7), (20008, 300), (20008, 2000)]


@pytest.mark.parametrize("V,M", CASES)
def test_head_against_all_logits(V, M):
    eng, _ = _llm_engine(V)
    lens = [max(3, M // 4 + 5)] * 5 if M > 7 else [12, 9]
    emb, pos = _inputs(eng, lens, seed=M)
    tg, rows = _targets(lens, M, V, seed=M)
    out = eng.loglik(emb, pos, lens, tg, want_greedy=True, want_all_logits=True, want_lse=True)
    torch.cuda.synchronize()
    rows_t = torch.from_numpy(rows).cuda()
    t = torch.from_numpy(tg[rows].astype(np.int64)).cuda()
    al = out["all_logits"][rows_t]
    # exactness: the epilogue's logits are the fp32 accumulators of the all_logits GEMM, the arg-max is torch's (first maximum)
    assert torch.equal(out["target_logits"], al.gather(1, t[:, None])[:, 0])
    assert torch.equal(out["greedy"][rows_t], (al.argmax(-1) == t).to(torch.int32))
    assert torch.equal(out["logprobs"][rows_t], out["target_logits"] - out["lse"])
    mask = torch.ones_like(out["logprobs"], dtype=torch.bool)
    mask[rows_t] = False
    assert (out["logprobs"][mask] == 0).all() and (out["greedy"][mask] == 0).all()
    # lse against fp64, per element
    x64 = al.double()
    bound, lse64 = lse_bound(x64)
    ratio = ((out["lse"].double() - lse64).abs() / bound).max().item()
    print(f"V={V} M={M}: worst |lse - lse64| / bound = {ratio:.3f}")
    assert ratio <= 1.0
    # sequence sums and counts
    off = np.cumsum([0] + lens)
    lp64 = out["logprobs"].double()
    for b in range(len(lens)):
        acc = 0.0
        for r in range(off[b], off[b + 1]):
            acc += float(lp64[r])
        assert float(out["seq_logprob"][b]) == acc
        assert int(out["seq_count"][b]) == int((tg[off[b]:off[b + 1]] != -100).sum())
    # the edge targets were scored, and the tied hot rows show the lowest-index rule
    if M >= 6:
        assert {0, V - 1, TILE - 1, TILE, 7, 129} <= set(tg[rows].tolist())
    tied = (al.argmax(-1) == 7)
    if tied.any():
        assert torch.equal(al[tied, 7], al[tied, 129])
    # negative controls: a target shifted by one row misses the exact check; lse without the max subtraction misses the bound
    if M > 1:
        t_shift = torch.roll(t, 1)
        assert not torch.equal(out["target_logits"], al.gather(1, t_shift[:, None])[:, 0])
    if M >= 300:
        naive = torch.log(torch.exp(al).sum(-1)).double()      # fp32 exp of the raw logits: overflows where a hot logit passes 88.7
        assert (~((naive - lse64).abs() <= bound)).any()


def test_nothing_scored():
    eng, _ = _llm_engine(20008)
    lens = [5, 3]
    emb, pos = _inputs(eng, lens, 1)
    out = eng.loglik(emb, pos, lens, np.full(8, -100, np.int32), want_greedy=True)
    assert (out["logprobs"] == 0).all() and (out["seq_count"] == 0).all() and (out["seq_logprob"] == 0).all()


# ------------------------------------------------------------------------------------------------------- 2. batch invariance
def test_batch_invariance_alone_8_33():
    V = 20008
    eng, _ = _llm_engine(V, seed=1)
    rng = np.random.default_rng(5)
    lens = [int(x) for x in rng.integers(3, 140, size=33)]
    emb, pos = _inputs(eng, lens, 9)
    tg = np.full(sum(lens), -100, np.int32)
    off = np.cumsum([0] + lens)
    for b, L in enumerate(lens):
        k = off[b] + rng.integers(0, L - 1)
        tg[k:off[b] + L - 1] = rng.integers(0, V, size=off[b] + L - 1 - k)

    def run(idx):
        sel = np.concatenate([np.arange(off[b], off[b + 1]) for b in idx])
        s = torch.from_numpy(sel).cuda()
        return eng.loglik(emb[s], pos[:, s], [lens[b] for b in idx], tg[sel], want_greedy=True)
    full = run(range(33))
    b8 = run(range(8))
    for b in range(8):
        alone = run([b])
        a, r8, r33 = (slice(0, lens[b]), slice(off[b], off[b + 1]), slice(off[b], off[b + 1]))
        for k in ("logprobs", "greedy"):
            assert torch.equal(alone[k][a], b8[k][r8]) and torch.equal(alone[k][a], full[k][r33]), (b, k)
        assert torch.equal(alone["seq_logprob"][0], full["seq_logprob"][b]) and torch.equal(alone["seq_logprob"][0], b8["seq_logprob"][b])


def _answers(base, K, seed=0):
    """K samples about base's image: the same question, then an answer of 2-12 tokens that is scored (labels on the answer only)."""
    P = import_module("vlm-fo1_b200.pipeline")
    rng = np.random.default_rng(seed)
    q = list(base.input_ids) + [151644, 77091, 198]
    samples, labels = [], []
    for k in range(K):
        ans = [int(x) for x in rng.integers(0, 151643, size=int(rng.integers(2, 13)))] + [151645]
        ids = q + ans
        samples.append(P.SampleInputs(ids, base.pixel_values.clone(), base.grid_hw, base.image_aux.clone(), base.boxes.clone()))
        labels.append([-100] * len(q) + ans)
    return samples, labels


def test_shared_prefix_equals_unshared(pipe):  # noqa: F811
    base = _sample(0, 224, 6)
    samples, labels = _answers(base, 8)
    shared = pipe.score(samples, labels, want_greedy=True)
    pipe._share_inputs = False
    try:
        alone = pipe.score(samples, labels, want_greedy=True)
        single = pipe.score(samples[3:4], labels[3:4], want_greedy=True)
    finally:
        pipe._share_inputs = True
    for k in ("logprobs", "greedy", "seq_logprob", "seq_count"):
        assert torch.equal(shared[k], alone[k]), k
    off = np.cumsum([0] + shared["prompt_lens"])
    assert torch.equal(single["logprobs"], shared["logprobs"][off[3]:off[4]])
    assert int(shared["seq_count"].sum()) == sum(sum(1 for x in lab if x != -100) for lab in labels)


# ------------------------------------------------------------------------------------------------------- 3. the HF surface
def _loss_bound(logits, labels):
    """fp64 ForCausalLMLoss over the fp32 logits, and a bound on the engine's loss: each token's log-probability carries the lse
    bound plus one rounding of x - lse, the fp64 sums are exact to 1e-15, and the fp32 loss rounds once."""
    from transformers.loss.loss_utils import ForCausalLMLoss
    V = logits.shape[-1]
    ref = ForCausalLMLoss(logits.double(), labels, V)
    shifted = torch.nn.functional.pad(labels, (0, 1), value=-100)[..., 1:][0]
    keep = (shifted != -100).nonzero().view(-1)
    b, lse64 = lse_bound(logits[0, keep].double())
    tok = logits[0, keep].double().gather(1, shifted[keep][:, None])[:, 0]
    per = b + U * (tok - lse64).abs() * 2
    return ref, (per.sum() / max(len(keep), 1) + U * ref.abs()).item()


def test_forward_matches_generate_and_hf_loss(fab):  # noqa: F811
    _, model, kw = fab
    a = kw(0)
    inputs = a["inputs"]
    P = inputs.shape[1]
    labels = inputs.clone()
    labels[0, : P // 2] = -100
    labels[inputs == -200] = -100
    labels[inputs == -300] = -100
    out = model(input_ids=inputs, images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"],
                bbox_list=a["bbox_list"], labels=labels)
    S = model._score_sample(inputs, a["images"], a["images_aux"], a["image_grid_thws"], a["bbox_list"], labels)
    sp = model.pipeline.score([S[0]], [S[1]], want_all_logits=True)
    # forward's logits are generate's all_logits bit for bit (same prefill, same head GEMM)
    gsam = import_module("vlm-fo1_b200.pipeline")
    gl = _generate_all_logits(model, S[0])
    assert out.logits.shape == (1, gl.shape[0], gl.shape[1]) and out.logits.dtype == torch.float32
    assert torch.equal(out.logits[0], gl)
    assert torch.equal(out.logits[0], sp["all_logits"])
    assert out.past_key_values is None and out.rope_deltas.shape == (1, 1)
    # the loss: HF's ForCausalLMLoss on those logits with the spliced labels, within the fp64-derived bound
    spl = torch.tensor([gsam.splice_labels(S[0].input_ids, S[1], gl.shape[0] - len(S[0].input_ids) + 1)], device=gl.device)
    ref_loss, bound = _loss_bound(gl[None], spl)
    assert abs(float(out.loss) - float(ref_loss)) <= bound, (float(out.loss), float(ref_loss), bound)
    # nothing scored: NaN, as torch gives it; no labels: no loss
    none = model(input_ids=inputs, images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"],
                 bbox_list=a["bbox_list"], labels=torch.full_like(inputs, -100))
    assert torch.isnan(none.loss)
    assert model.forward(input_ids=inputs, images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"],
                         bbox_list=a["bbox_list"]).loss is None


def _generate_all_logits(model, sample):
    """generate(..., all_logits) on the spliced inputs of one sample, through the engine."""
    pipe = model.pipeline
    eng = pipe.eng
    P = import_module("vlm-fo1_b200.pipeline")
    feats, _, region_tokens, _ = pipe.encode([sample])
    plan = P.splice_plan_batch([sample.input_ids], [[sample.grid_hw]], [region_tokens[0].shape[0]], eng.device,
                               merge=eng.cfg.vit["spatial_merge_size"], **pipe.ids)
    emb = eng.build_embeds(plan["kind"], plan["index"], feats, torch.cat(region_tokens, 0))
    out = eng.generate(emb, plan["position_ids"], plan["lens"], plan["rope_delta"], 1, [], 0, want_all_logits=True, early_exit_interval=0)
    return out["all_logits"]


def test_forward_refusals(fab):  # noqa: F811
    _, model, kw = fab
    a = kw(0)
    base = dict(input_ids=a["inputs"], images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"],
                bbox_list=a["bbox_list"])
    for extra in (dict(output_attentions=True), dict(output_hidden_states=True), dict(inputs_embeds=torch.zeros(1)),
                  dict(past_key_values=object()), dict(return_dict=False)):
        with pytest.raises(NotImplementedError):
            model(**base, **extra)


def test_score_batch_equals_forward(fab):  # noqa: F811
    _, model, kw = fab
    batch = [kw(i) for i in range(3)]
    labels = []
    for a in batch:
        lab = a["inputs"].clone()
        lab[0, : lab.shape[1] - 6] = -100
        labels.append(lab)
    res = model.score_batch(batch, labels)
    for a, lab, r in zip(batch, labels, res):
        f = model(input_ids=a["inputs"], images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"],
                  bbox_list=a["bbox_list"], labels=lab)
        _, bound = _loss_bound(f.logits, _spliced(model, a, lab, f.logits.shape[1]))
        assert abs(float(r["loss"]) - float(f.loss)) <= bound
        assert r["logprobs"].shape == r["greedy"].shape and r["logprobs"].numel() == 6      # rows P - 7 .. P - 2 predict the 6 labels


def _spliced(model, a, lab, L):
    P = import_module("vlm-fo1_b200.pipeline")
    ids = a["inputs"][0].tolist()
    return torch.tensor([P.splice_labels(ids, lab[0].tolist(), L - len(ids) + 1)], device="cuda")


def test_round_trip_with_generate(fab):  # noqa: F811
    """Score generate's own greedy output: the greedy flag is 1 wherever the top-1 / top-2 margin is clear, and the first generated
    token's log-probability equals generate(output_logprobs=True)'s within the lse bound."""
    _, model, kw = fab
    a = kw(1)
    (seq, lp), = model.generate_batch([a], output_logprobs=True)
    dec = model.generate(**a, return_dict_in_generate=True, output_logits=True)
    assert torch.equal(dec.sequences, seq)
    P = a["inputs"].shape[1]
    n = seq.shape[1] - P
    labels = seq.clone()
    labels[0, :P] = -100
    f = model(input_ids=seq, images=a["images"], images_aux=a["images_aux"], image_grid_thws=a["image_grid_thws"], bbox_list=a["bbox_list"])
    r, = model.score_batch([dict(a, inputs=seq)], [labels])
    assert r["logprobs"].numel() == n
    L = f.logits.shape[1]
    rows = f.logits[0, L - n - 1:L - 1]                       # the prefill rows that predict the generated tokens
    # sigma: the spread between the decode path's logits and the prefill's on the same positions (different GEMM shapes / paths)
    sigma = float(torch.cat([(rows[t] - dec.logits[t][0]) for t in range(n)]).std())
    top2 = rows.topk(2, -1).values
    clear = (top2[:, 0] - top2[:, 1]) > 6 * sigma
    assert clear.any()
    assert (r["greedy"][clear] == 1).all()
    # column 0 comes from the prefill's last row on both sides: generate's log-probability (fixed-point sum over the vocabulary, see
    # fo1_score_desc) and the head's agree within the lse bound plus generate's own rounding of the log-sum
    # (generate's row 0 is the prefill's last-row head, summed in another order: the two rows differ by d0 at most per logit)
    d0 = float((rows[0] - dec.logits[0][0]).abs().max())
    b, _ = lse_bound(rows[:1].double())
    tol = float(b[0]) + 2 * d0 + 8 * U * (abs(float(lp[0, 0])) + float(rows[0].abs().max()))
    assert abs(float(r["logprobs"][0]) - float(lp[0, 0])) <= tol, (float(r["logprobs"][0]), float(lp[0, 0]), tol)
