"""-m gpu: a sample's numbers do not depend on its batch (DESIGN.md section 2), bit for bit.

  A. every GEMM tile width gives the same bits per output element (the engine picks the width from the tile count, so an image
     alone and the same image in a batch run different widths);
  B. the two row-norm kernels against a float64 restatement, at every register-tile instantiation (the engine names one kernel per
     call site, tested here directly);
  C. every tower stage of a sample alone == the same sample inside same-size, mixed-size and (afterwards) no batch;
  D. prefill logits, every column's fp32 logits row, tokens and lengths of a sequence alone == the same sequence inside a batch, on
     both decode paths.  The one exception is pinned, not described: the split count of the decode attention depends on the batch
     (persistent kernel min(8, SMs / (B * kv_heads)), per-kernel path min(8, 2 * SMs / (B * kv_heads))); where it differs from a
     lone sequence's only the prefill logits and column 0 must agree.

One engine at the released widths (ViT 1280 with windowed and full blocks, DaViT 256..2048, FPN 512, HFRE D = 5888, 2-layer
projector, two Qwen2.5-3B decoder layers, vocabulary 151936) at reduced depth, so every tile-width and kernel choice is the
production one.  Every comparison is torch.equal."""
from importlib import import_module

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = (32, 64, 128, 192, 256)


def _ops():
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.ops")


def _first_diff(a, b):
    idx = tuple(int(i) for i in (a != b).nonzero()[0])
    return f"first differing element {idx}: {float(a[idx])} vs {float(b[idx])}, {int((a != b).sum())} of {a.numel()} differ"


# --------------------------------------------------------------------------------------------------------- A. GEMM tile width
# the towers' and the prefill's contractions: patch embed (K = 1176), ViT (1280, N = 3424 ragged), LLM / projector (2048, 5888,
# 11008), SimpleFPN 3x3 as a GEMM (9 * 512), a ragged N = 1000; M ragged, below and above one 128-row tile
GEMM_SHAPES = [(200, 1280, 1176), (64, 3424, 1280), (16, 3424, 1280), (300, 1000, 2048), (33, 2560, 2048), (77, 2048, 5888),
               (130, 2048, 11008), (256, 512, 9 * 512)]
EPILOGUES = ["none", "bias_bf16", "bias_f32", "gelu", "silu", "gated", "residual"]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_tile_width_bit_identical(M, N, K):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    Ng = 2 * ((N + 31) // 32 * 32)                           # gated: [32 gate | 32 up] row blocks, N / 2 outputs
    w = (torch.randn(max(N, Ng), K, device="cuda", generator=g) * K ** -0.5).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g) * 0.5
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    ref32 = a.float() @ w[:N].float().t()
    for epi in EPILOGUES:
        for dt in (torch.bfloat16, torch.float32):
            kw = dict(out_dtype=dt, split_k=1)
            ww = w[:N]
            if epi == "bias_bf16":
                kw["bias"] = bias.bfloat16()
            elif epi == "bias_f32":
                kw["bias"] = bias
            elif epi in ("gelu", "silu"):
                kw["act"] = epi
            elif epi == "gated":
                ww, kw["act"], kw["gated"] = w[:Ng], "silu", True
            elif epi == "residual":
                kw["residual"] = res
            first = None
            for tn in WIDTHS:
                if epi == "gated" and tn < 64:
                    continue
                out = ops.gemm(a, ww, tile_n=tn, **kw)
                if first is None:
                    first, first_tn = out, tn
                    assert torch.isfinite(out.float()).all(), (epi, dt)
                    if epi == "none":      # not vacuous: the bits agreed on are the product
                        err = float((out.float() - ref32).abs().max() / ref32.abs().max())
                        assert err < 1e-2, (dt, err)
                    continue
                assert torch.equal(first, out), f"{epi} {dt} tile {first_tn} vs {tn}: {_first_diff(first, out)}"


# --------------------------------------------------------------------------------------------------- B. the row-norm kernels
NORM_WARP, NORM_BLOCK = 0, 1
# columns -> register tiles: warp kernel MAXV 1 (8, 256), 2 (264), 4 (1024), 5 (1280), 8 (2048), 16 (2560, 4096), 32 (8192);
# block kernel MAXV 1 (<= 2048), 2 (2560, 4096)
WARP_COLS = [8, 256, 264, 1024, 1280, 2048, 2560, 4096, 8192]
NORM_CASES = [(NORM_WARP, c) for c in WARP_COLS] + [(NORM_BLOCK, c) for c in WARP_COLS if c <= 4096]
NORM_ROWS = [1, 31, 32, 33, 600]


def _ulp_bf16(v):
    """bf16 unit in the last place of |v| (8 significant bits), elementwise, float64."""
    _, e = torch.frexp(v.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), (e - 8).to(torch.int64))


def _norm_ref(x, gamma, beta, eps, rms):
    """-> (y, bound) in float64: Qwen2RMSNorm rounds the normalised value to bf16 before the gain; LayerNorm's variance is the
    two-pass one.  Bound: one bf16 ulp of y, plus (RMS) one bf16 ulp of the normalised value times the gain -- the pre-gain
    rounding may land on the neighbour when fp32 statistics sit at a rounding boundary -- or (LayerNorm) the fp32 error of a mean
    that is large against the spread (cancellation) and of the final a * gamma + beta."""
    xd = x.double()
    cols = x.shape[1]
    g = gamma.double() if gamma is not None else torch.ones(cols, dtype=torch.float64, device=x.device)
    b = beta.double() if beta is not None else torch.zeros(cols, dtype=torch.float64, device=x.device)
    if rms:
        r = xd * torch.rsqrt((xd * xd).mean(-1, keepdim=True) + eps)
        y = r.to(torch.bfloat16).double() * g + b
        return y, _ulp_bf16(y) + g.abs() * _ulp_bf16(r)
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    a = (xd - mean) * rstd
    y = a * g + b
    return y, _ulp_bf16(y) + ((a * g).abs() + b.abs()) * 2.0 ** -20 + g.abs() * rstd * mean.abs() * 2.0 ** -16


@pytest.mark.parametrize("rms", [True, False], ids=["rms", "layernorm"])
@pytest.mark.parametrize("kernel,cols", NORM_CASES, ids=[f"{'warp' if k == NORM_WARP else 'block'}-{c}" for k, c in NORM_CASES])
def test_row_norm_matches_fp64(kernel, cols, rms):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(cols * 4 + kernel * 2 + int(rms))
    eps = 1e-6 if rms else 1e-5
    gamma = (1.0 + 0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    beta = None if rms else (0.5 * torch.randn(cols, device="cuda", generator=g)).bfloat16()
    for rows in NORM_ROWS:
        for variant in ("plain", "no_affine", "pitched", "large_mean"):
            ldx, ldy = (cols + 24, cols + 40) if variant == "pitched" else (cols, cols)
            xf = torch.randn(rows, ldx, device="cuda", generator=g) * 2.0
            if variant == "large_mean":       # mean 1000, spread 4: a one-pass variance would cancel
                xf = xf * 2.0 + 1000.0
            x = xf.bfloat16()[:, :cols]
            yfull = torch.full((rows, ldy), 7.0, dtype=torch.bfloat16, device="cuda")
            y = yfull[:, :cols]
            ga, be = (None, None) if variant == "no_affine" else (gamma, beta)
            ops.row_norm(x, ga, be, eps, rms, kernel, out=y)
            ref, bound = _norm_ref(x, ga, be, eps, rms)
            err = (y.double() - ref).abs()
            bad = err > bound
            what = (rows, variant)
            assert not bad.any(), f"{what}: {int(bad.sum())} elements beyond the bound, worst excess {float((err - bound).max())}"
            if ldy > cols:
                assert bool((yfull[:, cols:] == 7.0).all()), f"{what}: wrote past cols"


def test_row_norm_block_kernel_width_limit():
    ops = _ops()
    x = torch.ones(2, 4104, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(import_module("vlm-fo1_b200._lib").Fo1Error):
        ops.row_norm(x, None, None, 1e-6, True, NORM_BLOCK)
    ops.row_norm(x, None, None, 1e-6, True, NORM_WARP)


# ------------------------------------------------------------------------------------------------------ the engine (C, D)
@pytest.fixture(scope="module")
def pipe():
    import fo1_b200  # noqa: F401
    E = import_module("vlm-fo1_b200.engine"); CK = import_module("vlm-fo1_b200.checkpoint"); P = import_module("vlm-fo1_b200.pipeline")
    cfg = E.EngineConfig()
    cfg.vit = dict(cfg.vit, depth=4, fullatt_block_indexes=[1, 3])
    cfg.davit = dict(cfg.davit, depths=[1, 1, 1, 1])
    cfg.llm = dict(cfg.llm, num_hidden_layers=2)
    assert cfg.fpn_out == 512 and cfg.region_dim == 5888 and cfg.proj_aux_layers == 2 and cfg.llm["vocab_size"] == 151936
    eng = CK.load_engine(cfg, CK.random_state_dicts(cfg, "cuda", 0))
    return P.Fo1Pipeline(eng)


def _sample(i, S, n_boxes):
    SY = import_module("vlm-fo1_b200.synthetic"); P = import_module("vlm-fo1_b200.pipeline")
    s = SY.synthetic_sample(i, S, n_boxes)
    return P.SampleInputs(s.input_ids, s.pixel_values.cuda(), s.grid_hw, s.image_aux.cuda(), s.boxes.cuda())


# ------------------------------------------------------------------------------------------------------ C. tower stages
def _stages(pipe, samples):
    """Every stage of encode, split per sample and copied out of the engine's arena before the next call reuses it."""
    st = pipe.encode_stages(samples)
    grids = [s.grid_hw for s in samples]
    tok = np.cumsum([0] + [gh * gw for gh, gw in grids])
    cell = np.cumsum([0] + [gh * gw // 4 for gh, gw in grids])
    per = []
    for b in range(len(samples)):
        d = {f"vit_tap{t}": st["taps"][t][tok[b]:tok[b + 1]].clone() for t in range(len(st["taps"]))}
        d["image_features"] = st["image_features"][cell[b]:cell[b + 1]].clone()
        for l in range(4):
            d[f"davit{l}"] = st["davit"][l][b].clone()
            d[f"fpn{l}"] = st["fpn"][l][b].clone()
        d["region_f32"] = st["region_f32"][b].clone()
        d["region_tokens"] = st["region_tokens"][b].clone()
        per.append(d)
    return per


def _assert_same_stages(alone, got, what):
    assert alone.keys() == got.keys()
    bad = [f"{k}: {_first_diff(alone[k], got[k])}" for k in alone
           if alone[k].shape != got[k].shape or not torch.equal(alone[k], got[k])]
    assert not bad, f"{what}: " + "; ".join(bad)


_ALONE = {}


def _alone_stages(pipe, key):
    if key not in _ALONE:
        _ALONE[key] = _stages(pipe, [_sample(*key)])[0]
    return _ALONE[key]


def _assert_batch_matches_alone(pipe, keys, what):
    """Every sample of the batch ``keys`` (synthetic_sample arguments) against the same sample alone."""
    got = _stages(pipe, [_sample(*k) for k in keys])
    for b, k in enumerate(keys):
        _assert_same_stages(_alone_stages(pipe, k), got[b], f"{what}, slot {b} ({k[1]} px)")


def _same_size(i, S, slot):
    x = (i, S, 3)
    others = [(i + k, S, 1 + 2 * k) for k in (1, 2, 3)]
    return others[:slot] + [x] + others[slot:]


X56, X448 = (0, 56, 3), (20, 448, 3)
MIXED = [X448, (30, 644, 4), (31, 336, 2), (10, 112, 3)]     # 336 px starts at row 3140 of the packed ViT rows: mid-tile


@pytest.mark.parametrize("S,slot", [(56, 0), (56, 3), (112, 0), (448, 2)])
def test_tower_stages_same_size_batch(pipe, S, slot):
    """Same-size batches: ViT packed, DaViT / FPN batched, the packed HFRE path.  At 56 / 112 px the deepest DaViT and FPN maps
    have 16 rows per image: 16 rows alone, 64 in the batch."""
    _assert_batch_matches_alone(pipe, _same_size({56: 0, 112: 10, 448: 20}[S], S, slot), f"{S} px batch")


def test_tower_stages_mixed_size_batch(pipe):
    """448, 644, 336 and 112 px together: ViT packed across sizes, DaViT / FPN per image, the unpacked HFRE path."""
    _assert_batch_matches_alone(pipe, MIXED, "mixed batch")


def test_tower_stages_alone_after_mixed_batch(pipe):
    """Alone again after a large mixed batch: a dirty arena and trimmed integer-table caches change nothing."""
    a56, a448 = _alone_stages(pipe, X56), _alone_stages(pipe, X448)
    _stages(pipe, [_sample(*k) for k in MIXED])
    _assert_same_stages(a56, _stages(pipe, [_sample(*X56)])[0], "56 px alone after the mixed batch")
    _assert_same_stages(a448, _stages(pipe, [_sample(*X448)])[0], "448 px alone after the mixed batch")


# ------------------------------------------------------------------------------------------------------ D. language side
MAX_NEW = 6
XL = (150, 112, 3)


def _companion(k):
    # shorter (56 px: 4 image tokens, one box) and longer (168 px: 36 image tokens, up to 7 boxes) prompts than X's
    return (200 + k, (56, 168, 112)[k % 3], 1 + (5 * k) % 7)


def _generate(pipe, samples, stop_ids):
    scored = pipe.generate(samples, MAX_NEW, stop_ids=stop_ids, early_exit_interval=0, want_prefill_logits=True, want_logits=True)
    out = dict(prefill=scored["prefill_logits"].clone(), logits=scored["logits"].clone(), path=pipe.eng.last_decode_path())
    plain = pipe.generate(samples, MAX_NEW, stop_ids=stop_ids, early_exit_interval=0)       # the tokens of an unscored call
    out.update(tokens=plain["tokens"].clone(), lens=plain["lens"].clone())
    return out


def _splits(B, per_kernel):
    """Key splits of the decode attention for B sequences (llm.cu: decode_persistent / decode_attention)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    slots = 2 * sms if per_kernel else sms
    return max(1, min(8, slots // (B * 2)))           # 2 KV heads at the 3B widths


_ALONE_LLM = {}


def _alone_llm(pipe, key, per_kernel):
    if "stop" not in _ALONE_LLM:             # a stop id X emits at column 3, so lengths and padding are compared too
        _ALONE_LLM["stop"] = [int(_generate(pipe, [_sample(*XL)], [])["tokens"][0, 3])]
    if (key, per_kernel) not in _ALONE_LLM:
        _ALONE_LLM[key, per_kernel] = _generate(pipe, [_sample(*key)], _ALONE_LLM["stop"])
        assert _ALONE_LLM[key, per_kernel]["path"] == (0 if per_kernel else 1)
    return _ALONE_LLM[key, per_kernel]


@pytest.mark.parametrize("B,per_kernel", [(2, False), (5, False), (8, False), (12, False), (2, True), (16, True), (24, True),
                                          (33, True), (64, True)])
def test_generate_alone_equals_in_batch(pipe, B, per_kernel, monkeypatch):
    """Every sequence of the batch (X in the middle, companions with shorter and longer prompts around it) against itself alone."""
    if per_kernel:
        monkeypatch.setenv("FO1_NO_MEGA", "1")
    slot = B // 2
    comps = [_companion(k) for k in range(B - 1)]
    keys = comps[:slot] + [XL] + comps[slot:]
    alone = [_alone_llm(pipe, k, per_kernel) for k in keys]
    got = _generate(pipe, [_sample(*k) for k in keys], _ALONE_LLM["stop"])
    assert got["path"] == (0 if per_kernel else 1)
    full = _splits(B, per_kernel) == _splits(1, per_kernel)   # else the decode attention splits the keys differently after column 0
    for b, (k, a) in enumerate(zip(keys, alone)):
        what = f"B={B} {'per-kernel' if per_kernel else 'persistent'} slot {b} {k}"
        assert torch.equal(a["prefill"][0], got["prefill"][b]), f"{what} prefill logits: {_first_diff(a['prefill'][0], got['prefill'][b])}"
        a0, g0 = a["logits"][0, 0], got["logits"][0, b]
        assert torch.equal(a0, g0), f"{what} column 0 logits: {_first_diff(a0, g0)}"
        assert int(a["tokens"][0, 0]) == int(got["tokens"][b, 0]), what
        if not full:
            continue
        n = int(a["lens"][0])
        assert int(got["lens"][b]) == n, what
        assert torch.equal(a["tokens"][0], got["tokens"][b]), (what, a["tokens"][0].tolist(), got["tokens"][b].tolist())
        for t in range(n):                    # rows past a sequence's stop column are unspecified
            at, gt = a["logits"][t, 0], got["logits"][t, b]
            assert torch.equal(at, gt), f"{what} column {t} logits: {_first_diff(at, gt)}"
