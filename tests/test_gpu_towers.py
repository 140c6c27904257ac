"""-m gpu: ViT (+taps), DaViT, SimpleFPN and the region projector, through the C ABI, vs the fp32 oracles
on the reference-module goldens' weights and inputs.

Tolerance: the engine keeps activations in bf16 between kernels (like the reference on GPU) while the oracle
is fp32 end to end, so the bound is 1e-3-per-stage compounded over depth: each test states its bound."""
import numpy as np
import pytest
import torch

from tests.golden_io import load, nerr

pytestmark = pytest.mark.gpu


def _mods():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.engine"), import_module("vlm-fo1_b200.weights")


def _small_engine(vit_cfg=None, davit_cfg=None, fpn_out=32, region_dim=64, llm_hidden=48):
    E, W = _mods()
    cfg = E.EngineConfig()
    cfg.use_llm = False
    cfg.llm = dict(cfg.llm, hidden_size=llm_hidden)
    if vit_cfg is not None:
        cfg.vit = dict(vit_cfg)
    else:
        cfg.use_vit = False
    if davit_cfg is not None:
        cfg.davit = dict(davit_cfg)
    else:
        cfg.use_davit = False
    cfg.fpn_out = fpn_out
    cfg.region_dim = region_dim
    cfg.proj_aux_layers = 0
    return E.Engine(cfg), W


def test_vit_forward_matches_oracle():
    from oracle import vit as OV
    sd, z = load("vit_small")
    eng, W = _small_engine(vit_cfg=z["cfg"], fpn_out=0)
    eng.set_weights(W.prepare_vit(sd, z["cfg"], eng.device))
    eng.finalize()
    tags = ["a", "b", "a"]                      # ragged batch: 6x10, 8x8, 6x10 grids packed in one sequence
    px = [torch.from_numpy(z[f"px_{t}"]) for t in tags]
    grids = [tuple(int(v) for v in z[f"grid_{t}"]) for t in tags]
    feats, taps = eng.vit_forward(px, grids)
    torch.cuda.synchronize()
    tok = cell = 0
    for t, (gh, gw) in zip(tags, grids):
        ref_m, ref_t = OV.vit_forward(sd, z["cfg"], torch.from_numpy(z[f"px_{t}"]), gh, gw)
        n, nm = gh * gw, gh * gw // 4
        # 4 blocks with bf16 activations between kernels (as the reference stores them) vs an fp32 oracle:
        # bf16 eps is 3.9e-3 per rounding; ~10 roundings per block accumulate with random sign -> 2e-2 bound
        assert nerr(feats[cell:cell + nm].cpu(), ref_m) < 2e-2, t
        for i, rt in enumerate(ref_t):
            got = taps[i][tok:tok + n].reshape(gh, gw, -1).cpu()
            assert nerr(got, rt) < 2e-2, (t, i)
        tok += n; cell += nm


def test_davit_forward_matches_oracle():
    from oracle import davit as OD
    sd, z = load("davit_small")
    cfg = z["cfg"]
    eng, W = _small_engine(davit_cfg=dict(depths=cfg["depths"], dim_embed=cfg["dim_embed"], num_heads=cfg["num_heads"],
                                          num_groups=cfg["num_groups"], window_size=cfg["window_size"]), fpn_out=0)
    eng.set_weights(W.prepare_davit(sd, cfg, eng.device))
    eng.finalize()
    for tag in ("a", "b"):
        img = torch.from_numpy(z[f"img_{tag}"])
        outs = eng.davit_forward([img, img])
        torch.cuda.synchronize()
        ref = OD.davit_forward(sd, cfg, img)
        for i, r in enumerate(ref):
            assert nerr(outs[i][0].cpu(), r) < 2e-2, (tag, i)
            assert torch.equal(outs[i][0], outs[i][1])   # batch entries are independent and deterministic


def test_fpn_forward_matches_oracle():
    from oracle import davit as OD
    sd, z = load("fpn_small")
    eng, W = _small_engine(vit_cfg=dict(depth=0, hidden_size=64, num_heads=2, intermediate_size=64, out_hidden_size=48, patch_size=14,
                                        spatial_merge_size=2, temporal_patch_size=2, in_channels=3, window_size=112,
                                        fullatt_block_indexes=[]), fpn_out=32)
    eng.set_weights(W.prepare_fpn(sd, eng.device))
    eng.finalize()   # vit depth 0: only the FPN weights are required
    for tag in ("a", "b"):
        tap = torch.from_numpy(z[f"tap_{tag}"]).to("cuda", torch.bfloat16)
        outs = eng.fpn_forward(torch.stack([tap, tap]))
        torch.cuda.synchronize()
        ref = OD.fpn_forward(sd, torch.from_numpy(z[f"tap_{tag}"]))
        for i, r in enumerate(ref):
            assert nerr(outs[i][0].cpu(), r) < 1e-2, (tag, i)


def test_region_projector_matches_oracle():
    from oracle import davit as OD
    E, W = _mods()
    g = torch.Generator().manual_seed(4)
    D, Hh = 5888, 2048
    sd = {"0.weight": (torch.randn(Hh, D, generator=g) * 0.02).bfloat16().float(), "0.bias": (torch.randn(Hh, generator=g) * 0.1).bfloat16().float(),
          "2.weight": (torch.randn(Hh, Hh, generator=g) * 0.02).bfloat16().float(), "2.bias": (torch.randn(Hh, generator=g) * 0.1).bfloat16().float()}
    cfg = E.EngineConfig(); cfg.use_vit = cfg.use_davit = cfg.use_llm = False
    eng = E.Engine(cfg)
    eng.set_weights(W.prepare_projector(sd, "proj_aux", eng.device))
    eng.finalize()
    x = torch.randn(100, D, generator=g).bfloat16()
    out = eng.region_project(x.cuda())
    torch.cuda.synchronize()
    ref = OD.projector_forward(sd, x.float())
    assert nerr(out.cpu(), ref) < 8e-3   # two GEMMs with a bf16 intermediate + bf16 output


@pytest.mark.parametrize("grid", [(32, 32), (16, 16), (64, 64)])
def test_fpn_implicit_conv_equals_im2col_path(grid, monkeypatch):
    """SimpleFPN's 3x3 convs run as an implicit GEMM (4-D TMA patches, zero padding by the out-of-range fill, gemm_wgmma.cu
    conv3x3_gemm); FO1_FPN_IM2COL forces the explicit column matrix + linear.  Same products in the same k order: bit-identical."""
    E, W = _mods()
    CK = __import__("importlib").import_module("vlm-fo1_b200.checkpoint")
    cfg = E.EngineConfig(); cfg.use_davit = cfg.use_llm = False; cfg.proj_aux_layers = 0
    cfg.vit = dict(cfg.vit, depth=0, fullatt_block_indexes=[])
    eng = E.Engine(cfg)
    g = torch.Generator(device="cuda").manual_seed(9)
    eng.set_weights(W.prepare_fpn(CK.random_fpn(cfg.vit["hidden_size"], cfg.fpn_out, g, "cuda"), eng.device))
    eng.finalize()
    gh, gw = grid
    tap = (torch.randn(2, gh, gw, cfg.vit["hidden_size"], device="cuda", generator=g) * 0.5).bfloat16()
    a = [t.clone() for t in eng.fpn_forward(tap)]
    monkeypatch.setenv("FO1_FPN_IM2COL", "1")
    b = eng.fpn_forward(tap)
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.isfinite(a[i].float()).all()
        rows = a[i].shape[0] * a[i].shape[1] * a[i].shape[2]
        diff = (a[i].float() - b[i].float()).abs()
        if rows >= 132 * 128:      # both paths run the same unsplit 256-wide tiles: same products, same order
            assert torch.equal(a[i], b[i]), (i, float(diff.max()))
        else:                      # the explicit path's small GEMM is split over K (other summation order): bf16-ulp flips before the LayerNorm
            assert float(diff.max()) <= 0.0625 and float(diff.mean()) < 2e-3 and float((diff == 0).float().mean()) > 0.8, \
                (i, float(diff.max()), float(diff.mean()), float((diff == 0).float().mean()))
