"""-m gpu: CTA pairs of the wgmma GEMM.  A launch with a pinned tile width, two or more m-tiles and no split-K runs as 2-CTA
clusters that multicast the W tile; a launch of one m-tile runs one CTA per tile.  Both sum every output element in the same k order
with the same wgmma shape, so each 128-row block of a paired launch must equal, bit for bit, the same rows launched alone."""
import pytest
import torch

pytestmark = pytest.mark.gpu

EPILOGUES = ["none", "bias_bf16", "bias_f32", "gelu", "silu", "gated", "residual"]


def _ops():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.ops")


def _operands(M, N, K, epi, out_dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    kw = dict(out_dtype=out_dtype)
    if epi in ("bias_bf16", "gelu", "silu", "gated"):
        kw["bias"] = torch.randn(N, device="cuda", generator=g).bfloat16()
    if epi == "bias_f32":
        kw["bias"] = torch.randn(N, device="cuda", generator=g)
    if epi in ("gelu", "silu"):
        kw["act"] = epi
    if epi == "gated":
        kw["act"], kw["gated"] = "silu", True
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16() if epi == "residual" else None
    return a, w, kw, res


def _paired_vs_alone(M, N, K, tile_n, epi, out_dtype, seed):
    ops = _ops()
    a, w, kw, res = _operands(M, N, K, epi, out_dtype, seed)
    paired = ops.gemm(a, w, residual=res, tile_n=tile_n, **kw)
    for r0 in range(0, M, 128):
        r1 = min(M, r0 + 128)
        alone = ops.gemm(a[r0:r1], w, residual=None if res is None else res[r0:r1], tile_n=tile_n, **kw)
        torch.cuda.synchronize()
        assert torch.isfinite(alone.float()).all()
        assert torch.equal(paired[r0:r1], alone), (r0, float((paired[r0:r1].float() - alone.float()).abs().max()))


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("tile_n", [32, 64, 128, 192, 256])
@pytest.mark.parametrize("M", [300, 256, 129])
def test_paired_rows_equal_rows_alone(M, tile_n, epi, out_dtype):
    """M = 300: three m-tiles, so the last pair's second CTA lies past M (zero-filled A, no epilogue) and still feeds its W half."""
    if epi == "gated" and tile_n < 64:
        pytest.skip("the gated epilogue needs 64-column tiles")
    # N = 320 leaves a partial n-tile at every width; K = 328 a partial k-block
    _paired_vs_alone(M, 320, 328, tile_n, epi, out_dtype, seed=M * 7 + tile_n + EPILOGUES.index(epi))


@pytest.mark.parametrize("tile_n,epi", [(128, "residual"), (256, "gated"), (64, "gelu")])
def test_paired_many_tiles_per_cluster(tile_n, epi):
    """More pair-tiles than clusters: each cluster walks several tiles through the grouped order, the ring wraps across tiles,
    and 17 m-tiles leave a last group of one (odd) pair."""
    _paired_vs_alone(17 * 128 - 50, 2048, 1024, tile_n, epi, torch.bfloat16, seed=tile_n)
