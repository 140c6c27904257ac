"""-m gpu: the wgmma GEMM (through the C ABI) vs a plain torch fp32 reference of the same op.
Inputs are bf16-rounded; accumulation is fp32 in both; tolerance 1e-3 relative on the fp32 result,
plus bf16 output rounding (2^-8) when the output is bf16."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from importlib import import_module
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.ops")


def _ref(a, w, bias=None, act=None, residual=None):
    y = a.float() @ w.float().t()
    if bias is not None:
        y = y + bias.float()
    if act == "gelu":
        y = torch.nn.functional.gelu(y)
    elif act == "silu":
        y = torch.nn.functional.silu(y)
    if residual is not None:
        y = y + residual.float()
    return y


def _check(got, ref, bf16_out):
    err = (got.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    tol = (1e-3 + (2 ** -8 if bf16_out else 0)) * scale
    assert err <= tol, f"max err {err} > tol {tol} (scale {scale})"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 256, 512), (4096, 1280, 1280), (1000, 3840, 1280),
                                   (37, 100, 72), (4096, 1280, 1176), (300, 2048, 5888), (129, 65, 136),
                                   (8192, 2048, 2048)])
def test_gemm_plain(M, N, K):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = ops.gemm(a, w, out_dtype=torch.float32)
    torch.cuda.synchronize()
    _check(out, _ref(a, w), False)
    out16 = ops.gemm(a, w)
    torch.cuda.synchronize()
    _check(out16, _ref(a, w), True)


def _check_rows(got, a, w, rows, bias=None, act=None, residual=None):
    """sampled rows of a problem too large for a full fp32 reference"""
    ref = _ref(a[rows], w, bias, act, None if residual is None else residual[rows])
    _check(got[rows], ref, got.dtype == torch.bfloat16)


@pytest.mark.parametrize("M,N,K", [(32768, 3840, 1280), (19000, 1280, 3456), (37888 + 77, 520, 1280)])
def test_gemm_large_plain(M, N, K):
    """the tower / prefill shapes of a 32-image batch: many waves of 256-wide tiles per persistent CTA, ragged last tiles"""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    out = ops.gemm(a, w)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    rows = torch.cat([torch.randint(0, M, (256,), device="cuda"), torch.arange(M - 130, M, device="cuda")])
    _check_rows(out, a, w, rows)


def test_gemm_large_epilogues():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(7)
    M, N, K = 38400, 2560, 1280
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16()
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    rows = torch.randint(0, M, (256,), device="cuda")
    out = ops.gemm(a, w, bias=bias, act="gelu", residual=res)
    _check_rows(out, a, w, rows, bias, "gelu", res)
    out = ops.gemm(a, w, out_dtype=torch.float32)
    _check_rows(out, a, w, rows)
    out = ops.gemm(a, w, bias=bias, act="silu", gated=True)        # W rows interleave [32 gate | 32 up] blocks
    y = (a[rows].float() @ w.float().t() + bias.float()).view(len(rows), N // 64, 2, 32)
    ref = (torch.nn.functional.silu(y[:, :, 0]) * y[:, :, 1]).reshape(len(rows), N // 2)
    _check(out[rows], ref, True)


@pytest.mark.parametrize("act", [None, "gelu", "silu"])
@pytest.mark.parametrize("bias_dtype", [torch.bfloat16, torch.float32])
def test_gemm_epilogues(act, bias_dtype):
    ops = _ops()
    M, N, K = 777, 1280, 640
    g = torch.Generator(device="cuda").manual_seed(11)
    a = (torch.randn(M, K, device="cuda", generator=g)).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.04).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g).to(bias_dtype)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    out = ops.gemm(a, w, bias=bias, act=act, residual=res, out_dtype=torch.float32)
    torch.cuda.synchronize()
    _check(out, _ref(a, w, bias, act, res), False)


@pytest.mark.parametrize("M,N,K", [(32, 2048, 11008), (32, 2560, 2048), (4, 2048, 2048), (1, 2048, 2048), (100, 2048, 5888),
                                   (32, 2048, 2048), (17, 96, 4096), (32, 151936, 2048)])
def test_gemm_skinny_splitk(M, N, K):
    """decode-shaped problems take the narrow-tile / split-K path (partials reduced in-kernel by the last CTA);
    run twice: the per-tile arrival counters must be self-cleaning."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.2).to(torch.bfloat16)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    ref = _ref(a, w, bias, "gelu", res)
    for _ in range(2):
        out = ops.gemm(a, w, bias=bias, act="gelu", residual=res, out_dtype=torch.float32)
        torch.cuda.synchronize()
        _check(out, ref, False)
    out2 = ops.gemm(a, w, bias=bias, act="gelu", residual=res, out_dtype=torch.float32)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)      # fixed reduction order -> bitwise reproducible


@pytest.mark.parametrize("tile_n,split_k", [(32, 1), (32, 4), (64, 3), (128, 8), (256, 5), (128, 1), (192, 1), (192, 3)])
@pytest.mark.parametrize("M", [32, 130])
def test_gemm_pinned_tile_and_split(tile_n, split_k, M):
    """every tile width x split-K variant the descriptor can pin: cooperative reduction by the last CTA of a tile,
    bias / activation / residual applied after the reduction, bit-reproducible"""
    ops = _ops()
    N, K = 1000, 2112        # ragged N tile, 33 k-blocks (uneven splits)
    g = torch.Generator(device="cuda").manual_seed(tile_n + split_k + M)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.2).to(torch.float32)
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    ref = _ref(a, w, bias, "silu", res)
    outs = []
    for dt in (torch.float32, torch.bfloat16, torch.float32):
        out = ops.gemm(a, w, bias=bias, act="silu", residual=res, out_dtype=dt, tile_n=tile_n, split_k=split_k)
        torch.cuda.synchronize()
        _check(out, ref, dt == torch.bfloat16)
        outs.append(out)
    assert torch.equal(outs[0], outs[2])


@pytest.mark.parametrize("tile_n,split_k", [(64, 1), (64, 3), (128, 4), (256, 2), (256, 7), (192, 1), (192, 2)])
def test_gemm_gated_split(tile_n, split_k):
    """the gated epilogue after a split-K reduction (decode gate/up projection)"""
    ops = _ops()
    M, K, I = 32, 2048, 1000
    g = torch.Generator(device="cuda").manual_seed(tile_n * 3 + split_k)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    wg = (torch.randn(I, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    wu = (torch.randn(I, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    bg = (torch.randn(I, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    bu = (torch.randn(I, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    w = ops.interleave_gate_up(wg, wu); b = ops.interleave_gate_up(bg, bu)
    ref = torch.nn.functional.silu(x.float() @ wg.float().t() + bg.float()) * (x.float() @ wu.float().t() + bu.float())
    for dt in (torch.float32, torch.bfloat16):
        out = ops.gemm(x, w, bias=b, act="silu", gated=True, out_dtype=dt, tile_n=tile_n, split_k=split_k)
        torch.cuda.synchronize()
        assert out.shape == (M, 1024)
        _check(out[:, :I], ref, dt == torch.bfloat16)
        assert out[:, I:].abs().max().item() == 0.0


def test_gemm_gated_silu():
    """Qwen2 MLP front half: silu(x Wg^T + bg) * (x Wu^T + bu) with the [32 gate | 32 up] row interleave;
    intermediate size 3420 is zero-padded to 3424 by the host-side weight prep."""
    ops = _ops()
    M, K, I = 520, 1280, 3420
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    wg = (torch.randn(I, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    wu = (torch.randn(I, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    bg = (torch.randn(I, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    bu = (torch.randn(I, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    w = ops.interleave_gate_up(wg, wu); b = ops.interleave_gate_up(bg, bu)
    out = ops.gemm(x, w, bias=b, act="silu", gated=True, out_dtype=torch.float32)
    torch.cuda.synchronize()
    ref = torch.nn.functional.silu(x.float() @ wg.float().t() + bg.float()) * (x.float() @ wu.float().t() + bu.float())
    assert out.shape == (M, 3424)  # 3420 padded to a multiple of the 32-row interleave block
    _check(out[:, :I], ref, False)
    assert out[:, I:].abs().max().item() == 0.0


def test_gemm_strided_views_and_errors():
    ops = _ops()
    from importlib import import_module
    L = import_module("vlm-fo1_b200._lib")
    g = torch.Generator(device="cuda").manual_seed(3)
    big = torch.randn(300, 512, device="cuda", generator=g).to(torch.bfloat16)
    a = big[:, 128:384]                      # K=256 view with pitch 512
    w = (torch.randn(192, 256, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    outbuf = torch.zeros(300, 400, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, w, out=outbuf[:, 8:200])
    torch.cuda.synchronize()
    _check(outbuf[:, 8:200], _ref(a, w), True)
    assert outbuf[:, :8].abs().max().item() == 0 and outbuf[:, 200:].abs().max().item() == 0
    with pytest.raises(L.Fo1Error):          # pitch not a multiple of 8 elements -> TMA cannot address it
        ops.gemm(torch.zeros(16, 68, device="cuda", dtype=torch.bfloat16)[:, :64], w[:, :64])
