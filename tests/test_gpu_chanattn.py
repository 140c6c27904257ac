"""-m gpu: DaViT channel-group attention (wgmma Gram over the token axis + wgmma mixing of v) vs a plain torch fp32 statement of
ChannelAttention.forward (modeling_davit.py:151-172), at the DaViT-large stage shapes, ragged token counts, channel counts that
are not a multiple of the 128-channel CTA tile, several token chunks (partial Grams summed in fixed order) and batch slots."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv, groups):
    B, N, C3 = qkv.shape
    C = C3 // 3
    x = qkv.float().reshape(B, N, 3, groups, C // groups).permute(2, 0, 3, 1, 4)      # [3, B, g, N, c]
    q, k, v = x[0] * float(N) ** -0.5, x[1], x[2]
    a = (q.transpose(-1, -2) @ k).softmax(-1)                                           # [B, g, c, c]
    o = (a @ v.transpose(-1, -2)).transpose(-1, -2)                                     # [B, g, N, c]
    return o.permute(0, 2, 1, 3).reshape(B, N, C)


@pytest.mark.parametrize("B,N,C", [(2, 50176, 256), (3, 3136, 1024), (2, 784, 2048), (1, 1000, 512), (2, 333, 64), (2, 130, 32), (5, 12544, 512)])
def test_channel_attention_matches_fp32(B, N, C):
    from importlib import import_module
    import fo1_b200  # noqa: F401
    ops = import_module("vlm-fo1_b200.ops")
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + C)
    qkv = torch.randn(B, N, 3 * C, device="cuda", generator=g).to(torch.bfloat16)
    qkv[1 % B] = qkv[0]                                   # the same map at two batch slots
    out = ops.channel_attention(qkv, C // 32)
    torch.cuda.synchronize()
    ref = _ref(qkv, C // 32)
    err = float((out.float() - ref).abs().max() / ref.abs().max())
    # the 32 softmax weights of a row are rounded to bf16 (the reference's attn tensor is bf16 too) and so is the output: two
    # storage points, each one ulp of the largest element
    assert err < 1e-3 + 2 * 2.0 ** -8, err
    if B > 1:
        assert torch.equal(out[0], out[1])                 # no atomics: independent of the batch slot, bit-reproducible
        # ... and of the batch SIZE: the token chunking (= the summation order of the Gram) may not change with the number of images
        assert torch.equal(out[0], ops.channel_attention(qkv[:1].contiguous(), C // 32)[0])
    assert torch.equal(out, ops.channel_attention(qkv, C // 32))
