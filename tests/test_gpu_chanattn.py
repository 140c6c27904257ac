"""-m gpu: DaViT channel-group attention (wgmma Gram over the token axis + wgmma mixing of v) vs a plain torch fp32 statement of
ChannelAttention.forward (modeling_davit.py:151-172), at the DaViT-large stage shapes, ragged token counts, channel counts that
are not a multiple of the 128-channel CTA tile, several token chunks (partial Grams summed in fixed order) and batch slots; every
element within the bound that follows from the kernels' rounding (tests/attention_bounds.py)."""
import pytest
import torch

from tests import attention_bounds as AB

pytestmark = pytest.mark.gpu


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
    ref, bound = AB.channel_reference(qkv, C // 32)
    r = AB.check(out, ref.reshape(B * N, C // 32, 32), bound.reshape(B * N, C // 32, 32), f"channel B {B} N {N} C {C}")
    print(f"chan_attn B {B} N {N} C {C}: max ratio {r:.3f}")
    if B > 1:
        assert torch.equal(out[0], out[1])                 # no atomics: independent of the batch slot, bit-reproducible
        # ... and of the batch SIZE: the token chunking (= the summation order of the Gram) may not change with the number of images
        assert torch.equal(out[0], ops.channel_attention(qkv[:1].contiguous(), C // 32)[0])
    assert torch.equal(out, ops.channel_attention(qkv, C // 32))
