"""-m gpu: varlen and decode attention kernels vs a float64 reference (softmax(QK^T*scale)V per segment), every element within
the bound that follows from the kernels' rounding (tests/attention_bounds.py)."""
import math

import pytest
import torch

from tests import attention_bounds as AB

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("hd,qh,kvh,causal,lens", [
    (80, 16, 16, False, [64, 64, 48, 36, 64]),          # ViT windows incl. ragged edge windows (46x46 grid)
    (80, 4, 4, False, [1024, 700]),                     # ViT full attention
    (32, 8, 8, False, [144] * 7),                       # DaViT 12x12 windows
    (128, 16, 2, True, [333, 1195, 64, 1]),             # LLM causal GQA prefill
    (128, 16, 2, False, [200]),
    (80, 2, 2, False, [2116, 2116]),                    # C4 geometry: 46x46 grid, whole images straddle the 128-row tiles
    (80, 2, 2, False, [64] * 33 + [48] * 2 + [36]),     # one 46x46 image's ragged window list (A2 table of SURVEY.md)
    (80, 2, 2, False, [1, 127, 128, 129, 2, 255]),      # segment edges on / around the tile and key-tile boundaries
    (32, 4, 4, False, [144] * 3 + [100]),               # last tile partly beyond T
    (128, 8, 2, True, [1259] * 3),                      # C4 prompt length (244 + 529 + ...): causal tiles across sequences
    (128, 4, 2, True, [64, 64, 64, 64, 5]),             # several short causal sequences inside one tile
    (64, 4, 2, False, [300, 20]),
])
def test_attention_varlen(hd, qh, kvh, causal, lens):
    from importlib import import_module
    import fo1_b200  # noqa: F401
    ops = import_module("vlm-fo1_b200.ops")
    g = torch.Generator().manual_seed(hd + len(lens))
    T = sum(lens)
    # packed qkv buffer like the engines use: [T, (qh + 2 kvh) * hd]
    qkv = torch.randn(T, (qh + 2 * kvh) * hd, generator=g).bfloat16()
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    dq = qkv.cuda()
    q, k, v = dq[:, : qh * hd], dq[:, qh * hd:(qh + kvh) * hd], dq[:, (qh + kvh) * hd:]
    scale = 1.0 / math.sqrt(hd)
    out = ops.attention_varlen(q, k, v, torch.tensor(cu, dtype=torch.int32, device="cuda"), max(lens), qh, kvh, hd, scale, causal)
    torch.cuda.synchronize()
    ref, bound = AB.varlen_reference(q, k, v, cu, qh, kvh, hd, scale, causal)
    r = AB.check(out, ref, bound, f"varlen hd {hd} {qh}/{kvh} causal {causal} lens {lens}")
    print(f"attn_tc_kernel hd {hd} {qh}/{kvh} causal {causal}: max ratio {r:.3f}")
    assert torch.isfinite(out).all()


def test_attention_large_logits_rescale():
    """Rows whose running maximum keeps growing (keys sorted by increasing score) force the lazy O rescale (in registers) on every
    key tile; a peaked softmax (logit range ~ 60) must still match fp32."""
    from importlib import import_module
    import fo1_b200  # noqa: F401
    ops = import_module("vlm-fo1_b200.ops")
    T, hd, h = 1000, 128, 2
    g = torch.Generator().manual_seed(7)
    q = torch.randn(T, h * hd, generator=g)
    k = torch.randn(T, h * hd, generator=g)
    ramp = torch.linspace(0.0, 6.0, T).unsqueeze(1)
    k = (k + ramp * torch.sign(q.mean(0, keepdim=True))).bfloat16()          # later keys score higher for most rows
    q = (q * 3.0).bfloat16()
    v = torch.randn(T, h * hd, generator=g).bfloat16()
    cu = torch.tensor([0, T], dtype=torch.int32, device="cuda")
    for causal in (False, True):
        out = ops.attention_varlen(q.cuda(), k.cuda(), v.cuda(), cu, T, h, h, hd, hd ** -0.5, causal)
        torch.cuda.synchronize()
        ref, bound = AB.varlen_reference(q, k, v, [0, T], h, h, hd, hd ** -0.5, causal)
        r = AB.check(out, ref, bound, f"large logits causal {causal}")
        print(f"attn_tc_kernel large logits causal {causal}: max ratio {r:.3f}")


def test_attention_strided_inputs_and_reuse():
    """q/k/v as column slices of one packed buffer with an odd number of heads in front, output with a pitch; the same
    call twice (the rowseg scratch and the tensor maps are rebuilt per call) gives identical bits."""
    from importlib import import_module
    import fo1_b200  # noqa: F401
    ops = import_module("vlm-fo1_b200.ops")
    T, hd, qh, kvh = 777, 80, 3, 3
    buf = torch.randn(T, 8 + 3 * qh * hd, device="cuda").to(torch.bfloat16)
    q, k, v = buf[:, 8: 8 + qh * hd], buf[:, 8 + qh * hd: 8 + 2 * qh * hd], buf[:, 8 + 2 * qh * hd:]
    cu = torch.tensor([0, 300, 301, 777], dtype=torch.int32, device="cuda")
    obuf = torch.zeros(T, qh * hd + 16, device="cuda", dtype=torch.bfloat16)
    o1 = ops.attention_varlen(q, k, v, cu, 476, qh, kvh, hd, hd ** -0.5, False, out=obuf[:, 8: 8 + qh * hd]).clone()
    o2 = ops.attention_varlen(q, k, v, cu, 476, qh, kvh, hd, hd ** -0.5, False, out=obuf[:, 8: 8 + qh * hd]).clone()
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    assert obuf[:, :8].abs().max().item() == 0 and obuf[:, 8 + qh * hd:].abs().max().item() == 0     # nothing written outside
    ref, bound = AB.varlen_reference(q, k, v, [0, 300, 301, 777], qh, kvh, hd, hd ** -0.5, False)
    AB.check(o1, ref, bound, "strided inputs")


@pytest.mark.parametrize("q_heads,kv_heads", [(16, 2), (8, 2), (4, 4), (8, 1)])
@pytest.mark.parametrize("lens", [[1, 15, 16, 17], [600, 1195, 33, 2, 257], [48] * 40])
def test_decode_attention_matches_reference(q_heads, kv_heads, lens):
    """One decode step of GQA attention over the K/V cache (tensor-core tile of the group's query heads, cp.async ring,
    split over the keys) vs torch fp32 on the same bf16 cache; ragged lengths incl. < 1 tile, tile edges, many splits."""
    from importlib import import_module
    import fo1_b200  # noqa: F401
    ops = import_module("vlm-fo1_b200.ops")
    B, cap, hd = len(lens), max(lens) + 3, 128
    g = torch.Generator(device="cuda").manual_seed(q_heads * 100 + kv_heads + len(lens))
    q = torch.randn(B, q_heads * hd, device="cuda", generator=g).to(torch.bfloat16)
    kc = torch.randn(B, cap, kv_heads * hd, device="cuda", generator=g).to(torch.bfloat16)
    vc = torch.randn(B, cap, kv_heads * hd, device="cuda", generator=g).to(torch.bfloat16)
    kc[:, -2:] = float("nan")      # slots beyond every length must never be read into the result
    vc[:, -2:] = float("inf")
    n = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = hd ** -0.5
    out = ops.decode_attention(q, kc, vc, n - 1, q_heads, kv_heads, scale)
    torch.cuda.synchronize()
    ref, bound = AB.decode_reference(q, kc, vc, lens, q_heads, kv_heads, scale)
    r = AB.check(out, ref, bound, f"decode {q_heads}/{kv_heads} lens {lens}")
    print(f"decode_attn {q_heads}/{kv_heads} lens {lens}: max ratio {r:.3f}")
