"""-m gpu: the attention kernels against a float64 reference with the per-element bounds of tests/attention_bounds.py,
on inputs that make masking mistakes visible and at the kernels' edges (head dims, GQA groups, tile / key-tile / split
boundaries, the ViT geometries, the lazy rescale, every cache slot past the end poisoned)."""
from importlib import import_module

import pytest
import torch

from tests import attention_bounds as AB

pytestmark = pytest.mark.gpu


def _ops():
    import fo1_b200  # noqa: F401
    return import_module("vlm-fo1_b200.ops")


def _varlen_run(lens, qh, kvh, hd, causal, seed, **kw):
    buf, q, k, v, cu = AB.varlen_inputs(lens, qh, kvh, hd, causal, seed, **kw)
    d = buf.cuda()
    qd, kd = qh * hd, kvh * hd
    T = cu[-1]
    # views into the poisoned buffer: only the first T rows are the tokens
    out = _ops().attention_varlen(d[:T, :qd], d[:T, qd:qd + kd], d[:T, qd + kd:], torch.tensor(cu, dtype=torch.int32, device="cuda"),
                                  max(lens), qh, kvh, hd, hd ** -0.5, causal)
    torch.cuda.synchronize()
    ref, bound = AB.varlen_reference(d[:, :qd], d[:, qd:qd + kd], d[:, qd + kd:], cu, qh, kvh, hd, hd ** -0.5, causal)
    return out, ref, bound


MIXED = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257]


@pytest.mark.parametrize("hd", [32, 64, 80, 128])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_bound_shapes(hd, G, causal):
    kvh = 2 if G < 8 else 1
    lens = MIXED[G % 3:] + MIXED[:G % 3]                      # the same lengths in a different order per G
    if causal:
        lens = [[1, 63, 65][(hd // 16) % 3]] + lens           # a causal segment starting at offset 1 / 63 / 65 of a query tile
    out, ref, bound = _varlen_run(lens, G * kvh, kvh, hd, causal, hd + G)
    r = AB.check(out, ref, bound, f"varlen hd {hd} G {G} causal {causal}")
    print(f"attn_tc_kernel hd {hd} G {G} causal {causal} lens {lens}: max ratio {r:.3f}")


@pytest.mark.parametrize("start", [1, 63, 65])
def test_varlen_bound_causal_offsets(start):
    """Causal segments starting 1, 63 and 65 rows into a 128-row query tile, at the LLM's head shape."""
    lens = [start, 300, 129, 64, 5]
    out, ref, bound = _varlen_run(lens, 16, 2, 128, True, start)
    r = AB.check(out, ref, bound, f"varlen causal start {start}")
    print(f"attn_tc_kernel causal start {start} lens {lens}: max ratio {r:.3f}")


@pytest.mark.parametrize("lens", [[2116, 2116], [5184]])
def test_varlen_bound_vit_geometry(lens):
    """The ViT's C4 images (46 x 46 merged grid, two images) and one 72 x 72 image in full attention (head_dim 80)."""
    out, ref, bound = _varlen_run(lens, 2, 2, 80, False, len(lens))
    r = AB.check(out, ref, bound, f"varlen ViT {lens}")
    print(f"attn_tc_kernel ViT {lens}: max ratio {r:.3f}")


@pytest.mark.parametrize("step", [7.75, 8.25])
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_bound_lazy_rescale(step, causal):
    """Keys rise by just under / just over kAtRescale = 8 log2 units per 64-key tile: the rescale is skipped and taken."""
    buf, q, k, v, cu = AB.varlen_inputs([1000], 2, 2, 128, causal, 11, tile_step_log2=step)
    d = buf.cuda()
    T = cu[-1]
    out = _ops().attention_varlen(d[:T, :256], d[:T, 256:512], d[:T, 512:], torch.tensor(cu, dtype=torch.int32, device="cuda"),
                                  T, 2, 2, 128, 128 ** -0.5, causal)
    torch.cuda.synchronize()
    ref, bound = AB.varlen_reference(d[:, :256], d[:, 256:512], d[:, 512:], cu, 2, 2, 128, 128 ** -0.5, causal)
    r = AB.check(out, ref, bound, f"varlen rescale step {step} causal {causal}")
    print(f"attn_tc_kernel rescale step {step} causal {causal}: max ratio {r:.3f}")


# ------------------------------------------------------------------------------------------------------------- decode
DECODE_HEADS = [(16, 2), (8, 1), (14, 2), (16, 16), (4, 4)]


def _batch_for_splits(sm, kvh, S):
    """A batch whose split count (llm.cu decode_attention) is S, or None: the largest one for the most splits (more
    lengths per call), else the smallest."""
    fits = [B for B in range(1, 4 * sm + 2) if AB.decode_split_count(sm, B, kvh) == S]
    if not fits:
        return None
    return max(fits) if S == AB.DEC_SPLITS else min(fits)


def _decode_lens(B, S):
    """B lengths: = 0, 1, 15, 16, 17 mod 16, both sides of the split-chunk edges (chunk grows by 16 after 16 S j keys),
    L = 1 and L = cap (the largest)."""
    edges = [16 * S * j + e for j in (1, 2, 5) for e in (0, 1)]
    base = [1, 15, 16, 17, 32, 33, 47, 48, 49, 600, 1195] + edges
    lens = [base[i % len(base)] for i in range(B)]
    lens[-1] = 1201
    return lens


@pytest.mark.parametrize("S", [1, 2, 3, 8])
@pytest.mark.parametrize("qh,kvh", DECODE_HEADS)
def test_decode_bound(qh, kvh, S):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = _batch_for_splits(sm, kvh, S)
    if B is None:
        pytest.skip(f"no batch size gives {S} splits with {kvh} kv heads on {sm} SMs")
    lens = _decode_lens(B, S)
    cap = max(lens)
    ops = _ops()
    worst = 0.0
    for poison in ("nan", "adversarial"):
        q, kc, vc = (t.cuda() for t in AB.decode_inputs(lens, qh, kvh, cap, qh * 100 + kvh + S, poison))
        n = torch.tensor(lens, dtype=torch.int32, device="cuda")
        out = ops.decode_attention(q, kc, vc, n - 1, qh, kvh, 128 ** -0.5)
        torch.cuda.synchronize()
        ref, bound = AB.decode_reference(q, kc, vc, lens, qh, kvh, 128 ** -0.5)
        worst = max(worst, AB.check(out, ref, bound, f"decode {qh}/{kvh} B {B} splits {S} poison {poison}"))
    print(f"decode_attn {qh}/{kvh} heads, B {B} -> {S} splits ({sm} SMs), lengths {sorted(set(lens))}: max ratio {worst:.3f}")


# ------------------------------------------------------------------------------------------------------------ channel
def _chan_cases():
    tok = AB.chan_constants()[0]
    base = [(2, 50176, 256), (3, 3136, 1024), (2, 784, 2048), (1, 1000, 512), (2, 333, 64), (2, 130, 32), (5, 12544, 512)]
    edges = [(2, tok - 1, 64), (2, tok + 1, 64), (1, 32 * tok - 1, 256), (1, 32 * tok + 1, 256)]
    return base + edges


@pytest.mark.parametrize("B,N,C", _chan_cases())
def test_channel_bound(B, N, C):
    qkv = AB.chan_inputs(B, N, C, B * 1000 + C + N).cuda()
    out = _ops().channel_attention(qkv, C // 32)
    torch.cuda.synchronize()
    ref, bound = AB.channel_reference(qkv, C // 32)
    G = C // 32
    r = AB.check(out, ref.reshape(B * N, G, 32), bound.reshape(B * N, G, 32), f"channel B {B} N {N} C {C}")
    print(f"chan_attn B {B} N {N} C {C} chunks {AB.chan_plan(N, C)}: max ratio {r:.3f}")
