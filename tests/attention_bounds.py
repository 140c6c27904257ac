"""Per-element error bounds for the attention kernels, against a float64 reference computed from the exact bf16 inputs.

A flat tolerance on an attention output is about one standard deviation of the output itself: a softmax average over
hundreds of keys is small, so a key dropped, counted twice or read from the wrong segment passes it.  The bounds here
follow from where the kernels round, element by element, so such a defect fails.

Notation for one output row: exact scores s_i = scale * q.k_i over the live keys, p = softmax(s), ref = sum_i p_i v_i,
A_i = scale * sum_d |q_d k_id|, M = max_i |s_i|.  The constants:

    U8  = 2^-8   bf16 unit roundoff (8 significant bits, round to nearest even; 2^-9 would be half of it)
    U23 = 2^-23  one fp32 step: tensor-core accumulation may truncate instead of rounding
    U24 = 2^-24  fp32 unit roundoff
    gamma(n) = 17 (ceil(n/16) + 1) U23
        an n-term dot product accumulated by k16 MMA steps (wgmma / mma.sync): each step adds 16 exact bf16 products to an
        fp32 accumulator, a 17-term sum whose error is at most 17 U23 of the running absolute sum; ceil(n/16) + 1 steps
        (one more for a range that is not 16-aligned), each running sum <= sum |terms|.

|out - ref| <= SAFETY * ( U8 sum p|v|                      P rounded to bf16 after the exponential, relative to the
                                                            normalised p (attention_tc.cu:284-296, llm.cu:198-201)
                        + U8 |ref|                          the output rounded to bf16 once
                        + c_fp32 sum p|v|                   fp32 P.V accumulation, row sum and merges (below)
                        + sum_i p_i e_i (|v_i| + |ref|) )   score errors: P_i carries a relative error e_i up to a
                                                            factor common to the row, which moves the output by
                                                            sum_i p_i e_i (v_i - ref); |v_i - ref| <= |v_i| + |ref|

    e_i = gamma(hd) A_i              fp32 Q.K^T
        + U23 (|s_i| + M)            scale * log2(e) rounded to fp32, fmaf(s, sl2, -m) / s * sc - m rounded (the running
                                     maximum m is one of the row's scores, so |t| <= log2(e) (|s_i| + M))
        + EXP_REL                    ex2.approx.ftz / exp2f / __expf, relative
The row sum l is taken from the unrounded fp32 P (attention_tc.cu:284-288, llm.cu:199), so only its fp32 summation and
the final 1/l enter.  A rescale multiplies O and l by the same alpha, so alpha's own error cancels.

c_fp32 for attn_tc_kernel (fo1_attention_varlen), n live keys of the row:
    gamma(n)                 O += P.V by wgmma
    + (n + n/32 + 3) U24     l summed in fp32, at most n/64 lazy rescales of O and l (kAtRescale), 1/l and O * (1/l)
c_fp32 for decode_attn_kernel + decode_attn_combine_kernel (fo1_decode_attention), the same plus
    + (n/16 + 2 (kDecWarps + kDecSplits) + 2) U24
                             O rescaled on every 16-key tile, the fp32 merge of the 4 warps of a split, the merge of up
                             to kDecSplits = 8 splits (a product and a sum each) and num / den
Channel attention (chan_gram_tc_kernel / chan_apply_tc_kernel, fo1_channel_attention) is the same form with the 32
channels c2 of a group as the keys and the tokens as the output columns; there the score error is dominated by the fp32
Gram over the token axis, which is bounded from the exact partial sums (see channel_reference).

SAFETY = 1.5 covers the second-order terms the first-order expansion drops (e^e - 1 vs e, the bf16 rounding of an
output that already carries the other errors, fp32 roundings of the merges of rounded values).

Everything is first order in the unit roundoffs and worst case in the signs; the only data dependence is through the
exact quantities above, computed in float64.
"""
import math
import re
from pathlib import Path

import torch

U8 = 2.0 ** -8
U23 = 2.0 ** -23
U24 = 2.0 ** -24
EXP_REL = 2.0 ** -21
SAFETY = 1.5
DEC_WARPS, DEC_SPLITS = 4, 8          # llm.cu: kDecWarps, kDecSplits

CSRC = Path(__file__).resolve().parent.parent / "vlm-fo1_b200" / "csrc"


def gamma(n):
    """fp32 error factor of an n-term dot product accumulated by k16 MMA steps (n: int or tensor)."""
    if torch.is_tensor(n):
        return 17.0 * (torch.ceil(n.double() / 16) + 1) * U23
    return 17.0 * (math.ceil(n / 16) + 1) * U23


def _softmax_bound(s, err_abs, v, live, c_fp32):
    """s [..., R, K] exact scores, err_abs [..., R, K] bound of the score's fp32 error from the dot product (absolute),
    v [..., K, D], live [..., R, K] bool, c_fp32 [..., R] -> (ref, bound) [..., R, D] float64."""
    s0 = s.masked_fill(~live, 0.0)
    p = torch.softmax(s.masked_fill(~live, float("-inf")), dim=-1).nan_to_num(0.0)
    va = v.abs()
    ref = p @ v
    pva = p @ va
    M = s0.abs().amax(dim=-1, keepdim=True)
    e = (err_abs.masked_fill(~live, 0.0) + U23 * (s0.abs() + M) + EXP_REL) * live
    pe = p * e
    score = pe @ va + ref.abs() * pe.sum(dim=-1, keepdim=True)
    bound = SAFETY * ((U8 + c_fp32.unsqueeze(-1)) * pva + U8 * ref.abs() + score)
    return ref, bound


# ------------------------------------------------------------------------------------------------------------- varlen
def varlen_reference(q, k, v, cu, q_heads, kv_heads, hd, scale, causal):
    """softmax(q k^T scale) v per segment of cu (causal: keys up to the row), GQA head h reading kv head h / G.
    q [T', qh*hd], k / v [T', kvh*hd] (rows past cu[-1] are not read) -> (ref, bound) float64 [T, qh, hd]."""
    cu = [int(x) for x in cu]
    T, G = cu[-1], q_heads // kv_heads
    dev = q.device
    ref = torch.zeros(T, q_heads, hd, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(ref)
    for a, b in zip(cu[:-1], cu[1:]):
        n = b - a
        if n == 0:
            continue
        qq = q[a:b].double().reshape(n, q_heads, hd).transpose(0, 1)                       # [qh, n, hd]
        kk = k[a:b].double().reshape(n, kv_heads, hd).transpose(0, 1).repeat_interleave(G, 0)
        vv = v[a:b].double().reshape(n, kv_heads, hd).transpose(0, 1).repeat_interleave(G, 0)
        live = torch.ones(n, n, dtype=torch.bool, device=dev)
        if causal:
            live = torch.tril(live)
        n_live = live.sum(-1)
        c_fp32 = gamma(n_live) + (n_live * (1 + 1 / 32) + 3) * U24
        for h0 in range(0, q_heads, 4):                                                   # bounded memory at 5000+ keys
            hs = slice(h0, h0 + 4)
            s = (qq[hs] @ kk[hs].transpose(1, 2)) * scale
            err = gamma(hd) * scale * (qq[hs].abs() @ kk[hs].abs().transpose(1, 2))
            r, bd = _softmax_bound(s, err, vv[hs], live.expand_as(s), c_fp32.expand(s.shape[:-1]))
            ref[a:b, hs] = r.transpose(0, 1)
            bound[a:b, hs] = bd.transpose(0, 1)
    return ref, bound


# ------------------------------------------------------------------------------------------------------------- decode
def decode_reference(q, k_cache, v_cache, lens, q_heads, kv_heads, scale):
    """One decode step: row b attends keys [0, lens[b]) of its cache slot.  q [B, qh*128], caches [B, cap, kvh*128]
    (anything past lens[b] is not read) -> (ref, bound) float64 [B, qh, 128]."""
    hd, G = 128, q_heads // kv_heads
    B, cap = k_cache.shape[0], k_cache.shape[1]
    dev = q.device
    lens_t = torch.as_tensor([int(x) for x in lens], device=dev)
    Lm = int(lens_t.max())
    ref = torch.zeros(B, q_heads, hd, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(ref)
    keys_live = torch.arange(Lm, device=dev)[None, :] < lens_t[:, None]                  # [B, Lm]
    step = max(1, (1 << 26) // max(1, q_heads * Lm * hd))
    for b0 in range(0, B, step):
        bs = slice(b0, min(B, b0 + step))
        nb = bs.stop - bs.start
        kl = keys_live[bs]
        qq = q[bs].double().reshape(nb, q_heads, 1, hd)
        kk = k_cache[bs, :Lm].double().reshape(nb, Lm, kv_heads, hd).permute(0, 2, 1, 3)
        vv = v_cache[bs, :Lm].double().reshape(nb, Lm, kv_heads, hd).permute(0, 2, 1, 3)
        kk = kk.masked_fill(~kl[:, None, :, None], 0.0).repeat_interleave(G, 1)            # [nb, qh, Lm, hd]
        vv = vv.masked_fill(~kl[:, None, :, None], 0.0).repeat_interleave(G, 1)
        s = (qq @ kk.transpose(-1, -2)) * scale                                            # [nb, qh, 1, Lm]
        err = gamma(hd) * scale * (qq.abs() @ kk.abs().transpose(-1, -2))
        live = kl[:, None, None, :].expand_as(s)
        n = lens_t[bs].double()[:, None, None].expand(nb, q_heads, 1)
        c_fp32 = gamma(n) + (n * (1 + 1 / 32) + 3) * U24 + (n / 16 + 2 * (DEC_WARPS + DEC_SPLITS) + 2) * U24
        r, bd = _softmax_bound(s, err, vv, live, c_fp32)
        ref[bs], bound[bs] = r[:, :, 0], bd[:, :, 0]
    return ref, bound


def decode_split_count(sm_count, n_seqs, kv_heads):
    """llm.cu decode_attention: one wave of 2 blocks per SM over (sequence, kv head), at most kDecSplits splits."""
    return max(1, min(DEC_SPLITS, (2 * sm_count) // max(1, n_seqs * kv_heads)))


def decode_chunk(n, n_splits):
    """Keys per split of a row with n keys (decode_attn_kernel): a multiple of the 16-key tile."""
    return ((n + n_splits - 1) // n_splits + 15) & ~15


# ------------------------------------------------------------------------------------------------------------ channel
def chan_constants():
    """kCaTok / kCaQuad / kCaMaxChunks as chanattn_tc.cu defines them."""
    src = (CSRC / "chanattn_tc.cu").read_text()
    get = lambda name: int(re.search(rf"constexpr int {name} = (\d+);", src).group(1))
    return get("kCaTok"), get("kCaQuad"), get("kCaMaxChunks")


def chan_plan(N, C):
    """chanattn_tc.cu chan_plan: (n_chunks, tiles_per_chunk) of the token axis; about two CTAs per SM of a 132-SM part
    for one image, independent of the batch size."""
    tok, quad, max_chunks = chan_constants()
    quads, tiles = -(-C // quad), -(-N // tok)
    n = -(-2 * 132 // max(1, quads))
    n = max(1, min(n, min(tiles, max_chunks)))
    tpc = -(-tiles // n)
    return -(-tiles // tpc), tpc


def channel_reference(qkv, groups):
    """DaViT channel attention (A = softmax_c2((q N^-0.5)^T k) per group of 32 channels, out = (A v^T)^T).
    qkv [B, N, 3C] -> (ref, bound) float64 [B, N, C].

    Gram term.  chan_gram_tc_kernel accumulates G[c1][c2] = sum_tok q k over the tokens of a chunk (tiles_per_chunk
    128-token tiles) with one wgmma chain of k16 steps, then chan_apply_tc_kernel adds the chunks' partial Grams in a
    fixed order.  A k16 step adds 16 exact products to the fp32 accumulator: error <= 17 U23 (|acc| + sum_block |qk|),
    with acc the chunk's partial sum before the step.  The worst case |acc| <= running absolute sum would be ~N U23
    sum|qk| and no bound at all at N = 50176, so the exact partial sums are used instead (first order: the kernel's acc
    differs from them by its own error).  The chunk sum adds U24 |partial over chunks| per chunk.  Then the scale
    (1/sqrtf(N) and the product: 2 U24 relative) and the softmax as for the other kernels: fp32 exponentials, the sum of
    32 weights and the product by 1/sum are a relative error common to the row (34 U24, no cancellation: the weights are
    used as they are), the weights rounded to bf16, A.v^T by wgmma over K = 128 (96 zero columns), the output to bf16."""
    B, N, C3 = qkv.shape
    C = C3 // 3
    tok = chan_constants()[0]
    n_chunks, tpc = chan_plan(N, C)
    steps = tpc * tok // 16
    Np = n_chunks * tpc * tok
    dev = qkv.device
    scale = float(N) ** -0.5
    ref = torch.zeros(B, N, C, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(ref)
    for b in range(B):
        x = qkv[b].double().reshape(N, 3, groups, 32)
        q = torch.zeros(Np, groups, 32, dtype=torch.float64, device=dev)
        k = torch.zeros_like(q)
        q[:N], k[:N] = x[:, 0], x[:, 1]
        v = x[:, 2].permute(1, 2, 0)                                                      # [g, 32 c2, N]
        qb = q.reshape(n_chunks, steps, 16, groups, 32)
        kb = k.reshape(n_chunks, steps, 16, groups, 32)
        blk = torch.einsum("cjtgx,cjtgy->cjgxy", qb, kb)                                   # per k16 step
        blk_abs = torch.einsum("cjtgx,cjtgy->cjgxy", qb.abs(), kb.abs())
        acc_before = torch.cumsum(blk, dim=1) - blk
        err_g = 17 * U23 * (acc_before.abs() + blk_abs).sum(dim=(0, 1))                    # [g, 32, 32]
        part = blk.sum(dim=1)                                                              # [chunks, g, 32, 32]
        err_g += U24 * torch.cumsum(part, dim=0).abs().sum(dim=0)
        G = part.sum(dim=0)
        s = G * scale
        err = err_g * scale + 2 * U24 * s.abs()
        live = torch.ones_like(s, dtype=torch.bool)
        c_fp32 = torch.full(s.shape[:-1], gamma(128) + 34 * U24, dtype=torch.float64, device=dev)
        r, bd = _softmax_bound(s, err, v, live, c_fp32)                                    # [g, 32 c1, N]
        ref[b] = r.permute(2, 0, 1).reshape(N, C)
        bound[b] = bd.permute(2, 0, 1).reshape(N, C)
    return ref, bound


# ----------------------------------------------------------------------------------------------------------- builders
# Inputs on which masking mistakes are large, not one standard deviation of random data.  All bf16, on the CPU.
POISON_ROWS = 64


def _orthonormal(g, n, hd):
    return torch.linalg.qr(torch.randn(hd, n, generator=g, dtype=torch.float64))[0].T.float()    # [n, hd]


def varlen_inputs(lens, q_heads, kv_heads, hd, causal, seed, tile_step_log2=None, plain=False):
    """Packed [T + POISON_ROWS, (qh + 2 kvh) hd] buffer -> (buf, q, k, v, cu).  Rows past T are NaN: a read past
    total_rows poisons the output.
      - Every kv head has a direction u.  Segment s's queries carry +6 sigma_s u, its keys -6 sigma_s u, sigma_s = (-1)^s:
        a key of a neighbouring segment scores ~6.4 nats above the row's own keys.  Odd segments' V are offset by +50, so
        a leaked weight p moves the output by ~50 p.
      - causal: queries also carry +6 w (w orthogonal to u) and keys a ramp along w rising ~min(0.1, 40/n) nats per
        position, so the keys after a row (and the previous segment's last keys) score highest.
      - tile_step_log2 (one segment): keys ramp along w by that many log2 units per 64-key tile and nothing else, so the
        running maximum grows by just under / just over kAtRescale per tile.
      - plain: unit normal q, k, v and nothing else (the data the flat tolerance was set on)."""
    g = torch.Generator().manual_seed(seed)
    G = q_heads // kv_heads
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    T = cu[-1]
    scale = hd ** -0.5
    q = torch.randn(T, q_heads, hd, generator=g)
    k = torch.randn(T, kv_heads, hd, generator=g)
    v = torch.randn(T, kv_heads, hd, generator=g)
    dirs = torch.stack([_orthonormal(g, 2, hd) for _ in range(kv_heads)])                  # [kvh, 2, hd]
    u, w = dirs[:, 0], dirs[:, 1]
    uq, wq = u.repeat_interleave(G, 0), w.repeat_interleave(G, 0)
    for s, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        pos = torch.arange(b - a, dtype=torch.float32)[:, None, None]
        if plain:
            continue
        if tile_step_log2 is not None:
            q[a:b] = 0.25 * q[a:b] + 8.0 * wq
            k[a:b] = 0.05 * k[a:b] + (torch.div(pos, 64, rounding_mode="floor") * tile_step_log2 * math.log(2) / (8.0 * scale)) * w
            continue
        sg = 1.0 if s % 2 == 0 else -1.0
        q[a:b] += 6.0 * sg * uq
        k[a:b] -= 6.0 * sg * u
        if s % 2:
            v[a:b] += 50.0
        if causal:
            q[a:b] += 6.0 * wq
            k[a:b] = 0.25 * k[a:b] + (pos * min(0.1, 40.0 / (b - a)) / (6.0 * scale)) * w
    buf = torch.full((T + POISON_ROWS, (q_heads + 2 * kv_heads) * hd), float("nan"))
    buf[:T] = torch.cat([q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)], dim=1)
    buf = buf.bfloat16()
    qd, kd = q_heads * hd, kv_heads * hd
    return buf, buf[:, :qd], buf[:, qd:qd + kd], buf[:, qd + kd:], cu


def decode_inputs(lens, q_heads, kv_heads, cap, seed, poison):
    """q [B, qh*128], caches [B, cap, kvh*128] bf16; every slot [L_b, cap) of every sequence poisoned:
      - "nan": K NaN, V inf: reading a slot at all poisons the output;
      - "adversarial": finite K = 4 x the sum of the group's queries (scores ~ +45 nats) and V = 1e4, so any nonzero
        weight on a slot past the end shows;
      - "random": nothing, unit normal data past the end as well."""
    g = torch.Generator().manual_seed(seed)
    hd, G, B = 128, q_heads // kv_heads, len(lens)
    q = torch.randn(B, q_heads, hd, generator=g)
    kc = torch.randn(B, cap, kv_heads, hd, generator=g)
    vc = torch.randn(B, cap, kv_heads, hd, generator=g)
    qb = q.bfloat16().float()
    for b, L in enumerate(lens):
        if poison == "nan":
            kc[b, L:], vc[b, L:] = float("nan"), float("inf")
        elif poison == "adversarial":
            kc[b, L:] = 4.0 * qb[b].reshape(kv_heads, G, hd).sum(1) / G ** 0.5
            vc[b, L:] = 1e4
    return q.reshape(B, -1).bfloat16(), kc.reshape(B, cap, -1).bfloat16(), vc.reshape(B, cap, -1).bfloat16()


def chan_inputs(B, N, C, seed, plain=False):
    """qkv [B, N, 3C] bf16, random; q and k of the last token chunk (chan_plan) are x4, so that chunk's share of the
    Gram is visible (plain: unit normal data only)."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, N, 3 * C, generator=g)
    if plain:
        return qkv.bfloat16()
    n_chunks, tpc = chan_plan(N, C)
    t0 = (n_chunks - 1) * tpc * chan_constants()[0]
    qkv[:, t0:, :2 * C] *= 4.0
    return qkv.bfloat16()


# -------------------------------------------------------------------------------------------------------------- check
def ratio(out, ref, bound):
    """-> (max |out - ref| / bound, (row, head, dim) of it); ref / bound are [rows, heads, dim], out any layout of the
    same elements.  A non-finite output element has ratio inf."""
    o = out.detach().to(device=ref.device, dtype=torch.float64).reshape(ref.shape)
    err = (o - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isnan(r) | ~torch.isfinite(o), torch.full_like(r, float("inf")), r)
    i = int(torch.argmax(r))
    idx = tuple(int(x) for x in torch.unravel_index(torch.tensor(i), r.shape))
    return float(r.reshape(-1)[i]), idx


def check(out, ref, bound, what=""):
    """Assert |out - ref| <= bound for every element; return the largest ratio.  On failure, report the worst
    (row, head, dim) with the kernel's value, the reference and the bound there."""
    r, idx = ratio(out, ref, bound)
    if not r <= 1.0:
        o = out.detach().to(device=ref.device, dtype=torch.float64).reshape(ref.shape)
        raise AssertionError(f"{what}: |out - ref| / bound = {r:.3g} at (row, head, dim) = {idx}: out {float(o[idx]):.6g}, "
                             f"ref {float(ref[idx]):.6g}, bound {float(bound[idx]):.3g}")
    return r
