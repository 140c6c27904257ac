"""numpy models of the CUDA kernels' arithmetic (tests only).  They let the CPU suite check the
ALGORITHM the kernels implement (separable weights, window sums) against the oracle before any GPU
time is spent; the kernels themselves are checked against the oracle in the -m gpu tests."""
import math

import numpy as np

f32 = np.float32


def axis_weights(lo, hi, scale, P, n_nat, n_up):
    """model of hfre_axis_weights_kernel: -> (start, weights[len]) on the native axis."""
    start = f32(f32(lo) * f32(scale)); end = f32(f32(hi) * f32(scale))
    extent = max(f32(end - start), f32(1.0))
    binsz = f32(extent / f32(P))
    g = int(math.ceil(float(f32(extent / f32(P)))))
    A = np.zeros(n_up, dtype=np.float64)
    for p in range(P):
        for i in range(g):
            y = f32(f32(start + f32(f32(p) * binsz)) + f32(f32(f32(f32(i) + f32(0.5)) * binsz) / f32(g)))
            ok = not (y < -1.0 or y > n_up)
            if y <= 0:
                y = f32(0)
            yl = int(y)
            if yl >= n_up - 1:
                yh = yl = n_up - 1
                y = f32(yl)
            else:
                yh = yl + 1
            ly = f32(y - f32(yl)); hy = f32(f32(1) - ly)
            if ok:
                A[yl] += hy
                A[yh] += ly
    A = A / (P * g)
    if n_up == n_nat:
        return A.astype(f32)
    us = f32(f32(n_nat) / f32(n_up))
    a = np.zeros(n_nat, dtype=np.float64)
    for i in range(n_up):
        s = f32(f32(us * f32(f32(i) + f32(0.5))) - f32(0.5))
        if s < 0:
            s = f32(0)
        i0 = int(s); i1 = i0 + (1 if i0 < n_nat - 1 else 0)
        l1 = f32(s - f32(i0)); l0 = f32(f32(1) - l1)
        a[i0] += l0 * A[i]
        a[i1] += l1 * A[i]
    return a.astype(f32)


def hfre_level(feat_hwc, boxes, scale, P, up_hw):
    """out[n, c] = a^T L[c] b over a channels-last [H, W, C] level."""
    H, W, C = feat_hwc.shape
    out = np.zeros((len(boxes), C), dtype=np.float32)
    for n, (x1, y1, x2, y2) in enumerate(boxes):
        a = axis_weights(y1, y2, scale, P, H, up_hw[0])
        b = axis_weights(x1, x2, scale, P, W, up_hw[1])
        out[n] = np.einsum("r,rkc,k->c", a.astype(np.float64), feat_hwc.astype(np.float64), b.astype(np.float64))
    return out


def _bf16_round(x):
    """fp32 -> nearest-even bf16 -> fp32 (numpy)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def hfre_level_tensor_sweep(feat_hwc, boxes, scale, P, up_hw, region_rows=8, region_cols=32):
    """Model of hfre_sweep_mma_kernel: per (8 x 32)-cell region and box, the row sums over the region's columns
    use the column weights as hi + lo bf16 halves against the bf16 map (products exact, fp32 accumulation), the row
    weight a_y is applied in fp32, regions are added into the output."""
    H, W, C = feat_hwc.shape
    L = _bf16_round(feat_hwc)                      # the kernels read bf16 maps
    out = np.zeros((len(boxes), C), dtype=np.float32)
    for n, (x1, y1, x2, y2) in enumerate(boxes):
        a = axis_weights(y1, y2, scale, P, H, up_hw[0]).astype(np.float32)
        b = axis_weights(x1, x2, scale, P, W, up_hw[1]).astype(np.float32)
        b_hi = _bf16_round(b)
        b_lo = _bf16_round(b - b_hi)
        for r0 in range(0, H, region_rows):
            for c0 in range(0, W, region_cols):
                aa, rows = a[r0:r0 + region_rows], L[r0:r0 + region_rows, c0:c0 + region_cols]
                if not aa.any() or not b[c0:c0 + region_cols].any():
                    continue
                row_sum = (np.einsum("rkc,k->rc", rows, b_hi[c0:c0 + region_cols]).astype(np.float32)
                           + np.einsum("rkc,k->rc", rows, b_lo[c0:c0 + region_cols]).astype(np.float32))
                out[n] += np.einsum("r,rc->c", aa, row_sum).astype(np.float32)
    return out


# ------------------------------------------------------------------------------------------------------------ attention
# Models of the attention kernels' rounding (tests/attention_bounds.py derives the bounds they must satisfy).  Inputs are
# float32 arrays holding bf16 values.  `defect` injects one mistake a kernel could make; the CPU suite checks that each
# one breaks the bound (tests/test_attention_bounds.py).
LOG2E = 1.4426950408889634


def _fma32(a, b, c):
    """fmaf: one rounding of a * b + c."""
    return (a.astype(np.float64) * np.float64(b) + c).astype(f32)


def attn_varlen_model(q, k, v, cu, q_heads, kv_heads, hd, scale, causal, defect=None):
    """attn_tc_kernel: 128-row query tiles, each reading the 64-key tiles of [lo(first row), hi(last row)); per row a
    running maximum that is updated only once it has grown by more than kAtRescale = 8 log2 units, P = ex2(fmaf(S, sl2,
    -m)) in fp32, l summed from that fp32 P, P rounded to bf16 for P.V, out = bf16(O * (1/l)).  Reads past the packed
    rows give zeros (the tensor maps span total_rows).  -> [T, qh * hd] float32.
    defect: "past_end" (hi + 1), "neighbour" (lo - 1), "tile_last" (the last key of every 64-key tile dropped),
    "diag" (causal: the row's own key excluded), "future" (causal: one key past the row included), "gqa_mod"."""
    T = int(cu[-1])
    G = q_heads // kv_heads
    sl2 = f32(f32(scale) * f32(LOG2E))
    lo, hi = np.zeros(T, np.int64), np.zeros(T, np.int64)
    for a, b in zip(cu[:-1], cu[1:]):
        lo[a:b], hi[a:b] = a, b
    rows = np.arange(T)
    if causal:
        hi = np.minimum(hi, rows + 1)
    if defect == "past_end":
        hi = hi + 1
    elif defect == "neighbour":
        lo = np.maximum(lo - 1, 0)
    elif defect == "diag":
        hi = np.maximum(hi - 1, lo)
    elif defect == "future":
        seg_hi = np.repeat(np.asarray(cu[1:]), np.diff(cu))
        hi = np.minimum(hi + 1, seg_hi)
    kvmap = np.arange(q_heads) % kv_heads if defect == "gqa_mod" else np.arange(q_heads) // G
    kz = np.zeros((T + 64 + 1, kv_heads * hd), f32); kz[:T] = k[:T]
    vz = np.zeros_like(kz); vz[:T] = v[:T]
    out = np.zeros((T, q_heads, hd), f32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for r0 in range(0, T, 128):
            rs = slice(r0, min(T, r0 + 128))
            kb, ke = int(lo[rs].min()), int(hi[rs].max())
            nk = ke - kb
            Q = q[rs].reshape(-1, q_heads, hd).transpose(1, 0, 2)
            K = kz[kb:ke].reshape(nk, kv_heads, hd)[:, kvmap].transpose(1, 0, 2)
            V = vz[kb:ke].reshape(nk, kv_heads, hd)[:, kvmap].transpose(1, 0, 2)
            S = np.matmul(Q, K.transpose(0, 2, 1)).astype(f32)                               # [qh, R, nk]
            keys = np.arange(kb, ke)
            live = (keys[None, :] >= lo[rs, None]) & (keys[None, :] < hi[rs, None])
            if defect == "tile_last":
                live &= ((keys - kb) % 64 != 63)[None, :]
            R = live.shape[0]
            m = np.full((q_heads, R), -np.inf, f32)
            l = np.zeros((q_heads, R), f32)
            O = np.zeros((q_heads, R, hd), f32)
            for j0 in range(0, nk, 64):
                Sj = np.where(live[None, :, j0:j0 + 64], S[:, :, j0:j0 + 64], f32(-np.inf))
                m_new = np.maximum(m, (Sj.max(-1) * sl2).astype(f32))
                resc = m_new > m + f32(8.0)
                alpha = np.where(resc & np.isfinite(m), np.exp2(m - m_new), f32(1.0)).astype(f32)
                l = (l * alpha).astype(f32)
                O = (O * alpha[..., None]).astype(f32)
                m = np.where(resc, m_new, m)
                m_use = np.where(np.isinf(m), f32(0.0), m)
                P = np.exp2(_fma32(Sj, sl2, -m_use[..., None].astype(np.float64))).astype(f32)
                l = (l + P.sum(-1, dtype=f32)).astype(f32)
                O = (O + np.matmul(_bf16_round(P), V[:, j0:j0 + 64])).astype(f32)
            inv = np.where(l > 0, f32(1.0) / l, f32(0.0)).astype(f32)
            out[rs] = _bf16_round((O * inv[..., None]).astype(f32)).transpose(1, 0, 2)
    return out.reshape(T, -1)


def decode_attn_model(q, kc, vc, lens, q_heads, kv_heads, scale, n_splits, defect=None):
    """decode_attn_kernel + decode_attn_combine_kernel: the n keys of a row split into chunks of
    ((n + S - 1)/S + 15) & ~15; in a split, warp w takes the 16-key tiles t_begin + 16 w, + 64, ...; per tile
    s = fp32(S * sc), the maximum updated and O, l rescaled on every tile, P = exp2(s - m) in fp32, l from that P, P
    rounded to bf16 for P.V; the 4 warps and then the splits merged in fp32 (a -inf part weighs 0), out = bf16(num / den).
    q [B, qh*128], caches [B, cap, kvh*128] -> [B, qh*128] float32.
    defect: "past_end" (n + 1 keys), "own_key" (n - 1 keys: the row's own key dropped), "tile_last" / "chunk_last" (the
    last key of every 16-key tile / split chunk dropped), "gqa_mod", "combine_drop_last" (the last split's partial left
    out of the combine)."""
    hd, G = 128, q_heads // kv_heads
    B, cap = kc.shape[0], kc.shape[1]
    sc = f32(f32(scale) * f32(LOG2E))
    kvmap = np.arange(q_heads) % kv_heads if defect == "gqa_mod" else np.arange(q_heads) // G
    out = np.zeros((B, q_heads, hd), f32)
    with np.errstate(invalid="ignore", over="ignore"):
        for b in range(B):
            n = int(lens[b]) + (1 if defect == "past_end" else -1 if defect == "own_key" else 0)
            chunk = ((n + n_splits - 1) // n_splits + 15) & ~15
            K = kc[b].reshape(cap, kv_heads, hd)[:, kvmap].transpose(1, 0, 2)                  # [qh, cap, hd]
            V = vc[b].reshape(cap, kv_heads, hd)[:, kvmap].transpose(1, 0, 2)
            Qb = q[b].reshape(q_heads, 1, hd)
            parts = []
            for sp in range(n_splits):
                tb, te = sp * chunk, min(n, sp * chunk + chunk)
                warps = []
                for w in range(4):
                    m = np.full(q_heads, -np.inf, f32); l = np.zeros(q_heads, f32); o = np.zeros((q_heads, hd), f32)
                    for t0 in range(tb + 16 * w, te, 64):
                        idx = np.arange(t0, t0 + 16)
                        ok = idx < te
                        if defect == "tile_last":
                            ok &= idx != t0 + 15
                        elif defect == "chunk_last":
                            ok &= idx != te - 1
                        ic = np.minimum(idx, te - 1)
                        Kt = np.where(ok[None, :, None], K[:, ic], f32(0.0))
                        Vt = np.where(ok[None, :, None], V[:, ic], f32(0.0))
                        s = (np.matmul(Qb, Kt.transpose(0, 2, 1))[:, 0].astype(f32) * sc).astype(f32)
                        s = np.where(ok[None, :], s, f32(-np.inf))
                        mn = np.maximum(m, s.max(-1))
                        alpha = np.exp2(m - mn).astype(f32)
                        p = np.exp2((s - mn[:, None]).astype(f32)).astype(f32)
                        l = (l * alpha + p.sum(-1, dtype=f32)).astype(f32)
                        o = (o * alpha[:, None] + np.matmul(_bf16_round(p)[:, None, :], Vt)[:, 0]).astype(f32)
                        m = mn
                    warps.append((m, l, o))
                parts.append(_merge_parts(warps))
            if defect == "combine_drop_last":
                parts = parts[:-1]
            mm, den, num = _merge_parts(parts)
            out[b] = _bf16_round((num / den[:, None]).astype(f32))
    return out.reshape(B, -1)


def _merge_parts(parts):
    """fp32 merge of (m, l, o) partials in order, a -inf maximum weighing 0 -> (m, l, o)."""
    mm = np.max([p[0] for p in parts], axis=0)
    num = np.zeros_like(parts[0][2]); den = np.zeros_like(parts[0][1])
    for m, l, o in parts:
        f = np.where(np.isinf(m), f32(0.0), np.exp2(m - mm)).astype(f32)
        num = (num + o * f[:, None]).astype(f32)
        den = (den + l * f).astype(f32)
    return mm, den, num


def chan_attn_model(qkv, groups, n_chunks, tiles_per_chunk, tok=128, defect=None):
    """chan_gram_tc_kernel + chan_apply_tc_kernel: per token chunk an fp32 Gram q^T k over its tokens, the chunks' Grams
    summed in order, scaled by 1/sqrtf(N), softmax over c2 in fp32, the 32 weights rounded to bf16, out = bf16(v A^T) in
    fp32.  qkv [B, N, 3C] -> [B, N, C] float32.
    defect: "scale_tile_n" (the scale taken from N rounded up to the 128-token tile), "drop_last_chunk" (the last, ragged
    token chunk left out of the Gram), "transposed" (the softmax over c1: the Gram transposed)."""
    B, N, C3 = qkv.shape
    C = C3 // 3
    x = qkv.reshape(B, N, 3, groups, 32)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]                                          # [B, N, g, 32]
    Gm = np.zeros((B, groups, 32, 32), f32)
    span = tiles_per_chunk * tok
    for c in range(n_chunks - (1 if defect == "drop_last_chunk" else 0)):
        t = slice(c * span, min(N, (c + 1) * span))
        Gm = (Gm + np.einsum("btgx,btgy->bgxy", q[:, t], k[:, t]).astype(f32)).astype(f32)
    n_scale = -(-N // tok) * tok if defect == "scale_tile_n" else N
    s = (Gm * f32(f32(1.0) / np.sqrt(f32(n_scale)))).astype(f32)
    if defect == "transposed":
        s = s.transpose(0, 1, 3, 2)
    e = np.exp((s - s.max(-1, keepdims=True)).astype(f32)).astype(f32)
    a = _bf16_round((e * (f32(1.0) / e.sum(-1, dtype=f32))[..., None]).astype(f32))
    out = np.einsum("bngy,bgxy->bngx", v, a).astype(f32)
    return _bf16_round(out).reshape(B, N, C)
