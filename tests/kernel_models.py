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
