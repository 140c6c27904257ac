// conv.cu -- spatial kernels of the DaViT tower and SimpleFPN over channels-last bf16 maps [B][H][W][C]:
// depth-wise 3x3 (+bias +residual), im2col feeders for the dense convolutions (which then run on the
// wgmma GEMM), 2x2 max-pool, and DaViT's channel-group attention.  All memory-bound SIMT kernels.
#include "kernels.cuh"

namespace fo1 {

// y = x + dwconv3x3(x) + bias   (PreNorm(None, DepthWiseConv2d), modeling_davit.py:29-48, 72-99)
// w9: [9][C] (tap-major, repacked from [C][1][3][3]); one thread = 8 channels of one pixel.
__global__ void __launch_bounds__(256) dwconv3x3_res_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w9,
                                                            const bf16* __restrict__ bias, bf16* __restrict__ y, int B, int H,
                                                            int W, int C) {
  const int cv = C >> 3;
  const long long total = (long long)B * H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long p = i / cv;
    const int px = (int)(p % W); p /= W;
    const int py = (int)(p % H);
    const int b = (int)(p / H);
    float acc[8];
    {
      const uint4 bv = *reinterpret_cast<const uint4*>(bias + c8 * 8);
      acc[0] = bf16_lo(bv.x); acc[1] = bf16_hi(bv.x); acc[2] = bf16_lo(bv.y); acc[3] = bf16_hi(bv.y);
      acc[4] = bf16_lo(bv.z); acc[5] = bf16_hi(bv.z); acc[6] = bf16_lo(bv.w); acc[7] = bf16_hi(bv.w);
    }
    float center[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const int yy = py + dy;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int xx = px + dx;
        if (xx < 0 || xx >= W) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * C + c8 * 8);
        const uint4 wv = *reinterpret_cast<const uint4*>(w9 + ((dy + 1) * 3 + (dx + 1)) * C + c8 * 8);
        const float xv[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y), bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
        const float ww[8] = {bf16_lo(wv.x), bf16_hi(wv.x), bf16_lo(wv.y), bf16_hi(wv.y), bf16_lo(wv.z), bf16_hi(wv.z), bf16_lo(wv.w), bf16_hi(wv.w)};
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv[j], ww[j], acc[j]);
        if (dy == 0 && dx == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) center[j] = xv[j];
        }
      }
    }
    // the conv output is a bf16 tensor in the reference; the residual add happens on bf16 values
    uint4 o;
    o.x = pack_bf16(center[0] + __bfloat162float(__float2bfloat16_rn(acc[0])), center[1] + __bfloat162float(__float2bfloat16_rn(acc[1])));
    o.y = pack_bf16(center[2] + __bfloat162float(__float2bfloat16_rn(acc[2])), center[3] + __bfloat162float(__float2bfloat16_rn(acc[3])));
    o.z = pack_bf16(center[4] + __bfloat162float(__float2bfloat16_rn(acc[4])), center[5] + __bfloat162float(__float2bfloat16_rn(acc[5])));
    o.w = pack_bf16(center[6] + __bfloat162float(__float2bfloat16_rn(acc[6])), center[7] + __bfloat162float(__float2bfloat16_rn(acc[7])));
    *reinterpret_cast<uint4*>(y + (((long long)b * H + py) * W + px) * C + c8 * 8) = o;
  }
}

// Same operator, HBM-bound layout (DaViT stages: C = 256 .. 2048, a multiple of 256).  A block is 8 adjacent pixels x 32 channel
// vectors (one warp = the 512 contiguous bytes of one pixel) and walks a strip of R rows downwards with the 3 x 3 window of every
// thread in registers: three 16-byte loads per output instead of nine, the horizontal neighbours are loaded by the neighbouring
// warps of the same block in the same iteration (L1 hits), so DRAM sees each input row once per strip (+ the 2 halo rows).
// Arithmetic identical to dwconv3x3_res_kernel (bias first, taps in (dy, dx) order, zero padding contributes exact zeros).
constexpr int kDwTx = 8;
__global__ void __launch_bounds__(256, 2) dwconv3x3_res_strip_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w9,
                                                                     const bf16* __restrict__ bias, bf16* __restrict__ y, int H, int W,
                                                                     int C, int R, int strips_x, int strips_y, int cblocks) {
  __shared__ uint4 s_w[9][32];     // the block's 9 x 256 weights (the eight warps read the same 512 B per tap)
  int bid = blockIdx.x;
  const int cb = bid % cblocks; bid /= cblocks;
  const int sx = bid % strips_x; bid /= strips_x;
  const int sy = bid % strips_y;
  const int b = bid / strips_y;
  const int lane = threadIdx.x & 31;
  const int c8 = cb * 32 + lane;
  const int px = sx * kDwTx + (threadIdx.x >> 5);
  const int y0 = sy * R, y1 = min(H, y0 + R);
  const bool active = px < W;
  for (int i = threadIdx.x; i < 9 * 32; i += 256) s_w[i >> 5][i & 31] = *reinterpret_cast<const uint4*>(w9 + (long long)(i >> 5) * C + (cb * 32 + (i & 31)) * 8);
  const uint4 bv = *reinterpret_cast<const uint4*>(bias + c8 * 8);
  const bf16* xb = x + (long long)b * H * W * C + c8 * 8;
  bf16* yb = y + (long long)b * H * W * C + c8 * 8;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  auto load_row = [&](int yy, uint4 (&r)[3]) {
    if (yy < 0 || yy >= H || !active) { r[0] = r[1] = r[2] = zero; return; }
    const bf16* row = xb + (long long)yy * W * C;
    r[0] = px > 0 ? *reinterpret_cast<const uint4*>(row + (long long)(px - 1) * C) : zero;
    r[1] = *reinterpret_cast<const uint4*>(row + (long long)px * C);
    r[2] = px + 1 < W ? *reinterpret_cast<const uint4*>(row + (long long)(px + 1) * C) : zero;
  };
  uint4 win[3][3], nxt[3];
  load_row(y0 - 1, win[0]);
  load_row(y0, win[1]);
  load_row(y0 + 1, win[2]);
  __syncthreads();
  for (int py = y0; py < y1; ++py) {
    load_row(py + 2, nxt);         // one row ahead of the window: its latency hides behind this row's arithmetic
    float acc[8] = {bf16_lo(bv.x), bf16_hi(bv.x), bf16_lo(bv.y), bf16_hi(bv.y), bf16_lo(bv.z), bf16_hi(bv.z), bf16_lo(bv.w), bf16_hi(bv.w)};
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const uint4 v = win[dy][dx], w = s_w[dy * 3 + dx][lane];
        acc[0] = fmaf(bf16_lo(v.x), bf16_lo(w.x), acc[0]); acc[1] = fmaf(bf16_hi(v.x), bf16_hi(w.x), acc[1]);
        acc[2] = fmaf(bf16_lo(v.y), bf16_lo(w.y), acc[2]); acc[3] = fmaf(bf16_hi(v.y), bf16_hi(w.y), acc[3]);
        acc[4] = fmaf(bf16_lo(v.z), bf16_lo(w.z), acc[4]); acc[5] = fmaf(bf16_hi(v.z), bf16_hi(w.z), acc[5]);
        acc[6] = fmaf(bf16_lo(v.w), bf16_lo(w.w), acc[6]); acc[7] = fmaf(bf16_hi(v.w), bf16_hi(w.w), acc[7]);
      }
    if (active) {
      const uint4 c = win[1][1];
      uint4 o;   // the conv output is a bf16 tensor in the reference; the residual add happens on bf16 values
      o.x = pack_bf16(bf16_lo(c.x) + __bfloat162float(__float2bfloat16_rn(acc[0])), bf16_hi(c.x) + __bfloat162float(__float2bfloat16_rn(acc[1])));
      o.y = pack_bf16(bf16_lo(c.y) + __bfloat162float(__float2bfloat16_rn(acc[2])), bf16_hi(c.y) + __bfloat162float(__float2bfloat16_rn(acc[3])));
      o.z = pack_bf16(bf16_lo(c.z) + __bfloat162float(__float2bfloat16_rn(acc[4])), bf16_hi(c.z) + __bfloat162float(__float2bfloat16_rn(acc[5])));
      o.w = pack_bf16(bf16_lo(c.w) + __bfloat162float(__float2bfloat16_rn(acc[6])), bf16_hi(c.w) + __bfloat162float(__float2bfloat16_rn(acc[7])));
      *reinterpret_cast<uint4*>(yb + ((long long)py * W + px) * C) = o;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { win[0][k] = win[1][k]; win[1][k] = win[2][k]; win[2][k] = nxt[k]; }
  }
}

// im2col for a 3x3 / pad 1 / stride s convolution over NHWC: dst[(b,oy,ox)][(ky,kx,c)]
__global__ void __launch_bounds__(256) im2col3x3_kernel(const bf16* __restrict__ x, bf16* __restrict__ col, int B, int H, int W,
                                                        int C, int Ho, int Wo, int stride) {
  const int cv = C >> 3;
  const long long total = (long long)B * Ho * Wo * 9 * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long p = i / cv;
    const int tap = (int)(p % 9); p /= 9;
    const int ox = (int)(p % Wo); p /= Wo;
    const int oy = (int)(p % Ho);
    const int b = (int)(p / Ho);
    const int yy = oy * stride - 1 + tap / 3, xx = ox * stride - 1 + tap % 3;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * C + c8 * 8);
    *reinterpret_cast<uint4*>(col + ((((long long)b * Ho + oy) * Wo + ox) * 9 + tap) * C + c8 * 8) = v;
  }
}

// DaViT stem: 7x7 / stride 4 / pad 3 over a fp32 CHW image -> bf16 rows [(oy,ox)][(c,ky,kx) padded to kpad]
__global__ void __launch_bounds__(256) im2col_stem_kernel(const float* __restrict__ img, bf16* __restrict__ col, int H, int W,
                                                          int Ho, int Wo, int kpad) {
  const long long total = (long long)Ho * Wo * kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % kpad);
    const long long p = i / kpad;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    float v = 0.f;
    if (k < 147) {
      const int c = k / 49, ky = (k % 49) / 7, kx = k % 7;
      const int yy = oy * 4 - 3 + ky, xx = ox * 4 - 3 + kx;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = img[((long long)c * H + yy) * W + xx];
    }
    col[i] = __float2bfloat16_rn(v);
  }
}

__global__ void __launch_bounds__(256) maxpool2x2_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2, cv = C >> 3;
  const long long total = (long long)B * Ho * Wo * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long p = i / cv;
    const int ox = (int)(p % Wo); p /= Wo;
    const int oy = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + oy * 2 + (d >> 1)) * W + ox * 2 + (d & 1)) * C + c8 * 8);
      const float xv[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y), bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], xv[j]);
    }
    uint4 o;
    o.x = pack_bf16(m[0], m[1]); o.y = pack_bf16(m[2], m[3]); o.z = pack_bf16(m[4], m[5]); o.w = pack_bf16(m[6], m[7]);
    *reinterpret_cast<uint4*>(y + (((long long)b * Ho + oy) * Wo + ox) * C + c8 * 8) = o;
  }
}

// DaViT window attention bookkeeping (modeling_davit.py:246-280): zero-pad H, W up to multiples of the
// window AFTER the LayerNorm, partition into ws x ws windows (rows of one window contiguous) ...
__global__ void __launch_bounds__(256) window_partition_kernel(const bf16* __restrict__ x, bf16* __restrict__ dst, int B, int H, int W,
                                                               int C, int ws, int nwh, int nww) {
  const int cv = C >> 3;
  const long long total = (long long)B * nwh * nww * ws * ws * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long r = i / cv;
    const int ix = (int)(r % ws); r /= ws;
    const int iy = (int)(r % ws); r /= ws;
    const int wx = (int)(r % nww); r /= nww;
    const int wy = (int)(r % nwh);
    const int b = (int)(r / nwh);
    const int y = wy * ws + iy, xx = wx * ws + ix;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (y < H && xx < W) v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + y) * W + xx) * C + c8 * 8);
    *reinterpret_cast<uint4*>(dst + (i / cv) * C + c8 * 8) = v;
  }
}
// ... and the inverse, cropped, fused with the residual add: y[b][yy][xx] = x[b][yy][xx] + p[window row]
__global__ void __launch_bounds__(256) window_reverse_add_kernel(const bf16* __restrict__ x, const bf16* __restrict__ p,
                                                                 bf16* __restrict__ y, int B, int H, int W, int C, int ws, int nwh, int nww) {
  const int cv = C >> 3;
  const long long total = (long long)B * H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long r = i / cv;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int b = (int)(r / H);
    const long long row = ((((long long)b * nwh + yy / ws) * nww + xx / ws) * ws + yy % ws) * ws + xx % ws;
    const uint4 a = *reinterpret_cast<const uint4*>(x + (i / cv) * C + c8 * 8);
    const uint4 q = *reinterpret_cast<const uint4*>(p + row * C + c8 * 8);
    uint4 o;
    o.x = pack_bf16(bf16_lo(a.x) + bf16_lo(q.x), bf16_hi(a.x) + bf16_hi(q.x));
    o.y = pack_bf16(bf16_lo(a.y) + bf16_lo(q.y), bf16_hi(a.y) + bf16_hi(q.y));
    o.z = pack_bf16(bf16_lo(a.z) + bf16_lo(q.z), bf16_hi(a.z) + bf16_hi(q.z));
    o.w = pack_bf16(bf16_lo(a.w) + bf16_lo(q.w), bf16_hi(a.w) + bf16_hi(q.w));
    *reinterpret_cast<uint4*>(y + (i / cv) * C + c8 * 8) = o;
  }
}

static inline int grid_for(long long items) {
  long long b = (items + 255) / 256;
  const long long cap = device_sm_count() * 32LL;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

int dwconv3x3_residual(const bf16* x, const bf16* w9, const bf16* bias, bf16* y, int B, int H, int W, int C, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0, "dwconv3x3: C=%d must be a multiple of 8", C);
  if ((long long)B * H * W == 0) return FO1_OK;
  if (C % 256 == 0 && getenv("FO1_DWCONV_SIMPLE") == nullptr) {
    const int R = H >= 48 ? 16 : (H >= 24 ? 12 : H);
    const int strips_x = ceil_div(W, kDwTx), strips_y = ceil_div(H, R), cblocks = C / 256;
    const long long blocks = (long long)B * strips_y * strips_x * cblocks;
    FO1_CHECK_ARG(blocks < (1LL << 31), "dwconv3x3: too many blocks");
    dwconv3x3_res_strip_kernel<<<(unsigned)blocks, 256, 0, s>>>(x, w9, bias, y, H, W, C, R, strips_x, strips_y, cblocks);
    FO1_LAUNCH_CHECK();
    return FO1_OK;
  }
  dwconv3x3_res_kernel<<<grid_for((long long)B * H * W * (C / 8)), 256, 0, s>>>(x, w9, bias, y, B, H, W, C);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
int im2col3x3(const bf16* x, bf16* col, int B, int H, int W, int C, int stride, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0 && (stride == 1 || stride == 2), "im2col3x3: C=%d stride=%d", C, stride);
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  if ((long long)B * Ho * Wo == 0) return FO1_OK;
  im2col3x3_kernel<<<grid_for((long long)B * Ho * Wo * 9 * (C / 8)), 256, 0, s>>>(x, col, B, H, W, C, Ho, Wo, stride);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
int im2col_stem(const float* img, bf16* col, int H, int W, int kpad, cudaStream_t s) {
  const int Ho = (H + 6 - 7) / 4 + 1, Wo = (W + 6 - 7) / 4 + 1;
  FO1_CHECK_ARG(kpad >= 147 && kpad % 8 == 0, "im2col_stem: kpad=%d", kpad);
  im2col_stem_kernel<<<grid_for((long long)Ho * Wo * kpad), 256, 0, s>>>(img, col, H, W, Ho, Wo, kpad);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
int maxpool2x2(const bf16* x, bf16* y, int B, int H, int W, int C, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0, "maxpool2x2: C=%d", C);
  if ((long long)B * (H / 2) * (W / 2) == 0) return FO1_OK;
  maxpool2x2_kernel<<<grid_for((long long)B * (H / 2) * (W / 2) * (C / 8)), 256, 0, s>>>(x, y, B, H, W, C);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
// qkv: [B][N][3C] (q | k | v, each group-major with 32 channels per group); gram: [B][groups][32][32] fp32 scratch
int window_partition(const bf16* x, bf16* dst, int B, int H, int W, int C, int ws, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0 && ws > 0, "window_partition: C=%d ws=%d", C, ws);
  const int nwh = ceil_div(H, ws), nww = ceil_div(W, ws);
  if ((long long)B * H * W == 0) return FO1_OK;
  window_partition_kernel<<<grid_for((long long)B * nwh * nww * ws * ws * (C / 8)), 256, 0, s>>>(x, dst, B, H, W, C, ws, nwh, nww);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
int window_reverse_add(const bf16* x, const bf16* p, bf16* y, int B, int H, int W, int C, int ws, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0 && ws > 0, "window_reverse_add: C=%d ws=%d", C, ws);
  const int nwh = ceil_div(H, ws), nww = ceil_div(W, ws);
  if ((long long)B * H * W == 0) return FO1_OK;
  window_reverse_add_kernel<<<grid_for((long long)B * H * W * (C / 8)), 256, 0, s>>>(x, p, y, B, H, W, C, ws, nwh, nww);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1

namespace fo1 {
// ConvTranspose2d(k=2, s=2) computed as a GEMM to [pixels][(dy,dx,co)], then this 2x pixel shuffle
__global__ void __launch_bounds__(256) pixel_shuffle2x_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int B, int H, int W, int C) {
  const int cv = C >> 3;
  const long long total = (long long)B * H * W * 4 * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long r = i / cv;
    const int d = (int)(r % 4); r /= 4;
    const int x = (int)(r % W); r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    const uint4 v = *reinterpret_cast<const uint4*>(src + (i / cv) * C + c8 * 8);
    *reinterpret_cast<uint4*>(dst + ((((long long)b * 2 * H + 2 * y + (d >> 1)) * 2 * W) + 2 * x + (d & 1)) * C + c8 * 8) = v;
  }
}
int pixel_shuffle2x(const bf16* src, bf16* dst, int B, int H, int W, int C, cudaStream_t s) {
  FO1_CHECK_ARG(C % 8 == 0, "pixel_shuffle2x: C=%d", C);
  if ((long long)B * H * W == 0) return FO1_OK;
  long long items = (long long)B * H * W * 4 * (C / 8);
  long long blocks = (items + 255) / 256;
  if (blocks > device_sm_count() * 32LL) blocks = device_sm_count() * 32LL;
  pixel_shuffle2x_kernel<<<(int)blocks, 256, 0, s>>>(src, dst, B, H, W, C);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}
}  // namespace fo1

extern "C" int fo1_dwconv3x3_residual(const void* x, const void* w9, const void* bias, void* y, int32_t n_images, int32_t height, int32_t width,
                                      int32_t channels, void* stream) {
  using namespace fo1;
  FO1_CHECK_ARG(x && w9 && bias && y && x != y && n_images >= 0 && height >= 0 && width >= 0 && channels > 0, "fo1_dwconv3x3_residual: bad argument");
  FO1_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(w9) | reinterpret_cast<uintptr_t>(bias)) & 15) == 0,
                "fo1_dwconv3x3_residual: pointers must be 16-byte aligned");
  return dwconv3x3_residual(static_cast<const bf16*>(x), static_cast<const bf16*>(w9), static_cast<const bf16*>(bias), static_cast<bf16*>(y), n_images,
                            height, width, channels, static_cast<cudaStream_t>(stream));
}
