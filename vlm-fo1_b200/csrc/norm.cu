// norm.cu -- row normalisations (memory-bound: one pass, fp32 statistics, 16-byte vector I/O).
#include "kernels.cuh"

namespace fo1 {

// one warp per row; each lane walks the row in 8-element (16 B) vectors, keeping them in registers
template <int MAXV, bool RMS>
__global__ void __launch_bounds__(256) rownorm_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ gamma,
                                                      const bf16* __restrict__ beta, bf16* __restrict__ y, long long ldy,
                                                      int rows, int cols, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const bf16* xr = x + (long long)row * ldx;
  bf16* yr = y + (long long)row * ldy;
  const int nvec = cols >> 3;
  uint4 v[MAXV];
  float sum = 0.f, sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      v[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
      const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = bf16_lo(u[j]), b = bf16_hi(u[j]);
        sum += a + b;
        sq += a * a + b * b;
      }
    }
  }
  sum = warp_sum(sum);
  sq = warp_sum(sq);
  const float inv_n = 1.0f / (float)cols;
  float mean = 0.f, rstd;
  if (RMS) {
    rstd = rsqrtf(sq * inv_n + eps);
  } else {
    mean = sum * inv_n;
    float var = 0.f;  // two-pass variance on the register copy (no cancellation)
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a = bf16_lo(u[j]) - mean, b = bf16_hi(u[j]) - mean;
          var += a * a + b * b;
        }
      }
    }
    var = warp_sum(var);
    rstd = rsqrtf(var * inv_n + eps);
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
      uint4 g = make_uint4(0x3f803f80u, 0x3f803f80u, 0x3f803f80u, 0x3f803f80u), bt = make_uint4(0, 0, 0, 0);
      if (gamma) g = *reinterpret_cast<const uint4*>(gamma + vi * 8);
      if (beta) bt = *reinterpret_cast<const uint4*>(beta + vi * 8);
      const uint32_t gu[4] = {g.x, g.y, g.z, g.w}, bu[4] = {bt.x, bt.y, bt.z, bt.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = (bf16_lo(u[j]) - mean) * rstd, b = (bf16_hi(u[j]) - mean) * rstd;
        if (RMS) {  // Qwen2RMSNorm rounds the normalised value to bf16 before the gain (:139-140)
          a = __bfloat162float(__float2bfloat16_rn(a));
          b = __bfloat162float(__float2bfloat16_rn(b));
        }
        a = a * bf16_lo(gu[j]) + bf16_lo(bu[j]);
        b = b * bf16_hi(gu[j]) + bf16_hi(bu[j]);
        o[j] = pack_bf16(a, b);
      }
      *reinterpret_cast<uint4*>(yr + vi * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// few rows (the decode step: one row per sequence): one BLOCK per row so a single 16-byte load per thread covers the
// row and the whole GPU shares the work instead of rows/8 SMs.  Same arithmetic as rownorm_kernel.
template <int MAXV, bool RMS>
__global__ void __launch_bounds__(256) rownorm_block_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ gamma,
                                                            const bf16* __restrict__ beta, bf16* __restrict__ y, long long ldy,
                                                            int cols, float eps) {
  __shared__ float red[2][8];
  griddep_launch();
  griddep_wait();
  const bf16* xr = x + (long long)blockIdx.x * ldx;
  bf16* yr = y + (long long)blockIdx.x * ldy;
  const int nvec = cols >> 3, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint4 v[MAXV], g[MAXV], bt[MAXV];
  float sum = 0.f, sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = tid + i * 256;
    g[i] = make_uint4(0x3f803f80u, 0x3f803f80u, 0x3f803f80u, 0x3f803f80u);
    bt[i] = make_uint4(0, 0, 0, 0);
    if (vi < nvec) {
      v[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
      if (gamma) g[i] = *reinterpret_cast<const uint4*>(gamma + vi * 8);
      if (beta) bt[i] = *reinterpret_cast<const uint4*>(beta + vi * 8);
      const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = bf16_lo(u[j]), b = bf16_hi(u[j]);
        sum += a + b;
        sq += a * a + b * b;
      }
    }
  }
  auto block_sum2 = [&](float& a, float& b) {
    a = warp_sum(a); b = warp_sum(b);
    __syncthreads();
    if (lane == 0) { red[0][warp] = a; red[1][warp] = b; }
    __syncthreads();
    a = 0.f; b = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { a += red[0][k]; b += red[1][k]; }
  };
  block_sum2(sum, sq);
  const float inv_n = 1.0f / (float)cols;
  float mean = 0.f, rstd;
  if (RMS) {
    rstd = rsqrtf(sq * inv_n + eps);
  } else {
    mean = sum * inv_n;
    float var = 0.f, dummy = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (tid + i * 256 < nvec) {
        const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a = bf16_lo(u[j]) - mean, b = bf16_hi(u[j]) - mean;
          var += a * a + b * b;
        }
      }
    }
    block_sum2(var, dummy);
    rstd = rsqrtf(var * inv_n + eps);
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = tid + i * 256;
    if (vi < nvec) {
      const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
      const uint32_t gu[4] = {g[i].x, g[i].y, g[i].z, g[i].w}, bu[4] = {bt[i].x, bt[i].y, bt[i].z, bt[i].w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = (bf16_lo(u[j]) - mean) * rstd, b = (bf16_hi(u[j]) - mean) * rstd;
        if (RMS) {
          a = __bfloat162float(__float2bfloat16_rn(a));
          b = __bfloat162float(__float2bfloat16_rn(b));
        }
        a = a * bf16_lo(gu[j]) + bf16_lo(bu[j]);
        b = b * bf16_hi(gu[j]) + bf16_hi(bu[j]);
        o[j] = pack_bf16(a, b);
      }
      *reinterpret_cast<uint4*>(yr + vi * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

template <bool RMS>
static int launch_rownorm(const bf16* x, long long ldx, const bf16* g, const bf16* b, bf16* y, long long ldy, int rows, int cols,
                          float eps, NormKernel kernel, cudaStream_t s) {
  FO1_CHECK_ARG(cols % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "rownorm: cols/pitches must be multiples of 8 (cols=%d)", cols);
  FO1_CHECK_ARG(cols <= 8 * 32 * 32, "rownorm: cols=%d too large", cols);
  FO1_CHECK_ARG(kernel == NORM_WARP || (kernel == NORM_BLOCK && cols <= kNormBlockMaxCols), "rownorm: kernel %d unsupported at cols=%d",
                (int)kernel, cols);
  if (rows == 0) return FO1_OK;
  const int nvec = cols / 8;
  if (kernel == NORM_BLOCK) {
    if (nvec <= 256) launch_k(rownorm_block_kernel<1, RMS>, dim3(rows), dim3(256), 0, s, x, ldx, g, b, y, ldy, cols, eps);
    else launch_k(rownorm_block_kernel<2, RMS>, dim3(rows), dim3(256), 0, s, x, ldx, g, b, y, ldy, cols, eps);
    FO1_LAUNCH_CHECK();
    return FO1_OK;
  }
  const int maxv = ceil_div(nvec, 32);
  dim3 grid(ceil_div(rows, 8));
#define FO1_RN(MV)                                                                              \
  if (maxv <= MV) {                                                                             \
    rownorm_kernel<MV, RMS><<<grid, 256, 0, s>>>(x, ldx, g, b, y, ldy, rows, cols, eps);        \
    FO1_LAUNCH_CHECK();                                                                         \
    return FO1_OK;                                                                              \
  }
  FO1_RN(1) FO1_RN(2) FO1_RN(4) FO1_RN(5) FO1_RN(8) FO1_RN(16) FO1_RN(32)
#undef FO1_RN
  return FO1_ERR_UNSUPPORTED;
}

int rmsnorm(const bf16* x, long long ldx, const bf16* w, bf16* y, long long ldy, int rows, int cols, float eps, NormKernel kernel,
            cudaStream_t s) {
  return launch_rownorm<true>(x, ldx, w, nullptr, y, ldy, rows, cols, eps, kernel, s);
}
int layernorm(const bf16* x, long long ldx, const bf16* gamma, const bf16* beta, bf16* y, long long ldy, int rows, int cols,
              float eps, NormKernel kernel, cudaStream_t s) {
  return launch_rownorm<false>(x, ldx, gamma, beta, y, ldy, rows, cols, eps, kernel, s);
}

}  // namespace fo1

extern "C" int fo1_row_norm(const void* x, int64_t ldx, const void* gamma, const void* beta, void* y, int64_t ldy, int32_t rows, int32_t cols,
                            float eps, int32_t rms, int32_t kernel, void* stream) {
  using namespace fo1;
  FO1_CHECK_ARG(x && y && rows >= 0 && cols > 0 && ldx >= cols && ldy >= cols && (kernel == NORM_WARP || kernel == NORM_BLOCK),
                "fo1_row_norm: bad argument");
  FO1_CHECK_ARG(!rms || beta == nullptr, "fo1_row_norm: RMSNorm takes no beta");
  FO1_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(gamma) |
                  reinterpret_cast<uintptr_t>(beta)) & 15) == 0,
                "fo1_row_norm: pointers must be 16-byte aligned");
  const bf16 *xb = static_cast<const bf16*>(x), *g = static_cast<const bf16*>(gamma), *b = static_cast<const bf16*>(beta);
  const NormKernel k = static_cast<NormKernel>(kernel);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return rms ? rmsnorm(xb, ldx, g, static_cast<bf16*>(y), ldy, rows, cols, eps, k, s)
             : layernorm(xb, ldx, g, b, static_cast<bf16*>(y), ldy, rows, cols, eps, k, s);
}
