// misc.cu -- data-movement kernels (row gathers/scatters, casts, simple elementwise); all memory-bound.
#include "kernels.cuh"

namespace fo1 {

// dst[r][:] = bf16(src[row_idx ? row_idx[r] : r][:]); cols % 4 == 0
__global__ void cast_gather_rows_kernel(const float* __restrict__ src, long long lds, const int* __restrict__ idx,
                                        bf16* __restrict__ dst, long long ldd, int rows, int cols) {
  const int r = blockIdx.x;  // rows on grid.x: a packed batch has > 65535 token rows
  const float* sp = src + (long long)(idx ? idx[r] : r) * lds;
  bf16* dp = dst + (long long)r * ldd;
  for (int c = threadIdx.x * 4; c < cols; c += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(sp + c);
    uint2 o;
    o.x = pack_bf16(v.x, v.y);
    o.y = pack_bf16(v.z, v.w);
    *reinterpret_cast<uint2*>(dp + c) = o;
  }
}

// GATHER: dst[r] = src[idx[r]]; SCATTER: dst[idx[r]] = src[r]; cols % 8 == 0
template <bool SCATTER>
__global__ void move_rows_kernel(const bf16* __restrict__ src, long long lds, const int* __restrict__ idx, bf16* __restrict__ dst,
                                 long long ldd, int rows, int cols) {
  const int r = blockIdx.x;
  const long long sr = SCATTER ? r : idx[r], dr = SCATTER ? idx[r] : r;
  const bf16* sp = src + sr * lds;
  bf16* dp = dst + dr * ldd;
  for (int c = threadIdx.x * 8; c < cols; c += blockDim.x * 8)
    *reinterpret_cast<uint4*>(dp + c) = *reinterpret_cast<const uint4*>(sp + c);
}

__global__ void add_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ o, long long n) {
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += (long long)gridDim.x * blockDim.x * 2) {
    if (i + 1 < n) {
      const uint32_t x = *reinterpret_cast<const uint32_t*>(a + i), y = *reinterpret_cast<const uint32_t*>(b + i);
      *reinterpret_cast<uint32_t*>(o + i) = pack_bf16(bf16_lo(x) + bf16_lo(y), bf16_hi(x) + bf16_hi(y));
    } else {
      o[i] = __float2bfloat16_rn(__bfloat162float(a[i]) + __bfloat162float(b[i]));
    }
  }
}

__global__ void gelu_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(gelu_erf(__bfloat162float(x[i])));
}

static inline int grid1d(long long work_items, int per_block) {
  long long b = (work_items + per_block - 1) / per_block;
  const long long cap = device_sm_count() * 32LL;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

int cast_gather_rows_f32_bf16(const float* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols,
                              cudaStream_t s) {
  FO1_CHECK_ARG(cols % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0, "cast_gather_rows: cols/pitches must be multiples of 4");
  if (rows == 0) return FO1_OK;
  cast_gather_rows_kernel<<<rows, 256, 0, s>>>(src, lds, row_idx, dst, ldd, rows, cols);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int gather_rows_bf16(const bf16* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols, cudaStream_t s) {
  FO1_CHECK_ARG(cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0, "gather_rows: cols/pitches must be multiples of 8");
  if (rows == 0) return FO1_OK;
  move_rows_kernel<false><<<rows, cols / 8 < 256 ? ((cols / 8 + 31) / 32) * 32 : 256, 0, s>>>(src, lds, row_idx, dst, ldd, rows, cols);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int scatter_rows_bf16(const bf16* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols, cudaStream_t s) {
  FO1_CHECK_ARG(cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0, "scatter_rows: cols/pitches must be multiples of 8");
  if (rows == 0) return FO1_OK;
  move_rows_kernel<true><<<rows, cols / 8 < 256 ? ((cols / 8 + 31) / 32) * 32 : 256, 0, s>>>(src, lds, row_idx, dst, ldd, rows, cols);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int add_bf16(const bf16* a, const bf16* b, bf16* out, long long n, cudaStream_t s) {
  if (n == 0) return FO1_OK;
  add_kernel<<<grid1d(n / 2 + 1, 256), 256, 0, s>>>(a, b, out, n);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int gelu_bf16(const bf16* x, bf16* y, long long n, cudaStream_t s) {
  if (n == 0) return FO1_OK;
  gelu_kernel<<<grid1d(n, 256), 256, 0, s>>>(x, y, n);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1
