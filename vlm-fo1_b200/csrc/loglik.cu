// loglik.cu -- the second half of the log-likelihood head: the LM-head GEMM's log-likelihood epilogue (gemm_wgmma.cu, loglik_frag)
// leaves per row one partial per 128-column tile, (m_t, index of the first maximum, s_t = sum over the tile of exp(x - m_t)); one warp
// per row merges them here into
//   lse = M* + log sum_t s_t exp(m_t - M*),   M* = max_t m_t,
// the lowest-index maximum of the row (greedy), and logprob = x[target] - lse.  Nothing vocabulary-sized is ever written.
#include <cfloat>

#include "kernels.cuh"

namespace fo1 {

// lane l takes partials l, l + 32, ... in ascending order, then the butterfly sums the lanes (every lane ends with the same bits): the
// order is a function of n_parts alone, so a row's results never depend on the other rows of the call
__global__ void loglik_merge_kernel(const float4* __restrict__ part, int n_parts, int M, const int* __restrict__ target,
                                    const float* __restrict__ x_tgt, const int* __restrict__ out_row, float* logprobs, int* greedy,
                                    float* lse_out, float* x_out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* p = part + (long long)row * n_parts;
  float mx = -INFINITY;
  int ix = 0x7fffffff;
  for (int t = lane; t < n_parts; t += 32) {
    const float4 v = p[t];
    const int i = __float_as_int(v.z);
    if (v.x > mx || (v.x == mx && i < ix)) { mx = v.x; ix = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, ix, o);
    if (om > mx || (om == mx && oi < ix)) { mx = om; ix = oi; }
  }
  float s = 0.f;
  for (int t = lane; t < n_parts; t += 32) {
    const float4 v = p[t];
    s += v.y * expf(v.x - mx);
  }
  s = warp_sum(s);
  if (lane != 0) return;
  const float lse = mx + logf(s);
  const float xt = x_tgt[row];
  const int r = out_row[row];
  logprobs[r] = xt - lse;
  if (greedy) greedy[r] = ix == target[row] ? 1 : 0;
  if (lse_out) lse_out[row] = lse;
  if (x_out) x_out[row] = xt;
}

int loglik_merge(const float4* part, int n_parts, int M, const int* target, const float* x_tgt, const int* out_row, float* logprobs,
                 int* greedy, float* lse, float* x_out, cudaStream_t s) {
  if (M == 0) return FO1_OK;
  constexpr int kWarps = 8;
  loglik_merge_kernel<<<ceil_div(M, kWarps), 32 * kWarps, 0, s>>>(part, n_parts, M, target, x_tgt, out_row, logprobs, greedy, lse, x_out);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

// one thread per sequence: its rows in ascending order, in fp64
__global__ void loglik_seq_sum_kernel(const float* __restrict__ logprobs, const int* __restrict__ off, int n_seqs, double* out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_seqs) return;
  double acc = 0.0;
  for (int r = off[b]; r < off[b + 1]; ++r) acc += (double)logprobs[r];
  out[b] = acc;
}

int loglik_seq_sum(const float* logprobs, const int* off, int n_seqs, double* seq_logprob, cudaStream_t s) {
  loglik_seq_sum_kernel<<<ceil_div(n_seqs, 128), 128, 0, s>>>(logprobs, off, n_seqs, seq_logprob);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1
