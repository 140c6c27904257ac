// sampling.cu -- the standalone sampling kernel over [n_rows][ld] fp32 logits (one CTA per row) and its C ABI.  The row
// routine (sampling.cuh) is the one the two decode paths run.
#include <cmath>
#include <vector>

#include "sampling.cuh"

namespace fo1 {

constexpr int kSampleThreads = 1024;

__global__ void __launch_bounds__(kSampleThreads) sample_rows_kernel(const float* __restrict__ logits, long long ld, int V,
                                                                     const SampleRowParams* __restrict__ prm, const int* __restrict__ step,
                                                                     int step_stride, int* __restrict__ out) {
  griddep_launch();
  griddep_wait();
  __shared__ SampleSmem<kSampleThreads> sm;
  const int r = blockIdx.x;
  const SampleRowParams p = prm[r];
  const int tok = sample_row<kSampleThreads>(logits + (long long)r * ld, V, p, __ldcg(step + (long long)r * step_stride), sm);
  if (threadIdx.x == 0) out[r] = tok;
}

int sampling_check(const fo1_sampling_desc* sp, int n, const char* fn) {
  FO1_CHECK_ARG(n > 0, "%s: n_rows %d must be positive", fn, n);
  FO1_CHECK_ARG(sp != nullptr && sp->temperature && sp->top_p && sp->top_k && sp->seed, "%s: null sampling parameter array", fn);
  for (int r = 0; r < n; ++r) {
    const float T = sp->temperature[r], p = sp->top_p[r];
    FO1_CHECK_ARG(std::isfinite(T) && T > 0.f, "%s: row %d: temperature %g must be > 0 and finite", fn, r, (double)T);
    FO1_CHECK_ARG(p > 0.f && p <= 1.f, "%s: row %d: top_p %g must be in (0, 1]", fn, r, (double)p);
    FO1_CHECK_ARG(sp->top_k[r] >= 0, "%s: row %d: top_k %d must be >= 0", fn, r, sp->top_k[r]);
  }
  return FO1_OK;
}

int sample_rows(const float* logits, long long ld, int n_rows, int V, const SampleRowParams* prm, const int* step, int step_stride,
                int* out, cudaStream_t s) {
  FO1_CHECK_ARG(n_rows <= 65535, "sample_rows: %d rows exceed the grid limit", n_rows);
  launch_k(sample_rows_kernel, dim3(n_rows), dim3(kSampleThreads), 0, s, logits, ld, V, prm, step, step_stride, out);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1

using namespace fo1;

extern "C" size_t fo1_sample_tokens_workspace_bytes(int32_t n_rows) {
  return align_up((size_t)(n_rows > 0 ? n_rows : 0) * sizeof(SampleRowParams), 256);
}

extern "C" int fo1_sample_tokens(const float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_sampling_desc* sp,
                                 const int32_t* step, int32_t* out_tokens, void* workspace, size_t workspace_bytes, void* stream) {
  FO1_TRY(sampling_check(sp, n_rows, "fo1_sample_tokens"));
  FO1_CHECK_ARG(vocab > 0 && ld >= vocab, "fo1_sample_tokens: vocab %d / ld %lld", vocab, (long long)ld);
  FO1_CHECK_ARG(logits && step && out_tokens, "fo1_sample_tokens: null device pointer");
  const size_t need = fo1_sample_tokens_workspace_bytes(n_rows);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("fo1_sample_tokens: workspace %zu B < required %zu B", workspace_bytes, need);
    return FO1_ERR_WORKSPACE;
  }
  std::vector<SampleRowParams> h(n_rows);
  for (int r = 0; r < n_rows; ++r) h[r] = SampleRowParams{sp->temperature[r], sp->top_p[r], sp->top_k[r], 0, sp->seed[r]};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  FO1_CUDA(cudaMemcpyAsync(workspace, h.data(), h.size() * sizeof(SampleRowParams), cudaMemcpyHostToDevice, s));
  return sample_rows(logits, ld, n_rows, vocab, static_cast<const SampleRowParams*>(workspace), step, 1, out_tokens, s);
}
