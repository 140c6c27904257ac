// sampling.cu -- the standalone sampling kernel over [n_rows][ld] fp32 logits (one CTA per row) and its C ABI.  The row
// routine (sampling.cuh) is the one the two decode paths run.
#include <cmath>
#include <vector>

#include "lookup.cuh"

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

// scored rows (one CTA per row): DRAW = the per-kernel decode step (tok[r] out: the token sample_rows_kernel would draw), else
// fo1_score_rows (tok[r] in)
template <bool DRAW>
__global__ void __launch_bounds__(kSampleThreads) score_rows_kernel(const float* __restrict__ logits, long long ld, int V,
                                                                    const SampleRowParams* __restrict__ prm, const int* __restrict__ col_p,
                                                                    int* __restrict__ tok, const int* __restrict__ finished, int max_new,
                                                                    float* __restrict__ logprobs, long long lp_stride, float* __restrict__ scores,
                                                                    float* __restrict__ logits_out, long long ld_out) {
  griddep_launch();
  griddep_wait();
  __shared__ SampleSmem<kSampleThreads> sm;
  const int r = blockIdx.x;
  const SampleRowParams p = prm[r];
  const float* row = logits + (long long)r * ld;
  const int col = col_p != nullptr ? __ldcg(col_p) : 0;
  int t;
  if constexpr (DRAW) {
    t = sample_row<kSampleThreads, SMP_DRAW_KEPT>(row, V, p, col, sm);
    if (threadIdx.x == 0) tok[r] = t;
  } else {
    sample_row<kSampleThreads, SMP_KEPT>(row, V, p, col, sm);
    t = __ldcg(tok + r);
  }
  if (finished != nullptr && (col >= max_new || __ldcg(finished + r))) return;     // past the sequence's stop: nothing is recorded
  const long long o = ((long long)col * gridDim.x + r) * ld_out;
  const float lp = score_row<kSampleThreads>(row, V, p.temperature, t, sm, scores ? scores + o : nullptr,
                                             logits_out ? logits_out + o : nullptr);
  if (threadIdx.x == 0 && logprobs != nullptr) logprobs[(long long)r * lp_stride + col] = lp;
}

// scored prompt-lookup verify rows (one CTA per row): score_rows_kernel<true>'s draw and scoring with row r's own column
// row_col[r] and sequence b = r / K1's parameters; the scores / logits rows go to (column, b), the log-probability to row_lp[r]
__global__ void __launch_bounds__(kSampleThreads) score_rows_lookup_kernel(const float* __restrict__ logits, long long ld, int V, int K1,
                                                                           const SampleRowParams* __restrict__ prm, const int* __restrict__ row_col,
                                                                           int* __restrict__ tok, float* __restrict__ row_lp,
                                                                           const int* __restrict__ finished, int max_new, int n_seqs,
                                                                           float* __restrict__ scores, float* __restrict__ logits_out) {
  griddep_launch();
  griddep_wait();
  __shared__ SampleSmem<kSampleThreads> sm;
  const int r = blockIdx.x, b = r / K1;
  const SampleRowParams p = prm[b];
  const float* row = logits + (long long)r * ld;
  const int col = __ldcg(row_col + r);
  const int t = sample_row<kSampleThreads, SMP_DRAW_KEPT>(row, V, p, col, sm);
  if (threadIdx.x == 0) tok[r] = t;
  if (col >= max_new || __ldcg(finished + b)) return;     // past the sequence's end: nothing is recorded
  const long long o = ((long long)col * n_seqs + b) * V;
  const float lp = score_row<kSampleThreads>(row, V, p.temperature, t, sm, scores ? scores + o : nullptr, logits_out ? logits_out + o : nullptr);
  if (threadIdx.x == 0) row_lp[r] = lp;
}

int score_rows_lookup(const float* logits, long long ld, int n_rows, int K1, int V, const SampleRowParams* prm, const int* row_col,
                      int* tok, float* row_lp, const int* finished, int max_new, int n_seqs, float* scores, float* logits_out, cudaStream_t s) {
  FO1_CHECK_ARG(n_rows <= 65535, "score_rows_lookup: %d rows exceed the grid limit", n_rows);
  launch_k(score_rows_lookup_kernel, dim3(n_rows), dim3(kSampleThreads), 0, s, logits, ld, V, K1, prm, row_col, tok, row_lp, finished, max_new,
           n_seqs, scores, logits_out);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
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

int score_rows(const float* logits, long long ld, int n_rows, int V, const SampleRowParams* prm, const int* col, int* tok, bool draw,
               const int* finished, int max_new, float* logprobs, long long lp_stride, float* scores, float* logits_out, long long ld_out,
               cudaStream_t s) {
  FO1_CHECK_ARG(n_rows <= 65535, "score_rows: %d rows exceed the grid limit", n_rows);
  if (draw)
    launch_k(score_rows_kernel<true>, dim3(n_rows), dim3(kSampleThreads), 0, s, logits, ld, V, prm, col, tok, finished, max_new, logprobs,
             lp_stride, scores, logits_out, ld_out);
  else
    launch_k(score_rows_kernel<false>, dim3(n_rows), dim3(kSampleThreads), 0, s, logits, ld, V, prm, col, tok, finished, max_new, logprobs,
             lp_stride, scores, logits_out, ld_out);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int raw_rows_check(const fo1_sampling_desc* sp, const int32_t* raw_rows, int n, const char* fn) {
  if (raw_rows == nullptr) return FO1_OK;
  for (int r = 0; r < n; ++r) {
    FO1_CHECK_ARG(raw_rows[r] == 0 || raw_rows[r] == 1, "%s: raw_rows[%d] = %d must be 0 or 1", fn, r, raw_rows[r]);
    if (sp != nullptr && raw_rows[r])
      FO1_CHECK_ARG(sp->top_k[r] == 1 && sp->temperature[r] == 1.0f,
                    "%s: row %d: a raw (greedy) row needs top_k 1 and temperature 1 (has %d, %g)", fn, r, sp->top_k[r],
                    (double)sp->temperature[r]);
  }
  return FO1_OK;
}

SampleRowParams score_row_params(const fo1_sampling_desc* sp, const int32_t* raw_rows, int r) {
  if (sp == nullptr || (raw_rows != nullptr && raw_rows[r])) return SampleRowParams{1.0f, 1.0f, 1, 1, sp ? sp->seed[r] : 0ull};
  return SampleRowParams{sp->temperature[r], sp->top_p[r], sp->top_k[r], 0, sp->seed[r]};
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

extern "C" int fo1_score_rows(const float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_sampling_desc* sp,
                              const int32_t* raw_rows, const int32_t* tokens, float* logprobs, float* scores, int64_t ld_scores,
                              void* stream) {
  FO1_CHECK_ARG(n_rows > 0, "fo1_score_rows: n_rows %d must be positive", n_rows);
  FO1_CHECK_ARG(n_rows <= 65535, "fo1_score_rows: %d rows exceed the grid limit", n_rows);
  FO1_CHECK_ARG(vocab > 0 && ld >= vocab, "fo1_score_rows: vocab %d / ld %lld", vocab, (long long)ld);
  FO1_CHECK_ARG(scores == nullptr || ld_scores >= vocab, "fo1_score_rows: ld_scores %lld < vocab %d", (long long)ld_scores, vocab);
  FO1_CHECK_ARG(logits && tokens && logprobs, "fo1_score_rows: null device pointer");
  if (sp) FO1_TRY(sampling_check(sp, n_rows, "fo1_score_rows"));
  FO1_TRY(raw_rows_check(nullptr, raw_rows, n_rows, "fo1_score_rows"));
  std::vector<SampleRowParams> h(n_rows);
  for (int r = 0; r < n_rows; ++r) h[r] = score_row_params(sp, raw_rows, r);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  SampleRowParams* d = nullptr;
  FO1_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d), h.size() * sizeof(SampleRowParams), s));
  int rc = FO1_OK;
  if (cudaMemcpyAsync(d, h.data(), h.size() * sizeof(SampleRowParams), cudaMemcpyHostToDevice, s) != cudaSuccess) {
    set_error("fo1_score_rows: parameter upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    rc = FO1_ERR_CUDA;
  } else {
    rc = score_rows(logits, ld, n_rows, vocab, d, nullptr, const_cast<int32_t*>(tokens), false, nullptr, 0, logprobs, 1, scores, nullptr,
                    ld_scores, s);
  }
  cudaFreeAsync(d, s);
  return rc;
}
