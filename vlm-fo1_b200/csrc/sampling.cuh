// sampling.cuh -- one row of sampled decoding (temperature -> top-k -> top-p -> draw), shared by the standalone kernel
// (sampling.cu), the per-kernel decode step (llm.cu) and the persistent decode kernel (decode_mega.cu).
//
// The contract is HF generate's sampling warper chain (TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper ->
// multinomial), with every order made explicit:
//   x = logits / T (fp32 IEEE division; T == 1: no scaling).
//   canonical order: x descending, then token index ascending (-0 and +0 are one value).
//   top-k (1 < k < V): keep every token whose x >= the k-th largest x (ties at the threshold kept).  k == 1 is greedy: the
//     lowest index among the maxima, the rule of both greedy kernels (so a greedy sample in a sampled batch is bit-identical).
//   top-p (p < 1): with weights exp(x - max) over the kept tokens, keep a token iff the weight ranked above it is < p * Z.
//   draw: u = (x0 >> 8) * 2^-24 of Philox4x32-10(key = seed, counter = (step, 0, 0, 0)); the first kept token whose
//     inclusive cumulative weight exceeds u * Z_kept.
//
// Every cut is one primitive: walk down the canonical order until a running weight crosses a target.  Four passes over
// 8-bit digits of the order-preserving uint32 key of x (256-bin shared-memory histograms) find the value of the crossing
// token; one more pass resolves the tie group of that value by index.  Weights are 1 (top-k) or exp(x - max) rounded to
// 64-bit fixed point with 40 fraction bits: integer sums do not depend on the order of the additions, so the token is a
// function of (row, T, p, k, seed, step) alone -- not of the thread count, the batch slot or the decode path.
//
// Scoring (HF generate's output_logits / output_scores, and the log-probability of each emitted token) reuses the row routine:
//   kept set: the domain the draw walks -- top-k keeps x >= the k-th largest (ties included), top-p as above.  For k == 1 it is
//     every token equal to the maximum (HF's TopK rule; then top-p), while the token drawn stays the lowest-index maximum.  A raw
//     row (a greedy sequence) keeps the whole vocabulary with T = 1.
//   scores row: x where kept, -inf elsewhere (a raw row: the logits unchanged).
//   logprob of token t: (x_t - x_max) - ln(Z_kept * 2^-40), Z_kept the order-free fixed-point sum of exp(x - x_max) over the kept
//     set; -inf for a token outside it.  Like the token, it depends on (row, T, p, k, t) alone.
//   A row of -inf only (the logits processors banned every token) draws token 0 and keeps nothing (log-probability -inf).
// sample_row<NT, SMP_DRAW> is the sampler; SMP_DRAW_KEPT also leaves the kept set in SampleSmem (the draw is unchanged) and
// SMP_KEPT stops before the draw; score_row then makes one pass over the row.
#pragma once
#include <climits>

#include "common.cuh"

namespace fo1 {

// per-row parameters as the kernels read them (one 24-byte record per row; host-validated by sampling_check)
struct SampleRowParams {
  float temperature, top_p;
  int top_k;
  int raw;        // scored rows only: 1 = a greedy sequence (T = 1, top_k = 1) scored on its raw logits; 0 for the sampler
  unsigned long long seed;
};

template <int NT>
struct SampleSmem {
  unsigned long long hist[256];
  unsigned long long part[NT / 32];
  unsigned long long mem_w[NT];     // the tie group of the crossing value, when it has at most NT members
  int mem_idx[NT];
  float maxv[NT / 32];
  int maxi[NT / 32];
  unsigned long long tgt, above, res_incl;
  uint32_t res_key;
  int n_mem, res_idx, res_bin, found;
  // the kept set {key > kept_key} u {key == kept_key, index <= kept_idx} and the row maximum (SMP_DRAW_KEPT / SMP_KEPT only)
  uint32_t kept_key;
  int kept_idx;
  float kept_max;
};

enum { SMP_DRAW = 0, SMP_DRAW_KEPT = 1, SMP_KEPT = 2 };

int sampling_check(const fo1_sampling_desc* sp, int n, const char* fn);   // host: parameter validation (no CUDA call)
// rows [n_rows] of `logits` (pitch ld) -> out[r]; step[r * step_stride] is the Philox counter of row r (stride 0: one step)
int sample_rows(const float* logits, long long ld, int n_rows, int V, const SampleRowParams* prm, const int* step, int step_stride,
                int* out, cudaStream_t s);
// scored rows [n_rows] of `logits` (pitch ld).  The output column is *col (nullptr: 0).  draw: tok[r] = the sampled token (the
// Philox step is the column), else tok[r] is the token to score.  finished (nullptr: none) / max_new: rows to skip (their token is
// still drawn).  logprobs[r * lp_stride + col]; optional scores / logits_out rows at ((col * n_rows + r) * ld_out).
int score_rows(const float* logits, long long ld, int n_rows, int V, const SampleRowParams* prm, const int* col, int* tok, bool draw,
               const int* finished, int max_new, float* logprobs, long long lp_stride, float* scores, float* logits_out, long long ld_out,
               cudaStream_t s);
// host: raw_rows (optional, 0 / 1 per row) validation -- with sp, a raw row must be greedy (top_k 1, temperature 1) -- and the
// device parameters of a scored row (sp == nullptr or a raw row: greedy, scored on the raw logits)
int raw_rows_check(const fo1_sampling_desc* sp, const int32_t* raw_rows, int n, const char* fn);
SampleRowParams score_row_params(const fo1_sampling_desc* sp, const int32_t* raw_rows, int r);

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smp_key(float x) {
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;                         // -0 == +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float smp_uniform(unsigned long long seed, uint32_t step) {
  uint32_t c0 = step, c1 = 0u, c2 = 0u, c3 = 0u, k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return (float)(c0 >> 8) * 0x1p-24f;
}

__device__ __forceinline__ unsigned long long smp_warp_incl_scan(unsigned long long v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// One cut: the first token (canonical order) of the domain {key > dk} u {key == dk, index <= di} whose inclusive running
// weight exceeds the target.  mode 0: weight 1, target k - 1 (top-k; only the VALUE is resolved).  mode 1: weight exp(x - xmax),
// target ceil(p Z) - 1 (top-p: the last kept token).  mode 2: weight exp(x - xmax), target floor(u Z) (the draw).  Z = the
// domain's total weight.  Result in sm: found, res_key (the crossing value's key), res_idx, res_incl (inclusive weight at the cut).
template <int NT>
__device__ void smp_cut(const float* __restrict__ row, int V, float T, float xmax, uint32_t dk, int di, int mode, double param,
                        SampleSmem<NT>& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool scale = T != 1.0f;
  uint32_t prefix = 0u;
  for (int d = 0; d < 4; ++d) {
    const int shift = 24 - 8 * d;
    for (int b = tid; b < 256; b += NT) sm.hist[b] = 0ull;
    __syncthreads();
    int cur = -1;
    unsigned long long cw = 0ull;
    for (int i = tid; i < V; i += NT) {
      const float raw = __ldcg(row + i);
      const float x = scale ? __fdiv_rn(raw, T) : raw;
      const uint32_t k = smp_key(x);
      if (k < dk || (k == dk && i > di)) continue;
      if (d > 0 && ((k ^ prefix) >> (shift + 8)) != 0u) continue;
      const unsigned long long w = mode == 0 ? 1ull : __float2ull_rn(expf(x - xmax) * 1099511627776.0f);   // 2^40
      const int bin = (int)((k >> shift) & 255u);
      if (bin != cur) {                       // runs of one bin go to shared memory as one atomic
        if (cw != 0ull) atomicAdd(&sm.hist[cur], cw);
        cur = bin; cw = w;
      } else {
        cw += w;
      }
    }
    if (cw != 0ull) atomicAdd(&sm.hist[cur], cw);
    __syncthreads();
    if (warp == 0) {
      // lane l owns bins 255 - 8l .. 248 - 8l: the walk goes down the canonical order
      unsigned long long s = 0ull;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += sm.hist[255 - 8 * lane - j];
      const unsigned long long incl = smp_warp_incl_scan(s);
      if (d == 0) {
        const unsigned long long Z = __shfl_sync(0xffffffffu, incl, 31);
        unsigned long long tgt;
        if (mode == 0) tgt = (unsigned long long)param - 1ull;
        else if (mode == 1) { const double c = ceil(param * (double)Z); tgt = c < 1.0 ? 0ull : (unsigned long long)c - 1ull; }
        else tgt = (unsigned long long)floor(param * (double)Z);
        if (lane == 0) { sm.tgt = tgt; sm.above = 0ull; sm.found = Z > tgt ? 1 : 0; }
        __syncwarp();
      }
      const unsigned long long above = sm.above, tgt = sm.tgt;
      const unsigned ball = __ballot_sync(0xffffffffu, above + incl > tgt);
      if (sm.found && ball != 0u && lane == __ffs(ball) - 1) {
        unsigned long long run = above + incl - s;
        for (int j = 0; j < 8; ++j) {
          const int bin = 255 - 8 * lane - j;
          if (run + sm.hist[bin] > tgt) { sm.res_bin = bin; sm.above = run; break; }
          run += sm.hist[bin];
        }
      }
    }
    __syncthreads();
    if (!sm.found) return;
    prefix |= (uint32_t)sm.res_bin << shift;
  }
  if (tid == 0) sm.res_key = prefix;
  if (mode == 0) {
    __syncthreads();
    return;
  }
  // ---- the tie group of the crossing value, in index order ----
  if (tid == 0) sm.n_mem = 0;
  __syncthreads();
  const unsigned long long above = sm.above, tgt = sm.tgt;
  for (int i = tid; i < V; i += NT) {
    const float raw = __ldcg(row + i);
    const float x = scale ? __fdiv_rn(raw, T) : raw;
    if (smp_key(x) != prefix || (prefix == dk && i > di)) continue;
    const int pos = atomicAdd(&sm.n_mem, 1);
    if (pos < NT) { sm.mem_idx[pos] = i; sm.mem_w[pos] = __float2ull_rn(expf(x - xmax) * 1099511627776.0f); }
  }
  __syncthreads();
  const int n = sm.n_mem;
  if (n <= NT) {
    if (tid < n) {
      const int me = sm.mem_idx[tid];
      unsigned long long ex = above;
      for (int j = 0; j < n; ++j)
        if (sm.mem_idx[j] < me) ex += sm.mem_w[j];
      const unsigned long long w = sm.mem_w[tid];
      if (ex <= tgt && ex + w > tgt) { sm.res_idx = me; sm.res_incl = ex + w; }
    }
    __syncthreads();
  } else {
    // a large tie group: block-wide running sums over index chunks
    unsigned long long carry = above;
    for (int base = 0; base < V; base += NT) {
      const int i = base + tid;
      unsigned long long w = 0ull;
      if (i < V) {
        const float raw = __ldcg(row + i);
        const float x = scale ? __fdiv_rn(raw, T) : raw;
        if (smp_key(x) == prefix && !(prefix == dk && i > di)) w = __float2ull_rn(expf(x - xmax) * 1099511627776.0f);
      }
      const unsigned long long incl = smp_warp_incl_scan(w);
      if (lane == 31) sm.part[warp] = incl;
      __syncthreads();
      unsigned long long off = carry, tot = 0ull;
      for (int ww = 0; ww < NT / 32; ++ww) {
        if (ww < warp) off += sm.part[ww];
        tot += sm.part[ww];
      }
      if (w != 0ull && off + incl - w <= tgt && off + incl > tgt) { sm.res_idx = i; sm.res_incl = off + incl; sm.found = 2; }
      __syncthreads();
      carry += tot;
      if (sm.found == 2) break;
    }
    __syncthreads();
  }
}

// the token of one row; every thread of the CTA calls it and gets the same value.  MODE != SMP_DRAW: the kept set is left in
// sm.kept_* (SMP_KEPT returns the arg-max without drawing)
template <int NT, int MODE = SMP_DRAW>
__device__ int sample_row(const float* __restrict__ row, int V, const SampleRowParams& prm, int step, SampleSmem<NT>& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float T = prm.temperature;
  const bool scale = T != 1.0f;
  // ---- max of x and the lowest index attaining it ----
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int i = tid; i < V; i += NT) {
    const float raw = __ldcg(row + i);
    const float x = scale ? __fdiv_rn(raw, T) : raw;
    if (x > bv || (x == bv && i < bi)) { bv = x; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { sm.maxv[warp] = bv; sm.maxi[warp] = bi; }
  __syncthreads();
  bv = sm.maxv[0]; bi = sm.maxi[0];
  for (int w = 1; w < NT / 32; ++w)
    if (sm.maxv[w] > bv || (sm.maxv[w] == bv && sm.maxi[w] < bi)) { bv = sm.maxv[w]; bi = sm.maxi[w]; }
  __syncthreads();
  if (bv == -INFINITY) {     // every token banned by the logits processors: token 0 (the arg-max rule), nothing kept
    if constexpr (MODE != SMP_DRAW) {
      if (tid == 0) { sm.kept_key = 0xffffffffu; sm.kept_idx = -1; sm.kept_max = bv; }
      __syncthreads();
    }
    return bi;
  }
  if constexpr (MODE == SMP_DRAW) {
    if (prm.top_k == 1) return bi;
  }
  uint32_t dk = 0u;
  int di = INT_MAX;
  bool cut = true;
  if constexpr (MODE != SMP_DRAW) {
    cut = !prm.raw;
    if (prm.top_k == 1) dk = smp_key(bv);        // HF's TopK(1): every token equal to the maximum
  }
  if (cut && prm.top_k > 1 && prm.top_k < V) {
    smp_cut<NT>(row, V, T, bv, dk, di, 0, (double)prm.top_k, sm);
    dk = sm.res_key;                    // kept: x >= the k-th largest (ties included)
    __syncthreads();
  }
  if (cut && prm.top_p < 1.0f) {
    smp_cut<NT>(row, V, T, bv, dk, di, 1, (double)prm.top_p, sm);
    if (sm.found) { dk = sm.res_key; di = sm.res_idx; }
    __syncthreads();
  }
  if constexpr (MODE != SMP_DRAW) {
    if (tid == 0) { sm.kept_key = cut ? dk : 0u; sm.kept_idx = cut ? di : INT_MAX; sm.kept_max = bv; }
    if (MODE == SMP_KEPT || prm.top_k == 1) { __syncthreads(); return bi; }
  }
  smp_cut<NT>(row, V, T, bv, dk, di, 2, (double)smp_uniform(prm.seed, (uint32_t)step), sm);
  // (the integer target floor(u Z) < Z always crosses; the arg-max stands in if it ever did not)
  const int tok = sm.found ? sm.res_idx : bi;
  __syncthreads();
  return tok;
}

// After sample_row<NT, SMP_DRAW_KEPT or SMP_KEPT> on the same row: one pass that sums Z_kept and writes the optional scores row
// (x kept, -inf elsewhere) and copy of the raw row.  Returns the log-probability of `tok` in thread 0 (-inf outside the kept set).
template <int NT>
__device__ float score_row(const float* __restrict__ row, int V, float T, int tok, SampleSmem<NT>& sm, float* __restrict__ scores,
                           float* __restrict__ raw_out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool scale = T != 1.0f;
  const uint32_t dk = sm.kept_key;
  const int di = sm.kept_idx;
  const float xmax = sm.kept_max;
  unsigned long long z = 0ull;
  for (int i = tid; i < V; i += NT) {
    const float raw = __ldcg(row + i);
    const float x = scale ? __fdiv_rn(raw, T) : raw;
    const uint32_t k = smp_key(x);
    const bool kept = !(k < dk || (k == dk && i > di));
    if (kept) z += __float2ull_rn(expf(x - xmax) * 1099511627776.0f);   // 2^40
    if (scores != nullptr) scores[i] = kept ? x : -INFINITY;
    if (raw_out != nullptr) raw_out[i] = raw;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  if (lane == 0) sm.part[warp] = z;
  __syncthreads();
  float lp = 0.f;
  if (tid == 0) {
    unsigned long long Z = 0ull;
    for (int w = 0; w < NT / 32; ++w) Z += sm.part[w];
    lp = -INFINITY;
    if (tok >= 0 && tok < V) {
      const float raw = __ldcg(row + tok);
      const float x = scale ? __fdiv_rn(raw, T) : raw;
      const uint32_t k = smp_key(x);
      if (!(k < dk || (k == dk && tok > di))) lp = (float)(((double)x - (double)xmax) - log((double)Z * 0x1p-40));
    }
  }
  __syncthreads();
  return lp;
}
#endif

}  // namespace fo1
