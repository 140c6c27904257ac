// beam.cu -- beam search kernels of the per-kernel decode loop (beam.cuh) and their host checks.
#include <algorithm>
#include <climits>
#include <cmath>

#include "beam.cuh"
#include "sampling.cuh"

namespace fo1 {

constexpr int kBeamRowThreads = 1024;
constexpr int kBeamSelThreads = 256;
constexpr int kBeamReorderThreads = 256;
constexpr float kBeamNeg = -1.0e9f;     // HF's -1e9 (an exact fp32 value)

// ------------------------------------------------------------------------------------------ kernels
__global__ void beam_init_kernel(BeamArgs a, DecodeState st, const int* __restrict__ seq_lens, const int* __restrict__ deltas) {
  const int R = a.S * a.N;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) { *st.step = 0; *st.n_active = a.S; }
  if (r >= R) return;
  const int b = r / a.N;
  st.cache_len[r] = seq_lens[b];
  const int p = seq_lens[b] + deltas[b];
  st.pos3[r] = p; st.pos3[R + r] = p; st.pos3[2 * R + r] = p;
  st.finished[r] = 0;
  a.run_score[r] = (r % a.N) == 0 ? 0.0f : kBeamNeg;
  a.fin_score[r] = kBeamNeg;
  a.fin_len[r] = 0; a.fin_tok[r] = 0; a.fin_par[r] = 0; a.fin_done[r] = 0; a.fin_lp[r] = 0.0f;
  if (r % a.N == 0) { a.unsat[b] = 1; a.done[b] = 0; a.steps_run[b] = 0; }
}

// One beam row of column *step: lp = log_softmax(row) (x - max - ln(Z 2^-40), Z the sampler's order-free fixed-point sum), acc =
// lp + running score, then the row's top K of acc in canonical order (key descending, token ascending) -> cand_*[r].  Column 0
// (col0) reads the prompt's one prefill row for all its N rows.
__global__ void __launch_bounds__(kBeamRowThreads) beam_rows_kernel(BeamArgs a, const float* __restrict__ logits, const int* __restrict__ step_p,
                                                                    int col0) {
  constexpr int NT = kBeamRowThreads;
  griddep_launch();
  griddep_wait();
  __shared__ SampleSmem<NT> sm;
  __shared__ float s_max[NT / 32];
  __shared__ int s_warp[NT / 32];
  __shared__ int s_cnt;
  __shared__ uint32_t s_key[kBeamMaxKeep];
  __shared__ int s_idx[kBeamMaxKeep];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r = blockIdx.x, b = r / a.N, V = a.V, K = a.K, R = a.S * a.N;
  if (__ldcg(a.done + b)) return;
  const int step = __ldcg(step_p);
  const float* row = logits + (long long)(col0 ? b : r) * V;
  float* acc = a.acc + (long long)r * V;
  const float running = __ldcg(a.run_score + r);
  // ---- max ----
  float mx = -INFINITY;
  for (int i = tid; i < V; i += NT) mx = fmaxf(mx, __ldcg(row + i));
  mx = warp_max(mx);
  if (lane == 0) s_max[warp] = mx;
  __syncthreads();
  mx = s_max[0];
  for (int w = 1; w < NT / 32; ++w) mx = fmaxf(mx, s_max[w]);
  // ---- Z (fixed point: independent of the summation order) ----
  unsigned long long z = 0ull;
  for (int i = tid; i < V; i += NT) z += __float2ull_rn(expf(__ldcg(row + i) - mx) * 1099511627776.0f);   // 2^40
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  if (lane == 0) sm.part[warp] = z;
  __syncthreads();
  unsigned long long Z = 0ull;
  for (int w = 0; w < NT / 32; ++w) Z += sm.part[w];
  const double logz = log((double)Z * 0x1p-40);
  // ---- lp, acc; the optional output rows ----
  const long long o = ((long long)step * R + r) * V;
  for (int i = tid; i < V; i += NT) {
    const float x = __ldcg(row + i);
    const float lp = (float)(((double)x - (double)mx) - logz);
    acc[i] = __fadd_rn(lp, running);
    if (a.scores != nullptr) a.scores[o + i] = lp;
    if (a.logits != nullptr) a.logits[o + i] = x;
  }
  __syncthreads();
  // ---- the K-th largest acc (its key and the count strictly above it) ----
  smp_cut<NT>(acc, V, 1.0f, 0.0f, 0u, INT_MAX, 0, (double)K, sm);
  const uint32_t rk = sm.res_key;
  const int above = (int)sm.above, need = K - above;
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  // ---- collect: every key above the cut, then the first `need` ties by index ----
  int tie_base = 0;
  for (int base = 0; base < V; base += NT) {
    const int i = base + tid;
    uint32_t k = 0u;
    bool gt = false, eq = false;
    if (i < V) { k = smp_key(__ldcg(acc + i)); gt = k > rk; eq = k == rk; }
    if (gt) { const int p = atomicAdd(&s_cnt, 1); s_key[p] = k; s_idx[p] = i; }
    const unsigned ball = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) s_warp[warp] = __popc(ball);
    __syncthreads();
    const int cnt = s_cnt;                               // every atomicAdd of this pass is before the barrier
    int off = tie_base, tot = 0;
    for (int w = 0; w < NT / 32; ++w) { if (w < warp) off += s_warp[w]; tot += s_warp[w]; }
    if (eq) {
      const int rank = off + __popc(ball & ((1u << lane) - 1u));
      if (rank < need) { s_key[above + rank] = k; s_idx[above + rank] = i; }
    }
    tie_base += tot;
    __syncthreads();
    if (tie_base >= need && cnt == above) break;         // uniform: every thread read the same count
  }
  __syncthreads();
  // ---- canonical order of the K and the candidate records ----
  if (tid < K) {
    const uint32_t k = s_key[tid];
    const int i = s_idx[tid];
    int rank = 0;
    for (int j = 0; j < K; ++j) rank += (s_key[j] > k || (s_key[j] == k && s_idx[j] < i)) ? 1 : 0;
    const long long c = (long long)r * K + rank;
    a.cand_score[c] = __ldcg(acc + i);
    a.cand_tok[c] = i;
    a.cand_lp[c] = (float)(((double)__ldcg(row + i) - (double)mx) - logz);
  }
}

// canonical "precedes": score descending, then position ascending
__device__ __forceinline__ bool beam_before(float s1, long long f1, float s2, long long f2) { return s1 > s2 || (s1 == s2 && f1 < f2); }

// One prompt's selection for column *step (HF's steps c - g for batch size 1).  `advance`: the column came from a decode step.
__global__ void __launch_bounds__(kBeamSelThreads) beam_select_kernel(BeamArgs a, DecodeState st, int advance) {
  griddep_launch();
  griddep_wait();
  constexpr int MC = kBeamMaxBeams * kBeamMaxKeep;
  __shared__ float c_score[MC], c_lp[MC];
  __shared__ int c_tok[MC];
  __shared__ float t_score[kBeamMaxKeep], t_lp[kBeamMaxKeep], t_run[kBeamMaxKeep], t_fin[kBeamMaxKeep + kBeamMaxBeams];
  __shared__ int t_tok[kBeamMaxKeep], t_par[kBeamMaxKeep], t_hit[kBeamMaxKeep];
  __shared__ int m_sel[kBeamMaxBeams];
  __shared__ float m_score[kBeamMaxBeams], m_lp[kBeamMaxBeams];
  __shared__ int m_len[kBeamMaxBeams], m_tok[kBeamMaxBeams], m_par[kBeamMaxBeams], m_done[kBeamMaxBeams];
  __shared__ float s_best;
  const int tid = threadIdx.x;
  const int b = blockIdx.x, N = a.N, K = a.K, V = a.V, R = a.S * a.N, base = b * N;
  if (__ldcg(a.done + b)) return;
  const int t = __ldcg(st.step);
  const int nc = N * K;
  for (int c = tid; c < nc; c += blockDim.x) {
    const long long g = (long long)base * K + c;         // row base + c / K, position c % K
    c_score[c] = __ldcg(a.cand_score + g); c_lp[c] = __ldcg(a.cand_lp + g); c_tok[c] = __ldcg(a.cand_tok + g);
  }
  __syncthreads();
  // ---- top K of the N * K (each row's list is sorted: a binary search per other row gives the global rank) ----
  for (int c = tid; c < nc; c += blockDim.x) {
    const int j = c / K;
    const float s = c_score[c];
    const long long f = (long long)j * V + c_tok[c];
    int rank = c - j * K;
    for (int j2 = 0; j2 < N; ++j2) {
      if (j2 == j) continue;
      int lo = 0, hi = K;                                // entries of row j2 that precede (s, f): a prefix of its list
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int e = j2 * K + mid;
        if (beam_before(c_score[e], (long long)j2 * V + c_tok[e], s, f)) lo = mid + 1; else hi = mid;
      }
      rank += lo;
    }
    if (rank < K) { t_score[rank] = s; t_lp[rank] = c_lp[c]; t_tok[rank] = c_tok[c]; t_par[rank] = j; }
  }
  __syncthreads();
  // ---- stop test; running scores (_get_running_beams_for_next_iteration) ----
  for (int k = tid; k < K; k += blockDim.x) {
    bool hit = t + 1 >= a.max_new;
    for (int i = 0; i < a.n_stop; ++i) hit |= t_tok[k] == a.stop_ids[i];
    t_hit[k] = hit ? 1 : 0;
    t_run[k] = __fadd_rn(t_score[k], hit ? kBeamNeg : -0.0f);
  }
  const int unsat = __ldcg(a.unsat + b);
  bool full = a.early_stopping == 1;
  for (int j = 0; j < N; ++j) full = full && __ldcg(a.fin_done + base + j) != 0;
  __syncthreads();
  for (int k = tid; k < K; k += blockDim.x) {
    int rank = 0;
    for (int k2 = 0; k2 < K; ++k2) rank += beam_before(t_run[k2], k2, t_run[k], k) ? 1 : 0;
    if (rank < N) {
      const int r = base + rank;
      a.run_score[r] = t_run[k];
      a.hist_tok[(long long)t * R + r] = t_tok[k];
      a.hist_par[(long long)t * R + r] = t_par[k];
      a.hist_lp[(long long)t * R + r] = t_lp[k];
      a.parent[r] = t_par[k];
      st.cur_tok[r] = t_tok[k];
      if (rank == 0) s_best = t_run[k];
    }
    // ---- finished candidates (_update_finished_beams): length penalty, then the three -1e9 terms in HF's order ----
    float fs = __fdiv_rn(t_score[k], a.lp_div[t + 1]);
    fs = __fadd_rn(fs, full ? kBeamNeg : -0.0f);
    fs = __fadd_rn(fs, unsat ? -0.0f : kBeamNeg);
    fs = __fadd_rn(fs, (t_hit[k] && k < N) ? -0.0f : kBeamNeg);
    t_fin[N + k] = fs;
  }
  for (int j = tid; j < N; j += blockDim.x) t_fin[j] = __ldcg(a.fin_score + base + j);
  __syncthreads();
  // ---- the merged set (old N, then the K new) -> its best N ----
  for (int m = tid; m < N + K; m += blockDim.x) {
    int rank = 0;
    for (int m2 = 0; m2 < N + K; ++m2) rank += beam_before(t_fin[m2], m2, t_fin[m], m) ? 1 : 0;
    if (rank < N) m_sel[rank] = m;
  }
  __syncthreads();
  if (tid < N) {
    const int m = m_sel[tid], e = base + m;
    if (m < N) {
      m_score[tid] = t_fin[m]; m_len[tid] = __ldcg(a.fin_len + e); m_tok[tid] = __ldcg(a.fin_tok + e);
      m_par[tid] = __ldcg(a.fin_par + e); m_lp[tid] = __ldcg(a.fin_lp + e); m_done[tid] = __ldcg(a.fin_done + e);
    } else {
      const int k = m - N;
      m_score[tid] = t_fin[m]; m_len[tid] = t + 1; m_tok[tid] = t_tok[k]; m_par[tid] = t_par[k]; m_lp[tid] = t_lp[k];
      m_done[tid] = (t_hit[k] && k < N) ? 1 : 0;
    }
  }
  __syncthreads();
  if (tid < N) {
    const int e = base + tid;
    a.fin_score[e] = m_score[tid]; a.fin_len[e] = m_len[tid]; a.fin_tok[e] = m_tok[tid]; a.fin_par[e] = m_par[tid];
    a.fin_lp[e] = m_lp[tid]; a.fin_done[e] = m_done[tid];
    if (advance) {
      st.cache_len[e] += 1;
      st.pos3[e] += 1; st.pos3[R + e] += 1; st.pos3[2 * R + e] += 1;
    }
  }
  if (tid == 0) {
    // ---- _check_early_stop_heuristic at cur_len + 1, then _beam_search_has_unfinished_sequences ----
    const int len_h = (a.early_stopping == 2 && a.lp_positive) ? a.max_new : t + 1;
    const float best = __fdiv_rn(s_best, a.lp_div[len_h]);
    float worst = m_score[0];
    bool all_fin = true, any_better = false, all_hit = true;
    for (int j = 1; j < N; ++j) worst = fminf(worst, m_score[j]);
    for (int j = 0; j < N; ++j) {
      any_better = any_better || best > (m_done[j] ? worst : kBeamNeg);
      all_fin = all_fin && m_done[j];
    }
    for (int k = 0; k < K; ++k) all_hit = all_hit && t_hit[k];
    const bool u = unsat && any_better;
    a.unsat[b] = u ? 1 : 0;
    a.steps_run[b] = t + 1;
    if (!(u && !(all_fin && a.early_stopping == 1) && !all_hit)) { a.done[b] = 1; atomicSub(st.n_active, 1); }
  }
}

// child <- parent for the generated rows [L_b, L_b + t) of one layer, for every beam of prompt blockIdx.z whose parent is not itself.
// Rows [c0, c0 + rows_per) per pass: all parent rows are staged in shared memory before any child row is written.
__global__ void __launch_bounds__(kBeamReorderThreads) beam_kv_reorder_kernel(BeamArgs a, const int* __restrict__ step_p, int rows_per) {
  griddep_launch();
  griddep_wait();
  extern __shared__ uint4 stage[];
  __shared__ int s_par[kBeamMaxBeams];
  const int b = blockIdx.z, N = a.N, base = b * N;
  if (__ldcg(a.done + b)) return;
  const int t = __ldcg(step_p), L = a.prompt_len[b];
  if (threadIdx.x < N) s_par[threadIdx.x] = __ldcg(a.parent + base + threadIdx.x);
  __syncthreads();
  const int ch = a.kv_dim / 8;                           // 16-byte chunks per row
  bf16* kc = a.kc + (long long)blockIdx.y * a.layer_stride;
  bf16* vc = a.vc + (long long)blockIdx.y * a.layer_stride;
  auto at = [&](int slot, int row, int kv, int c) -> uint4* {
    return reinterpret_cast<uint4*>((kv ? vc : kc) + ((long long)slot * a.cap + row) * a.kv_dim) + c;
  };
  for (int c0 = blockIdx.x * rows_per; c0 < t; c0 += gridDim.x * rows_per) {
    const int nr = min(rows_per, t - c0), per = nr * 2 * ch, n = N * per;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int j = i / per, q = i % per, rw = q / (2 * ch), kv = (q / ch) & 1, c = q % ch;
      if (s_par[j] != j) stage[i] = *at(base + s_par[j], L + c0 + rw, kv, c);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int j = i / per, q = i % per, rw = q / (2 * ch), kv = (q / ch) & 1, c = q % ch;
      if (s_par[j] != j) *at(base + j, L + c0 + rw, kv, c) = stage[i];
    }
    __syncthreads();
  }
}

__global__ void beam_step_end_kernel(int* step) {
  griddep_launch();
  griddep_wait();
  *step += 1;
}

// the best num_return hypotheses of each prompt: tokens, lengths, scores, beam indices and log-probs, walked back along the parents
__global__ void beam_finalize_kernel(BeamArgs a) {
  const int b = blockIdx.x, i = threadIdx.x, N = a.N, R = a.S * a.N, base = b * N, T = a.max_new;
  if (i >= a.num_return) return;
  const int e = base + i, o = b * a.num_return + i;
  const int len = a.fin_len[e];
  int* tok = a.out_tokens + (long long)o * T;
  int* bi = a.beam_indices + (long long)o * T;
  float* lp = a.out_logprobs != nullptr ? a.out_logprobs + (long long)o * T : nullptr;
  a.out_lens[o] = len;
  a.seq_scores[o] = a.fin_score[e];
  for (int s = len; s < T; ++s) { tok[s] = a.pad_id; bi[s] = -1; if (lp) lp[s] = 0.0f; }
  if (len == 0) return;
  tok[len - 1] = a.fin_tok[e]; bi[len - 1] = base + a.fin_par[e]; if (lp) lp[len - 1] = a.fin_lp[e];
  int j = a.fin_par[e];
  for (int s = len - 2; s >= 0; --s) {
    const long long h = (long long)s * R + base + j;
    tok[s] = a.hist_tok[h]; bi[s] = base + a.hist_par[h]; if (lp) lp[s] = a.hist_lp[h];
    j = a.hist_par[h];
  }
}

// ------------------------------------------------------------------------------------------ host
int beam_check(const fo1_generate_desc* d, const fo1_beam_desc* bm, int vocab) {
  const char* fn = "fo1_llm_generate: beam";
  const int N = bm->num_beams;
  FO1_CHECK_ARG(N >= 2 && N <= kBeamMaxBeams, "%s: num_beams %d must be in [2, %d]", fn, N, kBeamMaxBeams);
  FO1_CHECK_ARG(bm->num_return >= 1 && bm->num_return <= N, "%s: num_return %d must be in [1, num_beams = %d]", fn, bm->num_return, N);
  FO1_CHECK_ARG(bm->n_keep >= 2 * N && bm->n_keep <= kBeamMaxKeep && bm->n_keep <= vocab,
                "%s: n_keep %d must be in [2 * num_beams = %d, min(%d, vocab %d)]", fn, bm->n_keep, 2 * N, kBeamMaxKeep, vocab);
  FO1_CHECK_ARG(std::isfinite(bm->length_penalty), "%s: length_penalty %g must be finite", fn, bm->length_penalty);
  FO1_CHECK_ARG(bm->early_stopping >= 0 && bm->early_stopping <= 2, "%s: early_stopping %d must be 0 (False), 1 (True) or 2 (never)", fn,
                bm->early_stopping);
  FO1_CHECK_ARG(d->max_new_tokens >= 1, "%s: max_new_tokens %d must be >= 1", fn, d->max_new_tokens);
  FO1_CHECK_ARG(d->all_logits == nullptr, "%s: all_logits is not available with beam search", fn);
  FO1_CHECK_ARG(d->out_tokens && d->out_lens && bm->sequence_scores && bm->beam_indices && bm->steps_run, "%s: null output", fn);
  FO1_CHECK_ARG(d->n_seqs > 0 && (long long)d->n_seqs * N <= 65535, "%s: %d prompts x %d beams exceed the grid limit", fn, d->n_seqs, N);
  return FO1_OK;
}

void beam_alloc(Arena& A, BeamArgs& a) {
  const size_t R = (size_t)a.S * a.N, K = a.K, T = a.max_new;
  a.acc = A.alloc<float>(R * a.V);
  a.cand_score = A.alloc<float>(R * K); a.cand_lp = A.alloc<float>(R * K); a.cand_tok = A.alloc<int>(R * K);
  a.run_score = A.alloc<float>(R);
  a.hist_tok = A.alloc<int>(T * R); a.hist_par = A.alloc<int>(T * R); a.hist_lp = A.alloc<float>(T * R);
  a.parent = A.alloc<int>(R);
  a.fin_score = A.alloc<float>(R); a.fin_lp = A.alloc<float>(R);
  a.fin_len = A.alloc<int>(R); a.fin_tok = A.alloc<int>(R); a.fin_par = A.alloc<int>(R); a.fin_done = A.alloc<int>(R);
  a.unsat = A.alloc<int>(a.S); a.done = A.alloc<int>(a.S);
  a.prompt_len = A.alloc<int>(a.S);
  a.lp_div = A.alloc<float>(T + 1);
}

int beam_init(const BeamArgs& a, const DecodeState& st, const int* seq_lens, const int* deltas, cudaStream_t s) {
  const int R = a.S * a.N;
  beam_init_kernel<<<ceil_div(R, 128), 128, 0, s>>>(a, st, seq_lens, deltas);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

// rows of the reorder's staging pass: the parents of N beams x rows x (K, V) in 32 KB (more only when one row needs it)
static int reorder_rows(const BeamArgs& a) { return std::max(1, (32 << 10) / (a.N * 2 * a.kv_dim * (int)sizeof(bf16))); }

int beam_column(const BeamArgs& a, const float* logits, const DecodeState& st, int advance, cudaStream_t s) {
  const int R = a.S * a.N;
  {
    ProfScope prof("beam_rows", 0.0, 0.0, s);
    launch_k(beam_rows_kernel, dim3(R), dim3(kBeamRowThreads), 0, s, a, logits, (const int*)st.step, advance ? 0 : 1);
    FO1_LAUNCH_CHECK();
  }
  {
    ProfScope prof("beam_select", 0.0, 0.0, s);
    launch_k(beam_select_kernel, dim3(a.S), dim3(kBeamSelThreads), 0, s, a, st, advance);
    FO1_LAUNCH_CHECK();
  }
  if (advance) {       // column 0 has no generated rows to move
    const int rows = reorder_rows(a);
    const int chunks = std::max(1, std::min(ceil_div(a.max_new, rows), 8));
    const size_t smem = (size_t)a.N * rows * 2 * a.kv_dim * sizeof(bf16);
    static size_t smem_set = 32 << 10;
    if (smem > smem_set) {
      FO1_CUDA(cudaFuncSetAttribute(beam_kv_reorder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      smem_set = smem;
    }
    ProfScope prof("beam_kv_reorder", 0.0, 0.0, s);
    launch_k(beam_kv_reorder_kernel, dim3(chunks, a.layers, a.S), dim3(kBeamReorderThreads), smem, s, a, (const int*)st.step, rows);
    FO1_LAUNCH_CHECK();
  }
  launch_k(beam_step_end_kernel, dim3(1), dim3(1), 0, s, st.step);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int beam_finalize(const BeamArgs& a, cudaStream_t s) {
  beam_finalize_kernel<<<a.S, 32, 0, s>>>(a);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1
