// lookup.cu -- prompt-lookup decoding: the draft rule, the verify rows, the acceptance (lookup.cuh) and fo1_lookup_drafts.
#include <algorithm>
#include <climits>
#include <vector>

#include "lookup.cuh"

namespace fo1 {

// One CTA per sequence: HF's PromptLookupCandidateGenerator.get_candidates on corpus b.  For n = min(max_ngram, len - 1) down to
// 1, the leftmost i with corpus[i .. i + n) == the last n ids and i + n < len (a non-empty continuation) gives the drafts
// corpus[i + n .. i + n + cap), cut at the first stop id (HF's eos cut) or negative id; the first n with such an i decides, even
// when the cut leaves nothing.  cap = min(K, max_new - col[b] - 1) (col == nullptr: K).
__global__ void __launch_bounds__(256) lookup_drafts_kernel(const int* __restrict__ corpus, long long ld, const int* __restrict__ lens, int K,
                                                            int max_ngram, const int* __restrict__ stop_ids, int n_stop,
                                                            const int* __restrict__ col, int max_new, int* __restrict__ drafts,
                                                            int* __restrict__ n_draft) {
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x;
  const int* c = corpus + (long long)b * ld;
  const int len = lens[b];
  const int cap = col != nullptr ? min(K, max_new - col[b] - 1) : K;
  __shared__ int s_best;
  int start = -1;
  for (int n = min(max_ngram, len - 1); n >= 1 && cap > 0; --n) {
    if (threadIdx.x == 0) s_best = INT_MAX;
    __syncthreads();
    for (int i = threadIdx.x; i + n < len; i += blockDim.x) {
      bool eq = true;
      for (int t = 0; t < n && eq; ++t) eq = c[i + t] == c[len - n + t];
      if (eq) atomicMin(&s_best, i);
    }
    __syncthreads();
    const int best = s_best;
    __syncthreads();                 // every thread has read s_best before the next n resets it
    if (best != INT_MAX) { start = best + n; break; }
  }
  if (threadIdx.x != 0) return;
  int nd = 0;
  if (start >= 0) {
    const int end = min(start + cap, len);
    for (int i = start; i < end; ++i) {
      const int tok = c[i];
      bool stop = tok < 0;
      for (int s = 0; s < n_stop; ++s) stop |= tok == stop_ids[s];
      if (stop) break;
      drafts[(long long)b * K + nd++] = tok;
    }
  }
  n_draft[b] = nd;
}

// after the prefill's column 0: corpus b gets the column's token, the columns start at 1, slots and per-row parameters are fixed
__global__ void lookup_init_kernel(LookupArgs a, DecodeState st, const SampleRowParams* __restrict__ samp) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const int len = a.corpus_len[b];
  a.corpus[(long long)b * a.ld + len] = st.cur_tok[b];
  a.corpus_len[b] = len + 1;
  a.col[b] = 1;
  a.steps[b] = 0; a.accepted[b] = 0;
  const int K1 = a.K + 1;
  for (int j = 0; j < K1; ++j) {
    a.row_slot[b * K1 + j] = b;
    if (samp != nullptr) a.row_prm[b * K1 + j] = samp[b];
  }
}

// row (b, j): cur_tok[b] (j = 0), draft j (j <= n_draft[b]) or cur_tok[b] again (a padding row, computed and ignored), at position
// pos3[b] + j, cache index cache_len[b] + j and output column col[b] + j
__global__ void lookup_rows_kernel(LookupArgs a, DecodeState st) {
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, j = threadIdx.x, K1 = a.K + 1, B = a.B, R = B * K1;
  if (j >= K1) return;
  const int r = b * K1 + j;
  a.row_tok[r] = (j >= 1 && j <= a.n_draft[b]) ? a.drafts[(long long)b * a.K + j - 1] : st.cur_tok[b];
  for (int ax = 0; ax < 3; ++ax) a.row_pos[ax * R + r] = st.pos3[ax * B + b] + j;
  a.row_idx[r] = st.cache_len[b] + j;
  a.row_col[r] = a.col[b] + j;
}

// one thread per running sequence: n_matches = the longest draft prefix equal to the rows' tokens; tokens 0 .. n_matches of the
// rows are recorded in order (record_token: output, stop test, cur_tok, cache_len and pos3 advance) until a stop id or max_new,
// and appended to the corpus.  A sequence that reaches max_new ends here (the plain loop ends by its step count instead).
__global__ void lookup_accept_kernel(LookupArgs a, ColumnSink k) {
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x, B = a.B;
  if (b >= B || k.st.finished[b]) return;
  const int K1 = a.K + 1, r0 = b * K1, nd = a.n_draft[b];
  int nm = 0;
  while (nm < nd && a.drafts[(long long)b * a.K + nm] == a.row_out[r0 + nm]) ++nm;
  int col = a.col[b], len = a.corpus_len[b], emitted = 0;
  for (int i = 0; i <= nm && col < k.max_new; ++i) {
    const int tok = a.row_out[r0 + i];
    if (a.logprobs != nullptr) a.logprobs[(long long)b * k.max_new + col] = a.row_lp[r0 + i];
    record_token<false>(k, B, b, col, tok, true, false, false);
    a.corpus[(long long)b * a.ld + len++] = tok;
    ++col; ++emitted;
    if (k.st.finished[b]) break;
  }
  if (!k.st.finished[b] && col >= k.max_new) { k.st.finished[b] = 1; atomicSub(k.st.n_active, 1); }
  a.col[b] = col; a.corpus_len[b] = len;
  a.steps[b] += 1;
  a.accepted[b] += emitted - 1;
}

int lookup_check(const fo1_generate_desc* d, const fo1_lookup_desc* lk) {
  FO1_CHECK_ARG(lk->num_tokens >= 1, "fo1_llm_generate: lookup: num_tokens %d must be >= 1", lk->num_tokens);
  FO1_CHECK_ARG(lk->max_ngram >= 1, "fo1_llm_generate: lookup: max_ngram %d must be >= 1", lk->max_ngram);
  FO1_CHECK_ARG(d->n_seqs > 0 && d->seq_lens, "fo1_llm_generate: lookup: null argument");
  FO1_CHECK_ARG(lk->corpus_offsets != nullptr, "fo1_llm_generate: lookup: null corpus_offsets");
  FO1_CHECK_ARG(lk->corpus_offsets[0] == 0, "fo1_llm_generate: lookup: corpus_offsets[0] = %d must be 0", lk->corpus_offsets[0]);
  for (int b = 0; b < d->n_seqs; ++b)
    FO1_CHECK_ARG(lk->corpus_offsets[b + 1] >= lk->corpus_offsets[b], "fo1_llm_generate: lookup: corpus_offsets decrease at sequence %d", b);
  FO1_CHECK_ARG(lk->corpus != nullptr || lk->corpus_offsets[d->n_seqs] == 0, "fo1_llm_generate: lookup: null corpus");
  return FO1_OK;
}

int lookup_upload(const LookupArgs& a, const fo1_lookup_desc* lk, cudaStream_t s) {
  std::vector<int> h((size_t)a.B * a.ld, 0), lens(a.B);
  for (int b = 0; b < a.B; ++b) {
    const int o = lk->corpus_offsets[b];
    lens[b] = lk->corpus_offsets[b + 1] - o;
    std::copy(lk->corpus + o, lk->corpus + o + lens[b], h.begin() + (size_t)b * a.ld);
  }
  // from pageable memory: each copy returns once its source is staged, so the vectors may die with this call (issued before the
  // prefill, the copies find the stream idle; no synchronisation between the prefill and the decode loop)
  FO1_CUDA(cudaMemcpyAsync(a.corpus, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  FO1_CUDA(cudaMemcpyAsync(a.corpus_len, lens.data(), lens.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  return FO1_OK;
}

int lookup_init(const LookupArgs& a, const DecodeState& st, const SampleRowParams* samp, cudaStream_t s) {
  lookup_init_kernel<<<ceil_div(a.B, 128), 128, 0, s>>>(a, st, samp);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int lookup_drafts(const int* corpus, long long ld, const int* len, int B, int K, int max_ngram, const int* stop_ids, int n_stop,
                  const int* col, int max_new, int* drafts, int* n_draft, cudaStream_t s) {
  if (B == 0) return FO1_OK;
  launch_k(lookup_drafts_kernel, dim3(B), dim3(256), 0, s, corpus, ld, len, K, max_ngram, stop_ids, n_stop, col, max_new, drafts, n_draft);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int lookup_rows(const LookupArgs& a, const DecodeState& st, cudaStream_t s) {
  launch_k(lookup_rows_kernel, dim3(a.B), dim3(32), 0, s, a, st);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int lookup_accept(const LookupArgs& a, const ColumnSink& k, cudaStream_t s) {
  launch_k(lookup_accept_kernel, dim3(ceil_div(a.B, 128)), dim3(128), 0, s, a, k);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1

using namespace fo1;

extern "C" int fo1_lookup_drafts(const int32_t* corpus, int64_t ld, const int32_t* lens, int32_t n_seqs, int32_t num_tokens, int32_t max_ngram,
                                 const int32_t* stop_ids, int32_t n_stop, const int32_t* emitted, int32_t max_new_tokens, int32_t* drafts,
                                 int32_t* n_draft, void* stream) {
  FO1_CHECK_ARG(n_seqs >= 0 && n_seqs <= 65535, "fo1_lookup_drafts: n_seqs %d out of range [0, 65535]", n_seqs);
  FO1_CHECK_ARG(num_tokens >= 1 && num_tokens <= kLookupMaxDrafts, "fo1_lookup_drafts: num_tokens %d out of range [1, %d]", num_tokens,
                kLookupMaxDrafts);
  FO1_CHECK_ARG(max_ngram >= 1, "fo1_lookup_drafts: max_ngram %d must be >= 1", max_ngram);
  FO1_CHECK_ARG(n_stop >= 0 && (n_stop == 0 || stop_ids), "fo1_lookup_drafts: null stop_ids");
  if (n_seqs == 0) return FO1_OK;
  FO1_CHECK_ARG(corpus && lens && drafts && n_draft && ld > 0, "fo1_lookup_drafts: null argument");
  return lookup_drafts(corpus, ld, lens, n_seqs, num_tokens, max_ngram, stop_ids, n_stop, emitted, max_new_tokens, drafts, n_draft,
                       static_cast<cudaStream_t>(stream));
}
