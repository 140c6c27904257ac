// lookup.cuh -- prompt-lookup decoding (HF generate's prompt_lookup_num_tokens) on the per-kernel decode path.
//
// Each step drafts up to K tokens per sequence from its own corpus (the prompt ids, then every token emitted so far) with HF's
// PromptLookupCandidateGenerator rule, runs ONE verify step over B * (K + 1) rows -- row (b, j) feeds cur_tok[b] (j = 0) or draft j
// at position next + j, with its K/V at cache index cache_len[b] + j -- and emits the longest draft prefix the rows' own tokens
// confirm plus one more token.  Every verify row computes the bits the plain step would compute at its position (same per-row
// kernels, GEMMs pinned to the plain step's tile width and split-K, the decode attention's key split taken from B sequences, the
// sampler's Philox counter = the row's own column), so the tokens are those of plain decoding, greedy or sampled.
#pragma once
#include "decode_loop.cuh"
#include "sampling.cuh"

namespace fo1 {

constexpr int kLookupMaxDrafts = 16;   // drafts per sequence and step; a larger num_tokens proposes this many

// the device state of a lookup call (one arena carve-out; R = B * (K + 1) verify rows, row r = b * (K + 1) + j)
struct LookupArgs {
  int B, K, max_ngram, max_new;
  int* corpus;         // [B][ld]: the prompt ids, then every emitted token
  long long ld;
  int* corpus_len;     // [B]
  int* col;            // [B] the sequence's next output column
  int* drafts;         // [B][K]
  int* n_draft;        // [B]
  int* row_tok;        // [R] input token of each verify row
  int* row_pos;        // [3][R] its M-RoPE position
  int* row_slot;       // [R] its cache slot (b)
  int* row_idx;        // [R] the cache index of its K/V
  int* row_col;        // [R] its output column (the sampler's Philox counter)
  int* row_out;        // [R] the token each row chose
  float* row_lp;       // [R] scored: the log-probability of that token
  SampleRowParams* row_prm;   // [R] sampled: the sequence's parameters, once per row
  float* logprobs;     // scored: the caller's [B][max_new]
  int* steps;          // [B] verify steps the sequence took part in
  int* accepted;       // [B] drafts accepted
};

// host: the checks of fo1_llm_generate with d.lookup (no CUDA call)
int lookup_check(const fo1_generate_desc* d, const fo1_lookup_desc* lk);
// the arena carve-out (sized by the dry run like every other buffer)
template <typename ArenaT>
void lookup_alloc(ArenaT& A, LookupArgs& a, const fo1_lookup_desc* lk) {
  const int R = a.B * (a.K + 1);
  a.corpus = A.template alloc<int>((size_t)a.B * a.ld);
  a.corpus_len = A.template alloc<int>(a.B); a.col = A.template alloc<int>(a.B);
  a.drafts = A.template alloc<int>((size_t)a.B * a.K); a.n_draft = A.template alloc<int>(a.B);
  a.row_tok = A.template alloc<int>(R); a.row_pos = A.template alloc<int>((size_t)3 * R); a.row_slot = A.template alloc<int>(R);
  a.row_idx = A.template alloc<int>(R); a.row_col = A.template alloc<int>(R); a.row_out = A.template alloc<int>(R);
  a.row_lp = A.template alloc<float>(R); a.row_prm = A.template alloc<SampleRowParams>(R);
  a.steps = lk->steps != nullptr ? lk->steps : A.template alloc<int>(a.B);
  a.accepted = lk->accepted != nullptr ? lk->accepted : A.template alloc<int>(a.B);
}
// before the prefill: the corpora (host packed ids + offsets) into the device buffer [B][ld] and their lengths
int lookup_upload(const LookupArgs& a, const fo1_lookup_desc* lk, cudaStream_t s);
// after the prefill's column 0: append column 0 to each corpus, reset the columns and counters
int lookup_init(const LookupArgs& a, const DecodeState& st, const SampleRowParams* samp, cudaStream_t s);
// drafts [B][K] and n_draft [B] from the corpora (col == nullptr: no cap by max_new)
int lookup_drafts(const int* corpus, long long ld, const int* len, int B, int K, int max_ngram, const int* stop_ids, int n_stop,
                  const int* col, int max_new, int* drafts, int* n_draft, cudaStream_t s);
// the verify rows' tokens, positions, cache indices and columns
int lookup_rows(const LookupArgs& a, const DecodeState& st, cudaStream_t s);
// acceptance and the recording of the emitted tokens (one thread per sequence)
int lookup_accept(const LookupArgs& a, const ColumnSink& k, cudaStream_t s);
// scored verify rows: the draw at column row_col[r] with sequence r / K1's parameters, scores / logits rows at (column, sequence),
// the token's log-probability into row_lp (lookup_accept writes the emitted ones)
int score_rows_lookup(const float* logits, long long ld, int n_rows, int K1, int V, const SampleRowParams* prm, const int* row_col,
                      int* tok, float* row_lp, const int* finished, int max_new, int n_seqs, float* scores, float* logits_out, cudaStream_t s);

}  // namespace fo1
