// processors.cuh -- HF generate's logits processors on the device: one row of fp32 logits edited in place from its sequence's history.
// Shared by logits_process_kernel (processors.cu: the per-kernel decode step, column 0 after a prefill, fo1_logits_process) and the
// persistent decode kernel (decode_mega.cu, CTA b on row b before it draws).
//
// The contract is transformers' GenerationMixin._get_logits_processor, in its order:
//   SequenceBias -> NoRepeatNGram -> NoBadWords -> MinLength -> MinNewTokensLength -> SuppressTokens -> SuppressTokensAtBegin
// over HF's input_ids = the caller's prompt ids (placeholders included), then the L - Lp tokens emitted so far (L the history length,
// col = L - Lp the output column).  Every edit is x -> x + bias (fp32, the per-token sum formed as HF forms it: the length-1 bias
// first, then the multi-token sequences in their given order, each added to a zero start) or x -> -inf.  Every -inf edit commutes
// with the others and absorbs a finite bias, so only the bias pass is ordered (a barrier before the -inf passes).
//   SequenceBias / NoBadWords: sequence w (length m) applies when m == 1, or m <= L and the last m - 1 history ids equal w[0 .. m - 1);
//     it edits token w[m - 1].
//   NoRepeatNGram(n): when L + 1 >= n, every i with h[i .. i + n - 1) == h[L - n + 1 .. L) bans h[i + n - 1] (a negative id bans
//     V + id: HF's index wrap).
//   MinLength: eos ids -> -inf while L < min_length.  MinNewTokens: while col < min_new_tokens.  SuppressTokens: always.
//   SuppressTokensAtBegin: at col == 0.
#pragma once
#include <vector>

#include "common.cuh"

namespace fo1 {

// The packed sets (processors.cu builds them).  tab[0] = the offset of the sequence pairs; set s is the kProcSetInts ints at
// tab[1 + kProcSetInts * s]: n-gram size, min_length, min_new_tokens, then [begin, end) of the eos, suppress and begin-suppress id
// lists (offsets into tab), of the bias sequences and of the bad-word sequences (indices of the pairs).  Pair k = tab[base + 2k],
// tab[base + 2k + 1]: the ids' [begin, end) in tab; bias[k] its fp32 bias.  A set's bias sequences are grouped by last token, each
// group in HF's order, so one thread forms each biased token's sum.
constexpr int kProcSetInts = 13;
enum { PS_NGRAM, PS_MIN_LEN, PS_MIN_NEW, PS_EOS0, PS_EOS1, PS_SUP0, PS_SUP1, PS_BSUP0, PS_BSUP1, PS_BIAS0, PS_BIAS1, PS_BAD0, PS_BAD1 };

struct ProcArgs {
  const int* tab;        // nullptr: no processing in this call
  const float* bias;
  const int* set_of;     // [rows] the row's set, -1: never edited
  const int* prompt;     // [rows][ld] the caller's prompt ids
  const int* plen;       // [rows]
  long long ld;
};

#ifdef __CUDACC__
// Row b's processors at output column col: history = prompt[b][0 .. plen[b]) then out_row[0 .. col).  Every thread of the CTA calls it.
// raw_out (optional): the unedited row is copied there first (HF's output_logits), whether or not the row has a set.
template <int NT>
__device__ void process_row(const ProcArgs& p, int b, int col, float* __restrict__ row, int V, const int* __restrict__ out_row,
                            float* __restrict__ raw_out) {
  const int tid = threadIdx.x;
  if (raw_out != nullptr) {
    for (int i = tid; i < V; i += NT) raw_out[i] = __ldcg(row + i);
    __syncthreads();
  }
  const int set = __ldg(p.set_of + b);
  if (set < 0) return;
  const int* tab = p.tab;
  const int* S = tab + 1 + kProcSetInts * set;
  const int* pr = p.prompt + (long long)b * p.ld;
  const int Lp = __ldg(p.plen + b), L = Lp + col;
  auto h = [&](int j) -> int { return j < Lp ? __ldg(pr + j) : __ldcg(out_row + (j - Lp)); };
  const int* pairs = tab + __ldg(tab);
  // sequence k applies: length 1, or its prefix is the history's tail
  auto applies = [&](int k) -> bool {
    const int w0 = __ldg(pairs + 2 * k), m = __ldg(pairs + 2 * k + 1) - w0;
    if (m == 1) return true;
    if (m > L) return false;
    for (int j = 0; j < m - 1; ++j)
      if (h(L - m + 1 + j) != __ldg(tab + w0 + j)) return false;
    return true;
  };
  auto last_of = [&](int k) -> int { return __ldg(tab + __ldg(pairs + 2 * k + 1) - 1); };
  // ---- SequenceBias: the first thread of each last-token group sums the group in order and adds it once ----
  const int bias0 = __ldg(S + PS_BIAS0), bias1 = __ldg(S + PS_BIAS1);
  if (bias1 > bias0) {
    for (int k = bias0 + tid; k < bias1; k += NT) {
      const int t = last_of(k);
      if (k > bias0 && last_of(k - 1) == t) continue;
      float acc = 0.f;
      for (int j = k; j < bias1 && last_of(j) == t; ++j)
        if (applies(j)) acc += __ldg(p.bias + j);
      row[t] = __ldcg(row + t) + acc;
    }
    __syncthreads();
  }
  // ---- NoRepeatNGram: every earlier n-gram whose first n - 1 ids are the history's last n - 1 bans its last id ----
  const int n = __ldg(S + PS_NGRAM);
  if (n > 0 && L + 1 >= n) {
    for (int i = tid; i + n <= L; i += NT) {
      bool eq = true;
      for (int j = 0; j < n - 1 && eq; ++j) eq = h(i + j) == h(L - n + 1 + j);
      if (eq) {
        const int t = h(i + n - 1);
        row[t < 0 ? t + V : t] = -INFINITY;
      }
    }
  }
  // ---- NoBadWords ----
  for (int k = __ldg(S + PS_BAD0) + tid; k < __ldg(S + PS_BAD1); k += NT)
    if (applies(k)) row[last_of(k)] = -INFINITY;
  // ---- MinLength, MinNewTokensLength (the eos ids), SuppressTokens, SuppressTokensAtBegin ----
  if (L < __ldg(S + PS_MIN_LEN) || col < __ldg(S + PS_MIN_NEW))
    for (int i = __ldg(S + PS_EOS0) + tid; i < __ldg(S + PS_EOS1); i += NT) row[__ldg(tab + i)] = -INFINITY;
  for (int i = __ldg(S + PS_SUP0) + tid; i < __ldg(S + PS_SUP1); i += NT) row[__ldg(tab + i)] = -INFINITY;
  if (col == 0)
    for (int i = __ldg(S + PS_BSUP0) + tid; i < __ldg(S + PS_BSUP1); i += NT) row[__ldg(tab + i)] = -INFINITY;
  __syncthreads();
}
#endif

// ---- host (processors.cu) ----
// One set as the host keeps it (the pool deduplicates these); bias sequences in HF's order.
struct ProcSet {
  int ngram = 0, min_len = 0, min_new = 0;
  std::vector<int> eos, sup, bsup;
  std::vector<std::vector<int>> bias_seq, bad;
  std::vector<float> bias;
  std::vector<int> key() const;     // a serialisation for deduplication
};
// validation of a fo1_processor_desc for n_seqs sequences and vocabulary V (no CUDA call), then its sets
int proc_check(const fo1_processor_desc* pr, int n_seqs, int V, const char* fn);
std::vector<ProcSet> proc_sets(const fo1_processor_desc* pr);
// the device table of `sets` (tab, bias) as process_row reads it
void proc_table(const std::vector<ProcSet>& sets, std::vector<int>& tab, std::vector<float>& bias);
// rows [n_rows] of `logits` (pitch V): row r is sequence row_slot[r] (nullptr: r) at column col[b * col_stride]; rows with
// finished[b] or column >= max_new are skipped (finished == nullptr: none).  raw_out: rows at ((col * n_rows + r) * V).
int logits_process(const ProcArgs& p, float* logits, int n_rows, int V, const int* col, int col_stride, const int* row_slot,
                   const int* finished, int max_new, const int* out_tokens, float* raw_out, cudaStream_t s);

}  // namespace fo1
