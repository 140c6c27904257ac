// processors.cu -- logits processors (processors.cuh): the host checks and tables, logits_process_kernel, fo1_logits_process.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "processors.cuh"

namespace fo1 {

constexpr int kProcThreads = 256;

// One CTA per row: the decode step's processors ahead of its token choice (per-kernel path), column 0 after a prefill, or
// fo1_logits_process.  Reads the column from device memory, so a captured decode step replays it.
__global__ void __launch_bounds__(kProcThreads) logits_process_kernel(ProcArgs p, float* __restrict__ logits, long long ld, int V,
                                                                      const int* __restrict__ col_p, int col_stride,
                                                                      const int* __restrict__ row_slot, const int* __restrict__ finished,
                                                                      int max_new, const int* __restrict__ out_tokens, long long ld_out,
                                                                      float* __restrict__ raw_out) {
  griddep_launch();
  griddep_wait();
  const int r = blockIdx.x;
  const int b = row_slot != nullptr ? __ldg(row_slot + r) : r;
  const int col = __ldcg(col_p + (long long)b * col_stride);
  if (finished != nullptr && (col >= max_new || __ldcg(finished + b))) return;    // past the sequence's stop: nothing is recorded
  process_row<kProcThreads>(p, b, col, logits + (long long)r * ld, V, out_tokens + (long long)b * ld_out,
                            raw_out != nullptr ? raw_out + ((long long)col * gridDim.x + r) * V : nullptr);
}

int logits_process(const ProcArgs& p, float* logits, int n_rows, int V, const int* col, int col_stride, const int* row_slot,
                   const int* finished, int max_new, const int* out_tokens, float* raw_out, cudaStream_t s) {
  FO1_CHECK_ARG(n_rows <= 65535, "logits_process: %d rows exceed the grid limit", n_rows);
  launch_k(logits_process_kernel, dim3(n_rows), dim3(kProcThreads), 0, s, p, logits, (long long)V, V, col, col_stride, row_slot, finished,
           max_new, out_tokens, (long long)max_new, raw_out);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

static bool monotone(const int32_t* off, int n, int hi) {
  if (off == nullptr || off[0] < 0 || off[n] > hi) return false;
  for (int i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return false;
  return true;
}

int proc_check(const fo1_processor_desc* pr, int n_seqs, int V, const char* fn) {
  FO1_CHECK_ARG(pr->n_sets >= 1 && pr->n_ids >= 0 && pr->n_sequences >= 0, "%s: processors: n_sets %d / n_ids %d / n_sequences %d", fn,
                pr->n_sets, pr->n_ids, pr->n_sequences);
  FO1_CHECK_ARG(pr->seq_set && pr->prompt_offsets && pr->no_repeat_ngram_size && pr->min_length && pr->min_new_tokens, "%s: processors: null argument", fn);
  FO1_CHECK_ARG(pr->ids || pr->n_ids == 0, "%s: processors: null ids", fn);
  const int S = pr->n_sets;
  for (int b = 0; b < n_seqs; ++b)
    FO1_CHECK_ARG(pr->seq_set[b] >= -1 && pr->seq_set[b] < S, "%s: processors: sequence %d: set %d out of range [-1, %d)", fn, b, pr->seq_set[b], S);
  FO1_CHECK_ARG(pr->prompt_offsets[0] == 0, "%s: processors: prompt_offsets must start at 0", fn);
  for (int b = 0; b < n_seqs; ++b)
    FO1_CHECK_ARG(pr->prompt_offsets[b + 1] >= pr->prompt_offsets[b], "%s: processors: prompt_offsets decrease at sequence %d", fn, b);
  FO1_CHECK_ARG(pr->prompt || pr->prompt_offsets[n_seqs] == 0, "%s: processors: null prompt", fn);
  for (int i = 0; i < pr->prompt_offsets[n_seqs]; ++i)
    FO1_CHECK_ARG(pr->prompt[i] >= -V && pr->prompt[i] < V, "%s: processors: prompt id %d at %d out of range [-%d, %d)", fn, pr->prompt[i], i, V, V);
  for (int s = 0; s < S; ++s) {
    FO1_CHECK_ARG(pr->no_repeat_ngram_size[s] >= 0 && pr->min_length[s] >= 0 && pr->min_new_tokens[s] >= 0,
                  "%s: processors: set %d: no_repeat_ngram_size %d, min_length %d, min_new_tokens %d must be >= 0", fn, s,
                  pr->no_repeat_ngram_size[s], pr->min_length[s], pr->min_new_tokens[s]);
  }
  const int32_t* lists[3] = {pr->eos_offsets, pr->suppress_offsets, pr->begin_suppress_offsets};
  const char* names[3] = {"eos_offsets", "suppress_offsets", "begin_suppress_offsets"};
  for (int l = 0; l < 3; ++l)
    FO1_CHECK_ARG(monotone(lists[l], S, pr->n_ids), "%s: processors: %s missing, not non-decreasing or past n_ids", fn, names[l]);
  FO1_CHECK_ARG(monotone(pr->bias_offsets, S, pr->n_sequences) && monotone(pr->bad_offsets, S, pr->n_sequences),
                "%s: processors: bias_offsets / bad_offsets missing, not non-decreasing or past n_sequences", fn);
  FO1_CHECK_ARG(pr->n_sequences == 0 || (pr->seq_offsets && pr->bias && monotone(pr->seq_offsets, pr->n_sequences, pr->n_ids)),
                "%s: processors: seq_offsets / bias missing, not non-decreasing or past n_ids", fn);
  for (int k = 0; k < pr->n_sequences; ++k)
    FO1_CHECK_ARG(pr->seq_offsets[k + 1] > pr->seq_offsets[k], "%s: processors: sequence %d is empty", fn, k);
  for (int s = 0; s < S; ++s)
    for (int k = pr->bias_offsets[s]; k < pr->bias_offsets[s + 1]; ++k)
      FO1_CHECK_ARG(std::isfinite(pr->bias[k]), "%s: processors: sequence %d: bias %g is not finite", fn, k, (double)pr->bias[k]);
  for (int i = 0; i < pr->n_ids; ++i)
    FO1_CHECK_ARG(pr->ids[i] >= 0 && pr->ids[i] < V, "%s: processors: id %d at %d out of range [0, %d)", fn, pr->ids[i], i, V);
  return FO1_OK;
}

std::vector<int> ProcSet::key() const {
  std::vector<int> k = {ngram, min_len, min_new};
  auto list = [&](const std::vector<int>& v) { k.push_back((int)v.size()); k.insert(k.end(), v.begin(), v.end()); };
  list(eos); list(sup); list(bsup);
  k.push_back((int)bias_seq.size());
  for (size_t i = 0; i < bias_seq.size(); ++i) {
    int bits;
    memcpy(&bits, &bias[i], sizeof(bits));
    k.push_back(bits);
    list(bias_seq[i]);
  }
  k.push_back((int)bad.size());
  for (const auto& w : bad) list(w);
  return k;
}

std::vector<ProcSet> proc_sets(const fo1_processor_desc* pr) {
  std::vector<ProcSet> sets(pr->n_sets);
  auto ids = [&](int a, int b) { return std::vector<int>(pr->ids + a, pr->ids + b); };
  auto seq = [&](int k) { return ids(pr->seq_offsets[k], pr->seq_offsets[k + 1]); };
  for (int s = 0; s < pr->n_sets; ++s) {
    ProcSet& p = sets[s];
    p.ngram = pr->no_repeat_ngram_size[s]; p.min_len = pr->min_length[s]; p.min_new = pr->min_new_tokens[s];
    p.eos = ids(pr->eos_offsets[s], pr->eos_offsets[s + 1]);
    p.sup = ids(pr->suppress_offsets[s], pr->suppress_offsets[s + 1]);
    p.bsup = ids(pr->begin_suppress_offsets[s], pr->begin_suppress_offsets[s + 1]);
    for (int k = pr->bias_offsets[s]; k < pr->bias_offsets[s + 1]; ++k) { p.bias_seq.push_back(seq(k)); p.bias.push_back(pr->bias[k]); }
    for (int k = pr->bad_offsets[s]; k < pr->bad_offsets[s + 1]; ++k) p.bad.push_back(seq(k));
  }
  return sets;
}

void proc_table(const std::vector<ProcSet>& sets, std::vector<int>& tab, std::vector<float>& bias) {
  tab.assign(1 + kProcSetInts * sets.size(), 0);
  bias.clear();
  std::vector<const std::vector<int>*> seqs;     // the pairs, in order
  std::vector<int> rec;
  auto list = [&](const std::vector<int>& v, int at) {
    tab[at] = (int)tab.size();
    tab.insert(tab.end(), v.begin(), v.end());
    tab[at + 1] = (int)tab.size();
  };
  for (size_t s = 0; s < sets.size(); ++s) {
    const ProcSet& p = sets[s];
    const int o = 1 + kProcSetInts * (int)s;
    tab[o + PS_NGRAM] = p.ngram; tab[o + PS_MIN_LEN] = p.min_len; tab[o + PS_MIN_NEW] = p.min_new;
    list(p.eos, o + PS_EOS0); list(p.sup, o + PS_SUP0); list(p.bsup, o + PS_BSUP0);
    // bias sequences grouped by last token; within a group the length-1 sequence first, then the others in the given order (HF's
    // length_1_bias, then its loop over the multi-token sequences)
    std::vector<int> order(p.bias_seq.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
      const int ta = p.bias_seq[a].back(), tb = p.bias_seq[b].back();
      return ta != tb ? ta < tb : (p.bias_seq[a].size() == 1 && p.bias_seq[b].size() != 1);
    });
    tab[o + PS_BIAS0] = (int)seqs.size();
    for (int i : order) { seqs.push_back(&p.bias_seq[i]); bias.push_back(p.bias[i]); }
    tab[o + PS_BIAS1] = (int)seqs.size();
    tab[o + PS_BAD0] = (int)seqs.size();
    for (const auto& w : p.bad) { seqs.push_back(&w); bias.push_back(-INFINITY); }
    tab[o + PS_BAD1] = (int)seqs.size();
  }
  std::vector<int> pairs;
  for (const auto* w : seqs) {
    pairs.push_back((int)tab.size());
    tab.insert(tab.end(), w->begin(), w->end());
    pairs.push_back((int)tab.size());
  }
  tab[0] = (int)tab.size();
  tab.insert(tab.end(), pairs.begin(), pairs.end());
  if (bias.empty()) bias.push_back(0.f);
}

}  // namespace fo1

using namespace fo1;

extern "C" int fo1_logits_process(float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_processor_desc* pr,
                                  const int32_t* outputs, int64_t ld_out, const int32_t* cols, void* stream) {
  FO1_CHECK_ARG(pr && cols && logits, "fo1_logits_process: null argument");
  FO1_CHECK_ARG(n_rows > 0 && n_rows <= 65535, "fo1_logits_process: n_rows %d out of range [1, 65535]", n_rows);
  FO1_CHECK_ARG(vocab > 0 && ld >= vocab, "fo1_logits_process: vocab %d / ld %lld", vocab, (long long)ld);
  FO1_TRY(proc_check(pr, n_rows, vocab, "fo1_logits_process"));
  int max_col = 0;
  for (int r = 0; r < n_rows; ++r) {
    FO1_CHECK_ARG(cols[r] >= 0, "fo1_logits_process: row %d: column %d must be >= 0", r, cols[r]);
    max_col = std::max(max_col, cols[r]);
  }
  FO1_CHECK_ARG(max_col == 0 || (outputs && ld_out >= max_col), "fo1_logits_process: outputs / ld_out %lld for column %d", (long long)ld_out, max_col);
  std::vector<int> tab;
  std::vector<float> bias;
  proc_table(proc_sets(pr), tab, bias);
  long long lp = 1;
  for (int r = 0; r < n_rows; ++r) lp = std::max<long long>(lp, pr->prompt_offsets[r + 1] - pr->prompt_offsets[r]);
  // one int block: tab, set_of [n], plen [n], cols [n], prompts [n][lp]
  std::vector<int> h(tab);
  const size_t o_set = h.size(), o_len = o_set + n_rows, o_col = o_len + n_rows, o_pr = o_col + n_rows;
  h.resize(o_pr + (size_t)n_rows * lp, 0);
  for (int r = 0; r < n_rows; ++r) {
    const int a = pr->prompt_offsets[r], n = pr->prompt_offsets[r + 1] - a;
    h[o_set + r] = pr->seq_set[r]; h[o_len + r] = n; h[o_col + r] = cols[r];
    std::copy(pr->prompt + a, pr->prompt + a + n, h.begin() + o_pr + (size_t)r * lp);
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int* d = nullptr;
  float* db = nullptr;
  FO1_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d), h.size() * sizeof(int), s));
  int rc = FO1_OK;
  if (cudaMallocAsync(reinterpret_cast<void**>(&db), bias.size() * sizeof(float), s) != cudaSuccess ||
      cudaMemcpyAsync(d, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaMemcpyAsync(db, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, s) != cudaSuccess) {
    set_error("fo1_logits_process: table upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    rc = FO1_ERR_CUDA;
  } else {
    const ProcArgs p{d, db, d + o_set, d + o_pr, d + o_len, lp};
    launch_k(logits_process_kernel, dim3(n_rows), dim3(kProcThreads), 0, s, p, logits, (long long)ld, vocab, (const int*)(d + o_col), 1,
             (const int*)nullptr, (const int*)nullptr, 0, outputs, (long long)ld_out, (float*)nullptr);
    if (cudaGetLastError() != cudaSuccess) { set_error("fo1_logits_process: launch failed"); rc = FO1_ERR_CUDA; }
    else count_launch();
  }
  if (db) cudaFreeAsync(db, s);
  cudaFreeAsync(d, s);
  return rc;
}
