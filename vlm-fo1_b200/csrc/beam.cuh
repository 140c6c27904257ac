// beam.cuh -- beam search in the per-kernel decode loop (beam.cu): the device state of a beam-search call and its launchers.
//
// The contract is transformers' GenerationMixin._beam_search (generation/utils.py: _get_top_k_continuations,
// _get_running_beams_for_next_iteration, _update_finished_beams, _check_early_stop_heuristic,
// _beam_search_has_unfinished_sequences), run per prompt as if the prompt were alone in the call.  Every fp32 operation is the
// cited code's, in its order; where torch.topk leaves the order of equal scores unspecified, the device uses the sampler's
// canonical order: score descending, then flat index (beam * V + token, or the merged position) ascending.
//
// Rows: prompt b owns the N decode rows / cache slots b * N .. b * N + N - 1.  One output column is three launches plus a
// one-thread step increment:
//   beam_rows_kernel    one CTA per row: max, the fixed-point Z of the raw row, the log-prob row lp (written to `scores` when
//                       asked for), acc = lp + running score, and the row's top K of acc by the sampler's radix cut.
//   beam_select_kernel  one CTA per prompt: the top K of its N * K candidates, the stop test, the running set, the finished
//                       set with length penalty, the early-stop heuristic, and the new beams' tokens and parents.
//   beam_kv_reorder_kernel  child <- parent K/V of the generated rows [L_b, L_b + t) in every layer (prompt rows are equal across
//                       a prompt's slots and are never copied); one CTA stages every parent row of its (layer, prompt, row range)
//                       in shared memory before it writes any child, so no parent is overwritten before it is read.
// Histories are kept as per-step (token, parent) records of the running beams; beam_finalize_kernel walks the parents back.
#pragma once
#include "decode_loop.cuh"
#include "engine.cuh"

namespace fo1 {

constexpr int kBeamMaxBeams = 16;      // N
constexpr int kBeamMaxKeep = 128;      // K: N * K <= 2048 candidates per prompt in the select's shared memory

struct BeamArgs {
  int S, N, K, V, max_new, num_return, early_stopping, lp_positive, n_stop, pad_id;
  const int* prompt_len;               // [S]
  const float* lp_div;                 // [max_new + 1]: (float)pow((double)i, (double)length_penalty)
  const int* stop_ids;                 // [n_stop]
  float* acc;                          // [R][V] scratch: lp + running score
  float *cand_score, *cand_lp;         // [R][K], each row in canonical order
  int* cand_tok;
  float* run_score;                    // [R]
  int *hist_tok, *hist_par;            // [max_new][R]: token / parent beam (0..N-1) of running beam r chosen at step t
  float* hist_lp;
  int* parent;                         // [R]: the parent of running beam r at the current step (the reorder's source)
  float *fin_score, *fin_lp;           // [S][N]: the finished set, best first
  int *fin_len, *fin_tok, *fin_par, *fin_done;
  int *unsat, *done;                   // [S]: early-stop heuristic unsatisfied, prompt done
  bf16 *kc, *vc;                       // layer 0 of the K / V cache
  long long layer_stride;
  int layers, cap, kv_dim;
  // outputs (fo1_beam_desc / fo1_generate_desc)
  int *steps_run, *out_tokens, *out_lens, *beam_indices;
  float *seq_scores, *out_logprobs, *scores, *logits;
};

int beam_check(const fo1_generate_desc* d, const fo1_beam_desc* bm, int vocab);        // host argument checks, no CUDA call
void beam_alloc(Arena& A, BeamArgs& a);                                                  // the arena buffers (sizes from a.S/N/K/V/max_new)
int beam_init(const BeamArgs& a, const DecodeState& st, const int* seq_lens, const int* deltas, cudaStream_t s);
int beam_column(const BeamArgs& a, const float* logits, const DecodeState& st, int advance, cudaStream_t s);
int beam_finalize(const BeamArgs& a, cudaStream_t s);

}  // namespace fo1
