// decode_mega.cuh -- argument block of the persistent decode kernel (decode_mega.cu), filled by llm.cu.
#pragma once
#include "engine.cuh"
#include "decode_loop.cuh"
#include "processors.cuh"
#include "sampling.cuh"

namespace fo1 {

constexpr int kMgMaxSplits = 8;

struct MegaLayer { const bf16 *qkv_w, *qkv_b, *o_w, *gu_w, *down_w; };

struct MegaArgs {
  int B, layers, H, QD, KD, hd, q_heads, kv_heads, I, V;
  float eps, theta;
  int sec_t, sec_h;
  const MegaLayer* layer;     // [layers] (device)
  const bf16* head_w;         // [V][H], rows scaled by the final norm gain
  const bf16* embed;          // [V][H]
  bf16 *kc, *vc;              // K / V cache [layers][B][cap][KD] (K rotated)
  long long kv_layer_stride;
  int cap;
  // activations (global, L2 resident)
  bf16 *x, *x_mid, *qkv, *att, *h;
  float* ssq;                 // [2][grid][32] partial row sums of squares: [0] residual stream entering a layer, [1] after attention
  float* cs;                  // [2][B][hd/2] cos | sin of the current positions
  float* att_part;            // [B][q_heads][kMgMaxSplits][hd + 4]
  int* att_count;             // [B][kv_heads] arrival counters (self-resetting)
  float* amax_val; int* amax_idx;   // [grid][32]
  ColumnSink sink;            // loop state, outputs and (STREAM) their mirror; CTA 0 records every column
  int n_steps;                // decode iterations to run at most
  int exit_at;                // the loop ends once at most this many sequences are running (0: all stopped)
  unsigned* bar;              // grid barrier counter (zeroed by the host before the launch)
  int n_splits;
  unsigned long long* prof;   // [grid][prof_slots][2] barrier enter / leave stamps of the first iteration (FO1_MEGA_PROF; nullptr: off)
  int prof_slots;
  // sampled decoding (MODE DEC_SAMPLED or DEC_SCORED; all nullptr for greedy)
  float* logits;                    // [B][V] fp32 head output
  const SampleRowParams* samp;      // [B] per-sequence temperature, top-p, top-k, seed
  int* samp_tok;                    // [B] the token CTA b drew for sequence b
  // scored decoding (MODE DEC_SCORED; any may be nullptr): logprobs [B][max_new], scores / logits [max_new][B][V]
  float *sc_logprobs, *sc_scores, *sc_logits;
  // logits processors (MODE DEC_SAMPLED or DEC_SCORED; proc.tab == nullptr: none): CTA b edits row b before it draws, and stores the
  // raw row in sc_logits first
  ProcArgs proc;
};


int decode_mega_grid();                                   // CTAs of the cooperative launch (0: not available on this device)
// the model shapes the persistent kernel runs: hidden H, q / kv heads of hd, intermediate I, vocabulary V.  The one place that
// decides it; a model outside it decodes on the per-kernel path
bool decode_mega_supports(int H, int hd, int q_heads, int kv_heads, int I, int V);
// the whole decode loop, one launch (streamed when a.sink.stream.progress != nullptr); FO1_MEGA_PROF=1 reports where the first
// iteration spent its time on stderr (a.prof is set here)
int decode_mega_run(MegaArgs a, DecodeMode mode, cudaStream_t s);

}  // namespace fo1
