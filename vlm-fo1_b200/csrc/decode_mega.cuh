// decode_mega.cuh -- argument block of the persistent decode kernel (decode_mega.cu), filled by llm.cu.
#pragma once
#include "engine.cuh"
#include "sampling.cuh"

namespace fo1 {

constexpr int kMgMaxSplits = 8;

struct MegaLayer { const bf16 *qkv_w, *qkv_b, *o_w, *gu_w, *down_w; };

// Streamed decoding (fo1_stream_desc, include/fo1.h): the device aliases of the caller's mapped, pinned host buffers.  The code
// that records output column t mirrors it into tokens / lens, fences at system scope and release-stores progress = (t + 1) | done.
struct StreamArgs {
  int* tokens;          // [B][max_new] mirror of out_tokens
  int* lens;            // [B] mirror of out_lens
  int* progress;        // columns published | FO1_STREAM_DONE
  const int* cancel;    // optional: != 0 asks the loop to stop after the column it records next
};
__device__ __forceinline__ int stream_cancel_requested(const int* cancel) {
  int v = 0;
  if (cancel != nullptr) asm volatile("ld.relaxed.sys.global.b32 %0, [%1];" : "=r"(v) : "l"(cancel) : "memory");
  return v;
}
// by ONE thread after the bar.sync that follows the block's mirror writes: the system-scope fence and the release are cumulative, so
// they order every thread's writes the barrier made visible to this one (one fence per step instead of one per writing warp)
__device__ __forceinline__ void stream_publish(int* progress, int v) {
  __threadfence_system();
  asm volatile("st.release.sys.global.b32 [%0], %1;" ::"l"(progress), "r"(v) : "memory");
}

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
  // loop state (DecodeState of llm.cu) and outputs
  int *cache_len, *pos3, *cur_tok, *finished, *n_active, *step;
  const int* stop_ids; int n_stop, pad_id, max_new;
  int* out_tokens; int* out_lens;
  int n_steps;                // decode iterations to run at most
  unsigned* bar;              // grid barrier counter (zeroed by the host before the launch)
  int n_splits;
  unsigned long long* prof;   // optional [grid][prof_slots][2] barrier enter / leave stamps of the first iteration (nullptr: off)
  int prof_slots;
  // sampled decoding (decode_mega_kernel<MT, true>; all nullptr for greedy)
  float* logits;                    // [B][V] fp32 head output
  const SampleRowParams* samp;      // [B] per-sequence temperature, top-p, top-k, seed
  int* samp_tok;                    // [B] the token CTA b drew for sequence b
  // scored decoding (decode_mega_kernel<MT, true, true>; any may be nullptr): logprobs [B][max_new], scores / logits [max_new][B][V]
  float *sc_logprobs, *sc_scores, *sc_logits;
  // streamed decoding (decode_mega_kernel<MT, SAMPLE, SCORE, true>; progress == nullptr otherwise)
  StreamArgs stream;
};


int decode_mega_grid();                                   // CTAs of the cooperative launch (0: not available on this device)
int decode_mega_run(const MegaArgs& a, cudaStream_t s);   // the whole decode loop, one launch (sampled when a.samp != nullptr,
                                                          // streamed when a.stream.progress != nullptr)

}  // namespace fo1
