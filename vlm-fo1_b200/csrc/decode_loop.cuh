// decode_loop.cuh -- decode loop state and the recording of an output column: decode_update_kernel (llm.cu) and decode_mega_kernel.
#pragma once
#include "common.cuh"

namespace fo1 {

// how a column's tokens are chosen (a scored greedy call samples with top_k 1 on raw rows: the arg-max, bit for bit); DEC_BEAM: beam
// search (beam.cuh), per-kernel path only
enum DecodeMode { DEC_GREEDY, DEC_SAMPLED, DEC_SCORED, DEC_BEAM };

struct DecodeState {
  int* cache_len;  // [B] K/V entries in the cache
  int* pos3;       // [3][B] M-RoPE position of the next input token (all axes equal after the prompt, :1848-1860)
  int* cur_tok;    // [B] token to feed next
  int* new_tok;    // [B] the per-kernel path's token of the column being recorded
  int* finished;   // [B]
  int* n_active;   // [1] sequences still running
  int* step;       // [1] index of the next output column
  int* stop_ids;   // [n_stop]
};

// Streamed decoding (fo1_stream_desc, include/fo1.h): the device aliases of the caller's mapped, pinned host buffers.  The code
// that records output column t mirrors it into tokens / lens, fences at system scope and release-stores progress = (t + 1) | done.
struct StreamArgs {
  int* tokens;          // [B][max_new] mirror of out_tokens
  int* lens;            // [B] mirror of out_lens
  int* progress;        // columns published | FO1_STREAM_DONE (nullptr: not streamed)
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

// everything recording a column touches
struct ColumnSink {
  DecodeState st;
  int n_stop, pad_id, max_new;
  int *out_tokens, *out_lens;     // [B][max_new], [B]
  StreamArgs stream;
  // slot pool (nullptr: a generate call): slot b's own output column col[b] -- its output index and its Philox step -- and its own
  // limit max_new_row[b] <= max_new (the pitch of out_tokens)
  int *col, *max_new_row;
};

// Recording column `step` is one block's work: column_prologue and column_epilogue by every thread, record_token in between by one
// thread per sequence.  STREAM: published only while a sequence is active (nothing after `done`); cancel is read once per column.
template <bool STREAM>
__device__ __forceinline__ void column_prologue(const ColumnSink& k, int step, bool& publish, bool& cancel) {
  if constexpr (STREAM) {
    __shared__ int s_stream[2];
    if (threadIdx.x == 0) {
      s_stream[0] = __ldcg(k.st.n_active) > 0 && step < k.max_new;
      s_stream[1] = stream_cancel_requested(k.stream.cancel);
    }
    __syncthreads();
    publish = s_stream[0] != 0;
    cancel = publish && s_stream[1] != 0;
  }
  __syncthreads();
}

// sequence b's token: output (pad once finished), stop test, mirror, next input; `advance`: a decode step produced it (not the prefill)
template <bool STREAM>
__device__ __forceinline__ void record_token(const ColumnSink& k, int B, int b, int step, int tok, bool advance, bool publish, bool cancel) {
  const DecodeState& st = k.st;
  if (k.col != nullptr) {     // slot pool: a finished slot is idle (its row stays as recorded, its cache stops growing) until refilled
    if (st.finished[b]) return;
    const int c = k.col[b];
    k.out_tokens[(long long)b * k.max_new + c] = tok;
    k.out_lens[b] = c + 1;
    k.col[b] = c + 1;
    bool stop = c + 1 >= k.max_new_row[b];
    for (int i = 0; i < k.n_stop; ++i) stop |= (tok == st.stop_ids[i]);
    if (stop) { st.finished[b] = 1; atomicSub(st.n_active, 1); }
    st.cur_tok[b] = tok;
    if (advance) {
      st.cache_len[b] += 1;
      st.pos3[b] += 1; st.pos3[B + b] += 1; st.pos3[2 * B + b] += 1;
    }
    return;
  }
  if (step < k.max_new) {
    if (!st.finished[b]) {
      k.out_tokens[(long long)b * k.max_new + step] = tok;
      k.out_lens[b] = step + 1;
      bool stop = false;
      for (int i = 0; i < k.n_stop; ++i) stop |= (tok == st.stop_ids[i]);
      if constexpr (STREAM) stop |= cancel;                  // a cancelled sequence ends after this column
      if (stop) { st.finished[b] = 1; atomicSub(st.n_active, 1); }
      if constexpr (STREAM) {
        if (publish) { k.stream.tokens[(long long)b * k.max_new + step] = tok; k.stream.lens[b] = step + 1; }
      }
    } else {
      k.out_tokens[(long long)b * k.max_new + step] = k.pad_id;
      if constexpr (STREAM) {
        if (publish) k.stream.tokens[(long long)b * k.max_new + step] = k.pad_id;
      }
    }
  }
  st.cur_tok[b] = tok;
  if (advance) {
    st.cache_len[b] += 1;
    st.pos3[b] += 1; st.pos3[B + b] += 1; st.pos3[2 * B + b] += 1;
  }
}

// the bar.sync covers every thread's mirror writes before the publish
template <bool STREAM>
__device__ __forceinline__ void column_epilogue(const ColumnSink& k, int step, bool publish, bool cancel) {
  __syncthreads();
  if (threadIdx.x == 0) *k.st.step = step + 1;
  if constexpr (STREAM) {
    if (threadIdx.x == 0 && publish) {
      const bool done = cancel || __ldcg(k.st.n_active) <= 0 || step + 1 >= k.max_new;
      stream_publish(k.stream.progress, (step + 1) | (done ? FO1_STREAM_DONE : 0));
    }
  }
}

}  // namespace fo1
