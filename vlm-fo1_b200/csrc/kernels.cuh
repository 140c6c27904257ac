// kernels.cuh -- internal launcher declarations shared by the engine (host side of every .cu file).
#pragma once
#include <cuda.h>

#include <vector>

#include "common.cuh"

namespace fo1 {

typedef __nv_bfloat16 bf16;

// ---- gemm_wgmma.cu ----
int gemm_bf16(const fo1_gemm_desc* d, cudaStream_t stream);
int device_sm_count();
// convenience: D = act(A.W^T + bias) + residual, all row-major contiguous unless ld given
int conv3x3_gemm(const bf16* x, int B, int H, int W, int C, const bf16* Wm, bf16* out, long long ldo, int N, cudaStream_t stream);   // -1000: shape does not tile
int linear(const bf16* A, long long lda, const bf16* W, long long ldw, void* D, long long ldd, int d_dtype, int M, int N,
           int K, const void* bias, int bias_dtype, int act, const bf16* residual, long long ldr, int gated,
           cudaStream_t stream);

// ---- norm.cu ----
// Qwen2RMSNorm (modeling_qwen2_5_vl.py:126-140): y = w * bf16(x * rsqrt(mean(x^2) + eps))
int rmsnorm(const bf16* x, long long ldx, const bf16* w, bf16* y, long long ldy, int rows, int cols, float eps, cudaStream_t s);
// nn.LayerNorm over the last dim (fp32 statistics), optional gamma/beta
int layernorm(const bf16* x, long long ldx, const bf16* gamma, const bf16* beta, bf16* y, long long ldy, int rows, int cols,
              float eps, cudaStream_t s);

// ---- rope.cu ----
// ViT 2-D RoPE (modeling_qwen2_5_vl.py:162-169, 436-463): table[t][j] = pos_{h|w}[t] * inv_freq[j mod half]
int vit_rope_table(const int* pos_hw /*[T][2]*/, float* cos_sin /*[T][rot_dim] cos then [T][rot_dim] sin*/, int T, int head_dim,
                   float theta, cudaStream_t s);
// rotate q and k inside a packed qkv buffer [T][3*heads*head_dim] (non-interleaved halves)
int vit_rope_apply(bf16* qkv, const float* cos_sin, int T, int heads, int head_dim, cudaStream_t s);
// LLM M-RoPE (modeling_qwen2_5_vl.py:603-624, 643-685): cos/sin table [T][hd/2] x2 from the 3-axis ids, built once per forward
int mrope_table(const int* pos3 /*[3][T]*/, float* cos_sin, int T, int head_dim, int sec_t, int sec_h, int sec_w, float theta, cudaStream_t s);
// rotate n_heads consecutive heads (q then k) of every row in place with a [T][hd/2] cos / sin table
int rope_apply(bf16* x, long long ld, const float* cos_sin, int T, int n_heads, int head_dim, cudaStream_t s);
// decode step: rotate q in place, append rotated K and V of row b to the cache at cache_len[b]
int rope_kv_append(bf16* qkv, long long ld, const float* cos_sin, int T, int q_heads, int kv_heads, int head_dim, const int* cache_len,
                   bf16* kc, bf16* vc, int cap, cudaStream_t s);

// ---- attention_tc.cu ----
// varlen flash attention over packed rows (wgmma / TMA); q/k/v may live in one packed buffer (pitches in elements)
struct AttnArgs {
  const bf16* q; const bf16* k; const bf16* v; bf16* o;
  long long ldq, ldk, ldv, ldo;     // row pitches (elements)
  const int* cu_seqlens;            // [n_seqs + 1] token offsets (device); q and kv share them
  const int* rowseg = nullptr;      // optional [total_rows][2] (lo, hi) table from attention_rowseg(); built per call when null
  const int* tiles = nullptr;       // optional [n_tiles][2] (first row, rows <= 128) query-tile table from attention_tile_table(); null:
  int n_tiles = 0;                  //   128-row tiles from row 0 (a sample's bits then depend on its offset in the batch)
  int n_seqs;
  int total_rows;                   // cu_seqlens[n_seqs] (host knowledge: sizes the grid and the tensor maps)
  int max_seqlen;                   // longest segment (informational)
  int q_heads, kv_heads, head_dim;
  float scale;
  int causal;
  double flops = 0.0;               // algorithmic FLOPs of the call for the optional profiler (4 * sum len^2 * hd * heads, / 2 causal)
};
int attention_varlen(const AttnArgs& a, cudaStream_t s);
// (lo, hi) key range of every packed row: callers that reuse one cu_seqlens for many layers build it once
int attention_rowseg(const int* cu_seqlens, int n_seqs, int T, int* rowseg, cudaStream_t s);
// host helper: 128-row query tiles that restart at every group boundary (image / prompt) -> flat (row0, rows) pairs
void attention_tile_table(const std::vector<int>& group_cu, std::vector<int>& tiles);

// ---- misc.cu ----
int cast_gather_rows_f32_bf16(const float* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols, cudaStream_t s);
int gather_rows_bf16(const bf16* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols, cudaStream_t s);
int scatter_rows_bf16(const bf16* src, long long lds, const int* row_idx, bf16* dst, long long ldd, int rows, int cols, cudaStream_t s);
int add_bf16(const bf16* a, const bf16* b, bf16* out, long long n, cudaStream_t s);
int gelu_bf16(const bf16* x, bf16* y, long long n, cudaStream_t s);

}  // namespace fo1

namespace fo1 {
// ---- conv.cu ----
int dwconv3x3_residual(const bf16* x, const bf16* w9, const bf16* bias, bf16* y, int B, int H, int W, int C, cudaStream_t s);
int im2col3x3(const bf16* x, bf16* col, int B, int H, int W, int C, int stride, cudaStream_t s);
int im2col_stem(const float* img, bf16* col, int H, int W, int kpad, cudaStream_t s);
int maxpool2x2(const bf16* x, bf16* y, int B, int H, int W, int C, cudaStream_t s);
// ---- chanattn_tc.cu: DaViT channel-group attention as two wgmma contractions; ws = channel_attention_ws_floats() floats
size_t channel_attention_ws_floats(int B, int N, int C);
int channel_attention(const bf16* qkv, float* ws, bf16* out, int B, int N, int C, int groups, cudaStream_t s);
int window_partition(const bf16* x, bf16* dst, int B, int H, int W, int C, int ws, cudaStream_t s);
int window_reverse_add(const bf16* x, const bf16* p, bf16* y, int B, int H, int W, int C, int ws, cudaStream_t s);
int pixel_shuffle2x(const bf16* src, bf16* dst, int B, int H, int W, int C, cudaStream_t s);
}  // namespace fo1
