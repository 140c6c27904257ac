// rope.cu -- rotary position embeddings: ViT 2-D RoPE and the LLM's multimodal 3-axis M-RoPE.
#include "kernels.cuh"

namespace fo1 {

// cos_sin layout: [T][half] cos followed by [T][half] sin, half = head_dim / 2.
// rot_pos_emb (modeling_qwen2_5_vl.py:436-463): rotary dim = head_dim/2; inv_freq[j] = theta^(-2j/rot), j < rot/2;
// entries [0, rot/2) use the h position, [rot/2, rot) the w position; emb = cat(rotary, rotary) so the
// pair (x[j], x[j + half]) is rotated by angle[j], j < half (qwen2_5_vl_encoder.py:110-116).
__global__ void vit_rope_table_kernel(const int* __restrict__ pos_hw, float* __restrict__ cs, int T, int half, float theta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * half) return;
  const int t = i / half, j = i - t * half;
  const int q = half / 2;
  const int jj = j < q ? j : j - q;
  const float inv = 1.0f / powf(theta, (float)(2 * jj) / (float)half);
  const float ang = (float)pos_hw[2 * t + (j < q ? 0 : 1)] * inv;
  cs[i] = cosf(ang);
  cs[(long long)T * half + i] = sinf(ang);
}

// x: rows of pitch ld holding n_heads consecutive heads of hd dims (q heads then k heads); rotates the pair
// (x[j], x[j + hd/2]) by angle[j] (rotate_half convention).  One thread = 8 consecutive j: 16-byte loads/stores.
__global__ void __launch_bounds__(256) rope_apply_kernel(bf16* __restrict__ x, long long ld, const float* __restrict__ cs, int T,
                                                         int n_heads, int hd) {
  const int half = hd / 2, chunks = half / 8;
  const long long n = (long long)T * n_heads * chunks;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % chunks);
    long long r = i / chunks;
    const int h = (int)(r % n_heads);
    const int t = (int)(r / n_heads);
    bf16* p = x + (long long)t * ld + (long long)h * hd + c * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + half);
    const float4* cp = reinterpret_cast<const float4*>(cs + (long long)t * half + c * 8);
    const float4* sp = reinterpret_cast<const float4*>(cs + (long long)T * half + (long long)t * half + c * 8);
    const float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
    const float co[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w}, si[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const uint32_t au[4] = {a.x, a.y, a.z, a.w}, bu[4] = {b.x, b.y, b.z, b.w};
    uint32_t oa[4], ob[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x1l = bf16_lo(au[k]), x1h = bf16_hi(au[k]), x2l = bf16_lo(bu[k]), x2h = bf16_hi(bu[k]);
      oa[k] = pack_bf16(x1l * co[2 * k] - x2l * si[2 * k], x1h * co[2 * k + 1] - x2h * si[2 * k + 1]);
      ob[k] = pack_bf16(x2l * co[2 * k] + x1l * si[2 * k], x2h * co[2 * k + 1] + x1h * si[2 * k + 1]);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(p + half) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
  }
}

// decode step: the same rotation over the q and k heads of row b, with the rotated K head and the V row appended to
// the cache at index cache_len[b] in the same pass (one launch instead of rope + append)
__global__ void __launch_bounds__(256) rope_kv_append_kernel(bf16* __restrict__ x, long long ld, const float* __restrict__ cs, int T,
                                                             int q_heads, int kv_heads, int hd, const int* __restrict__ cache_len,
                                                             bf16* __restrict__ kc, bf16* __restrict__ vc, int cap) {
  griddep_launch();
  griddep_wait();
  const int half = hd / 2, chunks = half / 8, n_heads = q_heads + kv_heads, kv_dim = kv_heads * hd;
  const long long n_rot = (long long)T * n_heads * chunks, n_v = (long long)T * (kv_dim / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_rot + n_v; i += (long long)gridDim.x * blockDim.x) {
    if (i >= n_rot) {   // V row copy, 16 bytes per thread
      const long long j = i - n_rot;
      const int t = (int)(j / (kv_dim / 8)), c = (int)(j % (kv_dim / 8));
      const bf16* src = x + (long long)t * ld + (long long)n_heads * hd + c * 8;
      *reinterpret_cast<uint4*>(vc + ((long long)t * cap + cache_len[t]) * kv_dim + c * 8) = *reinterpret_cast<const uint4*>(src);
      continue;
    }
    const int c = (int)(i % chunks);
    long long r = i / chunks;
    const int h = (int)(r % n_heads);
    const int t = (int)(r / n_heads);
    bf16* p = x + (long long)t * ld + (long long)h * hd + c * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(p + half);
    const float4* cp = reinterpret_cast<const float4*>(cs + (long long)t * half + c * 8);
    const float4* sp = reinterpret_cast<const float4*>(cs + (long long)T * half + (long long)t * half + c * 8);
    const float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
    const float co[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w}, si[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const uint32_t au[4] = {a.x, a.y, a.z, a.w}, bu[4] = {b.x, b.y, b.z, b.w};
    uint32_t oa[4], ob[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x1l = bf16_lo(au[k]), x1h = bf16_hi(au[k]), x2l = bf16_lo(bu[k]), x2h = bf16_hi(bu[k]);
      oa[k] = pack_bf16(x1l * co[2 * k] - x2l * si[2 * k], x1h * co[2 * k + 1] - x2h * si[2 * k + 1]);
      ob[k] = pack_bf16(x2l * co[2 * k] + x1l * si[2 * k], x2h * co[2 * k + 1] + x1h * si[2 * k + 1]);
    }
    const uint4 va = make_uint4(oa[0], oa[1], oa[2], oa[3]), vb = make_uint4(ob[0], ob[1], ob[2], ob[3]);
    if (h < q_heads) {
      *reinterpret_cast<uint4*>(p) = va;
      *reinterpret_cast<uint4*>(p + half) = vb;
    } else {   // K heads are only consumed from the cache
      bf16* kp = kc + ((long long)t * cap + cache_len[t]) * kv_dim + (long long)(h - q_heads) * hd + c * 8;
      *reinterpret_cast<uint4*>(kp) = va;
      *reinterpret_cast<uint4*>(kp + half) = vb;
    }
  }
}

int rope_kv_append(bf16* qkv, long long ld, const float* cos_sin, int T, int q_heads, int kv_heads, int head_dim, const int* cache_len,
                   bf16* kc, bf16* vc, int cap, cudaStream_t s) {
  FO1_CHECK_ARG(head_dim % 16 == 0 && ld % 8 == 0, "rope_kv_append: head_dim %d must be a multiple of 16 and the pitch of 8", head_dim);
  if (T == 0) return FO1_OK;
  const long long n = (long long)T * (q_heads + kv_heads) * (head_dim / 16) + (long long)T * kv_heads * head_dim / 8;
  const int blocks = (int)((n + 255) / 256 < device_sm_count() * 16 ? (n + 255) / 256 : device_sm_count() * 16);
  launch_k(rope_kv_append_kernel, dim3(blocks), dim3(256), 0, s, qkv, ld, cos_sin, T, q_heads, kv_heads, head_dim, cache_len, kc, vc, cap);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int vit_rope_table(const int* pos_hw, float* cos_sin, int T, int head_dim, float theta, cudaStream_t s) {
  FO1_CHECK_ARG(head_dim % 4 == 0, "vit_rope_table: head_dim %d must be a multiple of 4", head_dim);
  if (T == 0) return FO1_OK;
  const int half = head_dim / 2;
  vit_rope_table_kernel<<<ceil_div(T * half, 256), 256, 0, s>>>(pos_hw, cos_sin, T, half, theta);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int rope_apply(bf16* x, long long ld, const float* cos_sin, int T, int n_heads, int head_dim, cudaStream_t s) {
  FO1_CHECK_ARG(head_dim % 16 == 0 && ld % 8 == 0, "rope_apply: head_dim %d must be a multiple of 16 and the pitch of 8", head_dim);
  if (T == 0) return FO1_OK;
  const long long n = (long long)T * n_heads * (head_dim / 16);
  const int blocks = (int)((n + 255) / 256 < device_sm_count() * 16 ? (n + 255) / 256 : device_sm_count() * 16);
  rope_apply_kernel<<<blocks, 256, 0, s>>>(x, ld, cos_sin, T, n_heads, head_dim);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int vit_rope_apply(bf16* qkv, const float* cos_sin, int T, int heads, int head_dim, cudaStream_t s) {
  return rope_apply(qkv, 3LL * heads * head_dim, cos_sin, T, 2 * heads, head_dim, s);   // q heads then k heads are contiguous
}

// M-RoPE: inv_freq[j] = theta^(-2j/hd), j < hd/2; frequency j takes its position from axis t / h / w according to
// the sections [sec_t, sec_h, sec_w] (sum = hd/2); cos/sin duplicated over the two halves
// (apply_multimodal_rotary_pos_emb, modeling_qwen2_5_vl.py:675-685).  The table is built once per forward and
// shared by all layers.
__global__ void mrope_table_kernel(const int* __restrict__ pos3, float* __restrict__ cs, int T, int half, int hd, int sec_t, int sec_h,
                                   float theta) {
  griddep_launch();
  griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * half) return;
  const int t = i / half, j = i - t * half;
  const int axis = j < sec_t ? 0 : (j < sec_t + sec_h ? 1 : 2);
  const float inv = 1.0f / powf(theta, (float)(2 * j) / (float)hd);
  const float ang = (float)pos3[(long long)axis * T + t] * inv;
  cs[i] = cosf(ang);
  cs[(long long)T * half + i] = sinf(ang);
}

int mrope_table(const int* pos3, float* cos_sin, int T, int head_dim, int sec_t, int sec_h, int sec_w, float theta, cudaStream_t s) {
  FO1_CHECK_ARG(sec_t + sec_h + sec_w == head_dim / 2, "mrope_table: sections %d+%d+%d != head_dim/2", sec_t, sec_h, sec_w);
  if (T == 0) return FO1_OK;
  const int half = head_dim / 2;
  launch_k(mrope_table_kernel, dim3(ceil_div(T * half, 256)), dim3(256), 0, s, pos3, cos_sin, T, half, head_dim, sec_t, sec_h, theta);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

}  // namespace fo1
