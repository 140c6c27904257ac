// llm.cu -- Qwen2.5 decoder on sm_90a: embedding splice, M-RoPE bookkeeping, varlen prefill, device-resident
// greedy decode with a static K/V cache.
//
// Reference: OmChatQwen25VLForCausalLM.forward + prepare_inputs_labels_for_qwen2_5_vl_multimodal
// (omchat_qwen2_5_vl.py:135-532), Qwen2_5_VLModel / DecoderLayer / Attention / MLP / RMSNorm
// (modeling_qwen2_5_vl.py:1126-1242, 1014-1095, 738-802, 627-640, 126-140), get_rope_index (:1546-1721),
// the decode position rule (:1848-1860) and HF's greedy loop with KeywordsStoppingCriteria (mm_utils.py:137-181).
// Differences from the reference: all sequences of the batch run packed (varlen), no padding tokens exist; K/V live
// in one static [layer][seq][cap][kv] cache written by the prefill and appended in place by each decode
// step (the reference torch.cat's a DynamicCache per layer per step); argmax, stop-token test and all loop
// state stay on the device, the host only enqueues kernels (no per-token sync); lm_head runs on the last
// prompt position only.
#include <algorithm>
#include <cmath>
#include <type_traits>

#include "beam.cuh"
#include "decode_loop.cuh"
#include "decode_mega.cuh"
#include "lookup.cuh"

namespace fo1 {

// ------------------------------------------------------------------------------------------ kernels
// inputs_embeds rows from three sources
__global__ void __launch_bounds__(256) build_embeds_kernel(const int* __restrict__ kind, const int* __restrict__ index,
                                                           const bf16* __restrict__ table, const bf16* __restrict__ img,
                                                           const bf16* __restrict__ reg, bf16* __restrict__ out, int H) {
  const int r = blockIdx.x;
  const int k = kind[r];
  const bf16* src = (k == 0 ? table : (k == 1 ? img : reg)) + (long long)index[r] * H;
  bf16* dst = out + (long long)r * H;
  for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) *reinterpret_cast<uint4*>(dst + c) = *reinterpret_cast<const uint4*>(src + c);
}

// x[b] = table[tok[b]]
__global__ void __launch_bounds__(256) embed_tokens_kernel(const int* __restrict__ tok, const bf16* __restrict__ table,
                                                           bf16* __restrict__ out, int H) {
  griddep_launch();
  griddep_wait();
  const bf16* src = table + (long long)tok[blockIdx.x] * H;
  bf16* dst = out + (long long)blockIdx.x * H;
  for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) *reinterpret_cast<uint4*>(dst + c) = *reinterpret_cast<const uint4*>(src + c);
}

// prefill: copy the rotated K and V of packed row r (position row_gt[r].y of group row_gt[r].x) into the cache slot of every member of
// the group (members[grp_off[g] .. grp_off[g + 1])).  prefill_plan() builds the groups of each kind of call.
__global__ void __launch_bounds__(64) kv_fanout_kernel(const bf16* __restrict__ qkv, long long ld, int q_dim, int kv_dim,
                                                       const int2* __restrict__ row_gt, const int* __restrict__ grp_off,
                                                       const int* __restrict__ members, bf16* __restrict__ kc, bf16* __restrict__ vc, int cap) {
  const int r = blockIdx.x;
  const int2 gt = row_gt[r];
  const int m0 = grp_off[gt.x], m1 = grp_off[gt.x + 1];
  const bf16* kp = qkv + (long long)r * ld + q_dim;            // K | V are contiguous in the packed row
  for (int c = threadIdx.x * 8; c < 2 * kv_dim; c += blockDim.x * 8) {
    const uint4 val = *reinterpret_cast<const uint4*>(kp + c);
    bf16* dst = c < kv_dim ? kc + c : vc + (c - kv_dim);
    for (int i = m0; i < m1; ++i) *reinterpret_cast<uint4*>(dst + ((long long)members[i] * cap + gt.y) * kv_dim) = val;
  }
}
// shared-prefix prefill: zero the V rows [L_b, L_b rounded up to 64) of every sequence in every layer.  The last 64-key tile of the
// cache-reading attention reads them with weight zero, which a non-finite leftover would turn into NaN; decode overwrites them.
__global__ void __launch_bounds__(128) kv_zero_tail_kernel(bf16* __restrict__ vc, long long layer_stride, const int* __restrict__ seq_lens,
                                                           int cap, int kv_dim) {
  const int b = blockIdx.x;
  const int t0 = seq_lens[b], t1 = min(cap, (t0 + 63) & ~63);
  bf16* base = vc + blockIdx.y * layer_stride + (long long)b * cap * kv_dim;
  for (long long c = (long long)t0 * kv_dim + threadIdx.x * 8; c < (long long)t1 * kv_dim; c += blockDim.x * 8)
    *reinterpret_cast<uint4*>(base + c) = make_uint4(0u, 0u, 0u, 0u);
}
// Single-query GQA attention over the cache, split over the sequence (flash-decoding) and run on the tensor pipe:
// one block per (sequence, kv head, split).  The G <= 8 query heads of the kv head are the rows of an m16n8k16 tile
// (rows G..15 are zero), so K and V are read ONCE per kv head instead of once per query head.  Every warp owns
// 16-key tiles of the split and streams them through a private cp.async ring (3 tiles = 24 KB, two in flight behind
// the one being reduced; 16-byte chunks XOR-swizzled by key) -- the load -> use chain of a register-fed version left
// a warp with one tile in flight.  S = Q.K^T takes its B fragments with ldmatrix, P.V with
// ldmatrix.trans; the block merges its warps' (m, l, acc) and writes one un-normalised partial per (head, split);
// decode_attn_combine_kernel merges the splits.
constexpr int kDecSplits = 8;   // most key splits per (sequence, kv head); the launch uses gridDim.z <= kDecSplits of them
constexpr int kDecWarps = 4;
constexpr int kDecStages = 3;
constexpr int kDecTileBytes = 16 * 256 * 2;                      // 16 keys x (K row 256 B + V row 256 B)
constexpr int kDecRingBytes = kDecWarps * kDecStages * kDecTileBytes;
constexpr int kDecSmemBytes = kDecRingBytes;                     // the warp merge staging aliases the ring
__device__ __forceinline__ void mma_m16n8k16(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
  // rows 8..15 of A (a1, a3) are zero: only the G query heads in rows 0..7 carry data
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%5}, {%7,%8}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(0u), "r"(a2), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack2_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ void dec_cp16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 -> 16 bytes of zeros
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void dec_ldsm(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void dec_ldsm_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// Query row b reads cache slot b, or (MAPPED: the prompt-lookup verify step) slot row_slot[b], up to its own index idx[b].  The verify
// launch takes the plain step's split count, so a row's bits are those of the plain step at its position.
template <bool MAPPED>
__global__ void __launch_bounds__(kDecWarps * 32) decode_attn_kernel(const bf16* __restrict__ q, long long ldq, const bf16* __restrict__ kc,
                                                                     const bf16* __restrict__ vc, const int* __restrict__ row_slot,
                                                                     const int* __restrict__ idx, int cap, int kv_heads, int G,
                                                                     float* __restrict__ part, float scale) {
  constexpr int HD = 128;
  extern __shared__ __align__(128) uint8_t dec_smem[];
  const int b = blockIdx.x, kvh = blockIdx.y, sp = blockIdx.z;
  griddep_launch();
  griddep_wait();
  const int slot = MAPPED ? row_slot[b] : b;
  const int n = idx[b] + 1;        // the row's own K/V was appended at index idx[b]
  const int n_splits = gridDim.z;
  const int chunk = ((n + n_splits - 1) / n_splits + 15) & ~15;
  const int t_begin = sp * chunk, t_end = min(n, t_begin + chunk);
  const int kv_dim = kv_heads * HD;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  // Q fragments (A operand, rows = heads): a0 = dims (16 ks + 2t, +1), a2 = dims (16 ks + 8 + 2t, +1) of head g
  uint32_t qa[8][2];
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) { qa[ks][0] = 0u; qa[ks][1] = 0u; }
  if (g < G) {
    const bf16* qp = q + (long long)b * ldq + (long long)(kvh * G + g) * HD + 2 * t;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qa[ks][0] = *reinterpret_cast<const uint32_t*>(qp + ks * 16);
      qa[ks][1] = *reinterpret_cast<const uint32_t*>(qp + ks * 16 + 8);
    }
  }
  const float sc = scale * 1.4426950408889634f;
  float m = -INFINITY, l = 0.f, o[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }

  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(dec_smem) + w * kDecStages * kDecTileBytes;
  // copy plan: instruction i moves chunk (key = 2i + lane/16, 16-byte chunk lane%16) of the K half and of the V half
  const int cp_key = lane >> 4, cp_chunk = lane & 15;
  const bf16* kbase = kc + (long long)slot * cap * kv_dim + kvh * HD + cp_chunk * 8;
  const bf16* vbase = vc + (long long)slot * cap * kv_dim + kvh * HD + cp_chunk * 8;
  int t_issue = t_begin + w * 16;
  uint32_t st_issue = 0, st_done = 0;
  auto issue_tile = [&]() {
    if (t_issue < t_end) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = 2 * i + cp_key, tok = t_issue + key;
        const bool ok = tok < t_end;                          // keys beyond the split: zero rows (their scores are masked)
        const long long off = (long long)(ok ? tok : t_begin) * kv_dim;
        const uint32_t dst = ring + st_issue + key * 256 + ((cp_chunk ^ (key & 7)) << 4);
        dec_cp16(dst, kbase + off, ok);
        dec_cp16(dst + 16 * 256, vbase + off, ok);
      }
      t_issue += kDecWarps * 16;
      st_issue = (st_issue == (kDecStages - 1) * kDecTileBytes) ? 0u : st_issue + kDecTileBytes;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  issue_tile();
  issue_tile();
  // ldmatrix lane roles: S: matrix m = lane/8 -> (keys (m/2)*8 + r, chunk 2 ks + (m&1)); PV (trans): (keys (m&1)*8 + r, chunk c + m/2)
  const int lr = lane & 7, lm = lane >> 3;
  for (int t0 = t_begin + w * 16; t0 < t_end; t0 += kDecWarps * 16) {
    issue_tile();
    asm volatile("cp.async.wait_group 2;" ::: "memory");
    __syncwarp();
    const uint32_t kt = ring + st_done, vt = kt + 16 * 256;
    float s[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      uint32_t bk[4];
      const int key = (lm >> 1) * 8 + lr;
      dec_ldsm(bk, kt + key * 256 + (((2 * ks + (lm & 1)) ^ (key & 7)) << 4));
      mma_m16n8k16(s[0], qa[ks][0], qa[ks][1], bk[0], bk[1]);
      mma_m16n8k16(s[1], qa[ks][0], qa[ks][1], bk[2], bk[3]);
    }
    float tmax = -INFINITY;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s[i][e] = (t0 + i * 8 + 2 * t + e < t_end) ? s[i][e] * sc : -INFINITY;
        tmax = fmaxf(tmax, s[i][e]);
      }
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
    const float mn = fmaxf(m, tmax);            // key t0 is always valid: mn is finite
    const float alpha = exp2f(m - mn);          // m = -inf on the first tile -> 0
    const float p00 = exp2f(s[0][0] - mn), p01 = exp2f(s[0][1] - mn), p10 = exp2f(s[1][0] - mn), p11 = exp2f(s[1][1] - mn);
    l = l * alpha + (p00 + p01) + (p10 + p11);
    m = mn;
    const uint32_t pa0 = pack2_bf16(p00, p01), pa2 = pack2_bf16(p10, p11);
#pragma unroll
    for (int c = 0; c < 16; c += 2) {
      uint32_t bv[4];
      const int key = (lm & 1) * 8 + lr;
      dec_ldsm_t(bv, vt + key * 256 + (((c + (lm >> 1)) ^ (key & 7)) << 4));
      o[c][0] *= alpha; o[c][1] *= alpha; o[c + 1][0] *= alpha; o[c + 1][1] *= alpha;
      mma_m16n8k16(o[c], pa0, pa2, bv[0], bv[1]);
      mma_m16n8k16(o[c + 1], pa0, pa2, bv[2], bv[3]);
    }
    __syncwarp();                               // the stage may be refilled by the next issue_tile()
    st_done = (st_done == (kDecStages - 1) * kDecTileBytes) ? 0u : st_done + kDecTileBytes;
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  l += __shfl_xor_sync(0xffffffffu, l, 1);
  l += __shfl_xor_sync(0xffffffffu, l, 2);
  __syncthreads();                              // every warp is done with its ring: reuse it for the merge
  float* sm_o = reinterpret_cast<float*>(dec_smem);                    // [kDecWarps][8][HD]
  float* sm_m = sm_o + kDecWarps * 8 * HD;                             // [kDecWarps][8]
  float* sm_l = sm_m + kDecWarps * 8;
  if (t == 0) { sm_m[w * 8 + g] = m; sm_l[w * 8 + g] = l; }
#pragma unroll
  for (int j = 0; j < 16; ++j)
    *reinterpret_cast<float2*>(&sm_o[(w * 8 + g) * HD + j * 8 + 2 * t]) = make_float2(o[j][0], o[j][1]);
  __syncthreads();
  const int d = threadIdx.x;   // kDecWarps * 32 == HD
  for (int r = 0; r < G; ++r) {
    float mm = -INFINITY;
#pragma unroll
    for (int ww = 0; ww < kDecWarps; ++ww) mm = fmaxf(mm, sm_m[ww * 8 + r]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int ww = 0; ww < kDecWarps; ++ww) {
      const float f = (sm_m[ww * 8 + r] == -INFINITY) ? 0.f : exp2f(sm_m[ww * 8 + r] - mm);
      num += sm_o[(ww * 8 + r) * HD + d] * f;
      den += sm_l[ww * 8 + r] * f;
    }
    // partial record per (b, head, split): [m, l, pad, pad, acc[128]]
    float* rec = part + (((long long)b * kv_heads * G + kvh * G + r) * kDecSplits + sp) * (HD + 4);
    if (d == 0) { rec[0] = mm; rec[1] = den; }
    rec[4 + d] = num;
  }
}

// merge the kDecSplits partials of one (sequence, q head): out = sum_s acc_s * 2^(m_s - m) / sum_s l_s * 2^(m_s - m)
__global__ void __launch_bounds__(128) decode_attn_combine_kernel(const float* __restrict__ part, bf16* __restrict__ out, long long ldo,
                                                                  int q_heads, int n_splits) {
  constexpr int HD = 128;
  const int b = blockIdx.x, h = blockIdx.y, d = threadIdx.x;
  griddep_launch();
  griddep_wait();
  const float* rec = part + (((long long)b * q_heads + h) * kDecSplits) * (HD + 4);
  float mm = -INFINITY;
#pragma unroll
  for (int s = 0; s < n_splits; ++s) mm = fmaxf(mm, rec[s * (HD + 4)]);
  float num = 0.f, den = 0.f;
#pragma unroll
  for (int s = 0; s < n_splits; ++s) {
    const float ms = rec[s * (HD + 4)];
    const float sc = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
    num += rec[s * (HD + 4) + 4 + d] * sc;
    den += rec[s * (HD + 4) + 1] * sc;
  }
  out[(long long)b * ldo + (long long)h * HD + d] = __float2bfloat16_rn(num / den);
}

// host side of the decode attention: split count = one wave of blocks (2 per SM: 96 KB of shared memory each) over n_seqs sequences.
// Row r reads its cache slot up to index idx[r]; row_slot (the prompt-lookup verify step) maps the rows to n_seqs slots, and the split
// count stays the plain step's, so each row's key chunks are those the plain step at its position would use.
static int decode_attention(const bf16* q, long long ldq, const bf16* kc, const bf16* vc, const int* idx, const int* row_slot, int rows,
                            int n_seqs, int cap, int q_heads, int kv_heads, int hd, float scale, bf16* out, long long ldo, float* part,
                            cudaStream_t s) {
  const int G = kv_heads > 0 ? q_heads / kv_heads : 0;
  if (kv_heads <= 0 || q_heads % kv_heads != 0 || G > 8 || hd != 128) {
    set_error("decode attention: %d/%d heads, head_dim %d unsupported (GQA group <= 8, head_dim 128)", q_heads, kv_heads, hd);
    return FO1_ERR_UNSUPPORTED;
  }
  if (rows == 0) return FO1_OK;
  static bool attr_set = false;
  if (!attr_set) {
    FO1_CUDA(cudaFuncSetAttribute(decode_attn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemBytes));
    FO1_CUDA(cudaFuncSetAttribute(decode_attn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemBytes));
    attr_set = true;
  }
  const int slots = 2 * device_sm_count();
  const int n_splits = std::max(1, std::min(kDecSplits, slots / std::max(1, n_seqs * kv_heads)));
  {
    ProfScope prof(row_slot != nullptr ? "decode_attn_rows" : "decode_attn", 0.0, 0.0, s);
    launch_k(row_slot != nullptr ? decode_attn_kernel<true> : decode_attn_kernel<false>, dim3(rows, kv_heads, n_splits), dim3(kDecWarps * 32),
             kDecSmemBytes, s, q, ldq, kc, vc, row_slot, idx, cap, kv_heads, G, part, scale);
    FO1_LAUNCH_CHECK();
  }
  launch_k(decode_attn_combine_kernel, dim3(rows, q_heads), dim3(128), 0, s, (const float*)part, out, ldo, q_heads, n_splits);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

// greedy token: lowest index among the maxima of a fp32 logits row
__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ logits, int V, int* __restrict__ out) {
  griddep_launch();
  griddep_wait();
  const float* row = logits + (long long)blockIdx.x * V;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float v = row[i];
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
  }
  __shared__ float sv[32];
  __shared__ int si[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x]; bi = si[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) out[blockIdx.x] = bi;
  }
}

// after the prefill: lengths, positions, first token
__global__ void decode_init_kernel(DecodeState st, const int* __restrict__ seq_lens, const int* __restrict__ deltas, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) { *st.step = 0; *st.n_active = B; }
  if (b >= B) return;
  st.cache_len[b] = seq_lens[b];
  const int p = seq_lens[b] + deltas[b];
  st.pos3[b] = p; st.pos3[B + b] = p; st.pos3[2 * B + b] = p;
  st.finished[b] = 0;
}
// record the column of new_tok (decode_loop.cuh).  ONE block; the output column is the device-resident step counter, so the launch is
// identical every iteration (CUDA-graph replayable).
template <bool STREAM>
__global__ void __launch_bounds__(1024) decode_update_kernel(ColumnSink k, int B, int advance_cache) {
  griddep_launch();
  griddep_wait();
  const int step = *k.st.step;
  bool publish = false, cancel = false;
  column_prologue<STREAM>(k, step, publish, cancel);
  for (int b = threadIdx.x; b < B; b += blockDim.x) record_token<STREAM>(k, B, b, step, k.st.new_tok[b], advance_cache, publish, cancel);
  column_epilogue<STREAM>(k, step, publish, cancel);
}
__global__ void fill_int_kernel(int* p, int v, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}
// slot pool: after the prefill of n admitted sequences, decode_init_kernel for the listed slots (B = the pool's slot count): lengths,
// positions, column 0, limit and sampling parameters (prm: the admitted rows', copied to pool_prm), output rows refilled with pad, then
// column 0 (tok[i], drawn from the prefill's last row) recorded as a decode step records one
__global__ void __launch_bounds__(256) slots_admit_kernel(ColumnSink k, int B, int n, const int* __restrict__ slots,
                                                          const int* __restrict__ max_new, const int* __restrict__ seq_lens,
                                                          const int* __restrict__ deltas, const int* __restrict__ tok,
                                                          const SampleRowParams* __restrict__ prm, SampleRowParams* __restrict__ pool_prm) {
  const DecodeState& st = k.st;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int b = slots[i];
    st.cache_len[b] = seq_lens[i];
    const int p = seq_lens[i] + deltas[i];
    st.pos3[b] = p; st.pos3[B + b] = p; st.pos3[2 * B + b] = p;
    st.finished[b] = 0;
    k.col[b] = 0;
    k.max_new_row[b] = max_new[i];
    if (prm != nullptr) pool_prm[b] = prm[i];
  }
  for (long long j = threadIdx.x; j < (long long)n * k.max_new; j += blockDim.x)
    k.out_tokens[(long long)slots[j / k.max_new] * k.max_new + j % k.max_new] = k.pad_id;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    atomicAdd(st.n_active, 1);
    record_token<false>(k, B, slots[i], 0, tok[i], false, false, false);
  }
}

// ------------------------------------------------------------------------------------------ host
struct LlmState {
  int* ints = nullptr;   // one allocation for the DecodeState arrays
  int cap_b = 0, cap_stop = 0;
  int* h_flag = nullptr; // pinned
};

static int llm_resolve(Model* m) {
  const fo1_model_config& c = m->cfg;
  WeightGetter g{m, ""};
  LlmW& w = m->llm;
  const int64_t H = c.llm_hidden, V = c.llm_vocab, QD = (int64_t)c.llm_heads * c.llm_head_dim, KD = (int64_t)c.llm_kv_heads * c.llm_head_dim;
  const int64_t Ip = (c.llm_inter + 31) / 32 * 32;
  w.embed = g.bf("llm.embed", {V, H});
  w.norm = g.bf("llm.norm.w", {H});
  w.lm_head = g.bf("llm.lm_head", {V, H});
  w.layer.resize(c.llm_layers);
  for (int i = 0; i < c.llm_layers; ++i) {
    const std::string p = "llm.l" + std::to_string(i) + ".";
    LlmLayerW& L = w.layer[i];
    L.ln1 = g.bf(p + "ln1.w", {H});
    L.qkv_w = g.bf(p + "qkv.w", {QD + 2 * KD, H});
    L.qkv_b = g.bf(p + "qkv.b", {QD + 2 * KD});
    L.o_w = g.bf(p + "o.w", {H, QD});
    L.ln2 = g.bf(p + "ln2.w", {H});
    L.gateup_w = g.bf(p + "gateup.w", {2 * Ip, H});
    L.down_w = g.bf(p + "down.w", {H, Ip});
  }
  if (!g.err.empty()) { set_error("LLM weights: %s", g.err.c_str()); return FO1_ERR_NOT_FOUND; }
  w.ok = true;
  // optional decode copies (weights.py::prepare_llm): W diag(g) for the two normed projections and the LM head, gate / up in the
  // decode kernel's 8 + 8 row interleave.  All present and a model shape the kernel supports -> the persistent decode kernel is used.
  w.mega_ok = m->find("llm.head_dec") != nullptr &&
              decode_mega_supports(c.llm_hidden, c.llm_head_dim, c.llm_heads, c.llm_kv_heads, c.llm_inter, c.llm_vocab);
  for (int i = 0; i < c.llm_layers && w.mega_ok; ++i) {
    const std::string p = "llm.l" + std::to_string(i) + ".";
    w.mega_ok = m->find(p + "qkv_dec.w") != nullptr && m->find(p + "gu_dec.w") != nullptr;
  }
  if (w.mega_ok) {
    WeightGetter g2{m, ""};
    w.head_dec = g2.bf("llm.head_dec", {V, H});
    std::vector<MegaLayer> ml(c.llm_layers);
    for (int i = 0; i < c.llm_layers; ++i) {
      const std::string p = "llm.l" + std::to_string(i) + ".";
      LlmLayerW& L = w.layer[i];
      L.qkv_dec = g2.bf(p + "qkv_dec.w", {QD + 2 * KD, H});
      L.gu_dec = g2.bf(p + "gu_dec.w", {2 * (int64_t)c.llm_inter, H});
      ml[i].qkv_w = L.qkv_dec; ml[i].qkv_b = L.qkv_b; ml[i].o_w = L.o_w; ml[i].gu_w = L.gu_dec; ml[i].down_w = L.down_w;
    }
    if (!g2.err.empty()) { set_error("LLM decode weights: %s", g2.err.c_str()); return FO1_ERR_NOT_FOUND; }
    // the kernel reads down_w with K = intermediate size: a supported intermediate (a multiple of 64) is already its own padding
    if (w.mega_layers) cudaFree(w.mega_layers);
    FO1_CUDA(cudaMalloc(&w.mega_layers, ml.size() * sizeof(MegaLayer)));
    FO1_CUDA(cudaMemcpy(w.mega_layers, ml.data(), ml.size() * sizeof(MegaLayer), cudaMemcpyHostToDevice));
  }
  return FO1_OK;
}
int llm_finalize(Model* m) { return m->cfg.llm_layers > 0 ? llm_resolve(m) : FO1_OK; }

static void slots_free(Model* m);
void llm_destroy_state(Model* m) {
  slots_free(m);
  if (m->llm.mega_layers) { cudaFree(m->llm.mega_layers); m->llm.mega_layers = nullptr; }
  LlmState* s = static_cast<LlmState*>(m->llm_state);
  if (!s) return;
  if (s->ints) cudaFree(s->ints);
  if (s->h_flag) cudaFreeHost(s->h_flag);
  delete s;
  m->llm_state = nullptr;
}

static int ensure_kv(Model* m, int B, int cap) {
  const fo1_model_config& c = m->cfg;
  const size_t per = (size_t)c.llm_layers * B * cap * c.llm_kv_heads * c.llm_head_dim * sizeof(bf16);
  if (2 * per > m->kv_bytes) {
    FO1_CUDA(cudaDeviceSynchronize());
    if (m->kv_cache) FO1_CUDA(cudaFree(m->kv_cache));
    m->kv_cache = nullptr; m->kv_bytes = 0;
    FO1_CUDA(cudaMalloc(&m->kv_cache, 2 * per));
    m->kv_bytes = 2 * per;
  }
  m->kv_batch = B; m->kv_cap = cap;
  return FO1_OK;
}

static int ensure_state(Model* m, int B, int n_stop, DecodeState* st) {
  LlmState* s = static_cast<LlmState*>(m->llm_state);
  if (!s) { s = new LlmState(); m->llm_state = s; }
  if (B > s->cap_b || n_stop > s->cap_stop) {
    FO1_CUDA(cudaDeviceSynchronize());
    if (s->ints) FO1_CUDA(cudaFree(s->ints));
    s->cap_b = std::max(B, s->cap_b); s->cap_stop = std::max(n_stop, std::max(s->cap_stop, 8));
    FO1_CUDA(cudaMalloc(reinterpret_cast<void**>(&s->ints), ((size_t)9 * s->cap_b + s->cap_stop + 64) * sizeof(int)));
  }
  if (!s->h_flag) FO1_CUDA(cudaMallocHost(reinterpret_cast<void**>(&s->h_flag), 64));
  int* p = s->ints;
  const int cb = s->cap_b;
  st->cache_len = p; p += cb;
  st->pos3 = p; p += 3 * cb;
  st->cur_tok = p; p += cb;
  st->new_tok = p; p += cb;
  st->finished = p; p += cb;
  st->n_active = p; p += 16;
  st->step = p; p += 16;
  st->stop_ids = p;
  return FO1_OK;
}

// norm kernel of the launches with one row per sequence (decode steps, the prefill's last rows): the block-per-row kernel at any batch
// size; the width alone decides for models wider than it serves
static NormKernel seq_norm_kernel(int H) { return H <= kNormBlockMaxCols ? NORM_BLOCK : NORM_WARP; }

// an open slot pool (fo1_slots_open): its loop state, column sink and per-slot sampling parameters live across calls
struct SlotPool {
  int n_slots, interval;
  DecodeMode mode;                  // DEC_SAMPLED when any slot may sample, else DEC_GREEDY
  ColumnSink k;                     // k.col / k.max_new_row: [n_slots] each, in `ints`
  int* ints = nullptr;              // col, max_new_row, then the admission's slots / max_new / 0 (n_slots each, + 1)
  SampleRowParams* prm = nullptr;   // [n_slots]
  std::vector<int> busy;            // host: admitted and not seen finished by the last fo1_slots_decode
  // logits processors: the distinct sets the running requests use (host; an admission that brings a new set drops the ones no
  // running slot uses, so they number at most n_slots + the admitted requests), their device table, and per slot its set, prompt
  // length and prompt ids (proc.set_of / plen / prompt: `proc_ints`, [n_slots] + [n_slots] + [n_slots][cap]; slot_set mirrors
  // set_of).  proc.tab stays nullptr until an admission brings a set; from then on a greedy pool decodes through the sampler with
  // top_k 1 (bit-identical)
  ProcArgs proc{};
  int* proc_ints = nullptr;
  std::vector<ProcSet> proc_sets;
  std::map<std::vector<int>, int> proc_index;
  std::vector<int> slot_set;
  size_t proc_tab_cap = 0, proc_bias_cap = 0;
};

// the decode mode of a pool: a greedy pool with logits processors draws with top_k 1 from its stored logits rows
static DecodeMode pool_mode(const SlotPool& p) { return p.mode == DEC_GREEDY && p.proc.tab != nullptr ? DEC_SAMPLED : p.mode; }

// one generate call, described once by llm_generate: the caller's descriptors (the options as generate_check normalised them), the
// decode mode, the column sink, and the device state of beam search (with its host table of length-penalty divisors) or of prompt
// lookup; or one admission into / decode segment of a slot pool (`pool`; an admission's host slot list `slots`)
struct GenerateCall {
  fo1_generate_desc* d;
  const fo1_prefix_desc* px;        // shared prefix (null: none)
  const fo1_sampling_desc* sp;
  const fo1_score_desc* sc;
  const fo1_stream_desc* stm;
  DecodeMode mode;
  ColumnSink k;
  const fo1_beam_desc* bmd;         // beam search (null: none): `beam`, `lp_div`
  BeamArgs beam;
  std::vector<float> lp_div;
  const fo1_lookup_desc* lkd;       // prompt lookup (null: none): `lookup`
  LookupArgs lookup;
  SlotPool* pool;
  const int* slots;
  int exit_at;                      // the decode loop ends once at most this many sequences run (0: all stopped)
  const fo1_processor_desc* pr;     // logits processors (null: none): `proc` on the device, uploaded from proc_ints / proc_bias
  ProcArgs proc;
  std::vector<int> proc_ints;       // the table, then set_of [B], plen [B], prompts [B][proc.ld]
  std::vector<float> proc_bias;
  size_t proc_tab_n;
};

// the scratch buffers of a decoder layer over packed rows
struct LayerBuf { bf16 *xn, *qkv, *att, *x_mid, *h; float* dec_part; int* rowseg; };

// the attention of a prefill layer: the rotated K/V of every packed row into the cache through the write map (kv_fanout_kernel), the
// causal attention over the packed segments, and with a shared prefix the own rows (the rows after the segments) against the cache
// (own.k / own.v are the layer's cache, set per layer)
struct PrefillAttn {
  const int2* row_gt;
  const int *grp_off, *members;
  AttnArgs causal, own;             // own.total_rows == 0: no shared prefix
};
// the attention of a decode step: row r appends its K/V at index idx[r] of cache slot r, or of slot row_slot[r], and attends the slot up
// to there; n_seqs sequences set the key split
struct DecodeAttn {
  const int* idx;
  const int* row_slot;
  int n_seqs;
};

static int layer_attention(Model* m, const PrefillAttn& p, const LayerBuf& b, int rows, const float* cs, bf16* kc, bf16* vc, cudaStream_t s,
                           bool dry) {
  const fo1_model_config& c = m->cfg;
  const int hd = c.llm_head_dim, QD = c.llm_heads * hd, KD = c.llm_kv_heads * hd, ldq = QD + 2 * KD;
  FO1_RUN(rope_apply(b.qkv, ldq, cs, rows, c.llm_heads + c.llm_kv_heads, hd, s));   // q|k heads are contiguous in the packed row
  if (!dry) {
    kv_fanout_kernel<<<rows, 64, 0, s>>>(b.qkv, ldq, QD, KD, p.row_gt, p.grp_off, p.members, kc, vc, m->kv_cap);
    FO1_LAUNCH_CHECK();
  }
  FO1_RUN(attention_varlen(p.causal, s));
  if (p.own.total_rows > 0) {
    AttnArgs o = p.own;
    o.k = kc; o.v = vc;
    FO1_RUN(attention_varlen(o, s));
  }
  return FO1_OK;
}

static int layer_attention(Model* m, const DecodeAttn& p, const LayerBuf& b, int rows, const float* cs, bf16* kc, bf16* vc, cudaStream_t s,
                           bool dry) {
  const fo1_model_config& c = m->cfg;
  const int hd = c.llm_head_dim, QD = c.llm_heads * hd, KD = c.llm_kv_heads * hd, ldq = QD + 2 * KD;
  FO1_RUN(rope_kv_append(b.qkv, ldq, cs, rows, c.llm_heads, c.llm_kv_heads, hd, p.idx, p.row_slot, kc, vc, m->kv_cap, s));
  FO1_RUN(decode_attention(b.qkv, ldq, kc, vc, p.idx, p.row_slot, rows, p.n_seqs, m->kv_cap, c.llm_heads, c.llm_kv_heads, hd,
                           1.0f / sqrtf((float)hd), b.att, QD, b.dec_part, s));
  return FO1_OK;
}

// one decoder layer over `rows` packed rows, x_in -> x_out, with the attention of a prefill (PrefillAttn) or of a decode step
// (DecodeAttn).  `dry` (the pass that sizes the arena) skips every launch.
template <class Attn>
static int llm_layer(Model* m, int li, const bf16* x_in, bf16* x_out, const LayerBuf& b, int rows, const float* cs, const Attn& at,
                     cudaStream_t s, bool dry) {
  const fo1_model_config& c = m->cfg;
  const LlmLayerW& L = m->llm.layer[li];
  const int H = c.llm_hidden, hd = c.llm_head_dim, QD = c.llm_heads * hd, KD = c.llm_kv_heads * hd, ldq = QD + 2 * KD;
  const int Ip = (c.llm_inter + 31) / 32 * 32;
  const size_t layer_stride = (size_t)m->kv_batch * m->kv_cap * KD;
  bf16* kc = static_cast<bf16*>(m->kv_cache) + (size_t)li * layer_stride;
  bf16* vc = static_cast<bf16*>(m->kv_cache) + ((size_t)c.llm_layers + li) * layer_stride;
  const NormKernel nk = std::is_same<Attn, PrefillAttn>::value ? NORM_WARP : seq_norm_kernel(H);
  FO1_RUN(rmsnorm(x_in, H, L.ln1, b.xn, H, rows, H, c.rms_eps, nk, s));
  FO1_RUN(linear(b.xn, H, L.qkv_w, H, b.qkv, ldq, FO1_BF16, rows, ldq, H, L.qkv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
  FO1_TRY(layer_attention(m, at, b, rows, cs, kc, vc, s, dry));
  FO1_RUN(linear(b.att, QD, L.o_w, QD, b.x_mid, H, FO1_BF16, rows, H, QD, nullptr, 0, FO1_EPI_NONE, x_in, H, 0, s));
  FO1_RUN(rmsnorm(b.x_mid, H, L.ln2, b.xn, H, rows, H, c.rms_eps, nk, s));
  FO1_RUN(linear(b.xn, H, L.gateup_w, H, b.h, Ip, FO1_BF16, rows, 2 * Ip, H, nullptr, 0, FO1_EPI_SILU, nullptr, 0, 1, s));
  FO1_RUN(linear(b.h, Ip, L.down_w, Ip, x_out, H, FO1_BF16, rows, H, Ip, nullptr, 0, FO1_EPI_NONE, b.x_mid, H, 0, s));
  return FO1_OK;
}

// CTAs of the persistent decode kernel for B sequences, or 0 (the per-kernel path): the persistent kernel serves every batch it
// supports (1..32 sequences; scripts/mega_prof.py times the two paths alternately).  FO1_MEGA_MAX_B lowers the threshold,
// FO1_NO_MEGA disables the kernel.
static int mega_grid_for(Model* m, int B) {
  int mega_max_b = 32;
  if (const char* e = getenv("FO1_MEGA_MAX_B")) mega_max_b = std::max(0, std::min(32, atoi(e)));
  return m->llm.mega_ok && B <= mega_max_b && getenv("FO1_NO_MEGA") == nullptr ? decode_mega_grid() : 0;
}

// the buffers both decode paths use after the prefill, carved from the arena (the dry run sizes it)
struct DecodeBufs {
  int mega_grid;                  // CTAs of the persistent kernel (0: the per-kernel path)
  LayerBuf layer;
  bf16 *xa, *xb, *lastn;
  float *cs_dec, *logits, *mg_ssq, *mg_amax_v;
  int *mg_amax_i, *mg_sync, *samp_tok;
  SampleRowParams* samp;
};

// the buffers of DecodeBufs every decode path reads: the layer buffers and the two residual streams for R rows, the per-row decode
// scratch for RD rows, and the persistent kernel's per-CTA slots (g.mega_grid set) and barrier words for B sequences
static void decode_bufs_alloc(Model* m, DecodeBufs& g, int R, int RD, int B) {
  const fo1_model_config& c = m->cfg;
  Arena& A = m->arena;
  const int H = c.llm_hidden, hd = c.llm_head_dim, QD = c.llm_heads * hd, KD = c.llm_kv_heads * hd;
  const int Ip = (c.llm_inter + 31) / 32 * 32;
  LayerBuf& buf = g.layer;
  g.xa = A.alloc<bf16>((size_t)R * H);
  g.xb = A.alloc<bf16>((size_t)R * H);
  buf.xn = A.alloc<bf16>((size_t)R * H);
  buf.qkv = A.alloc<bf16>((size_t)R * (QD + 2 * KD));
  buf.att = A.alloc<bf16>((size_t)R * QD);
  buf.x_mid = A.alloc<bf16>((size_t)R * H);
  buf.h = A.alloc<bf16>((size_t)R * Ip);
  g.cs_dec = A.alloc<float>((size_t)RD * hd);
  buf.dec_part = A.alloc<float>((size_t)RD * c.llm_heads * kDecSplits * (128 + 4));
  g.lastn = A.alloc<bf16>((size_t)RD * H);
  g.logits = A.alloc<float>((size_t)RD * c.llm_vocab);
  g.mg_ssq = A.alloc<float>((size_t)2 * std::max(g.mega_grid, 1) * 32);
  g.mg_amax_v = A.alloc<float>((size_t)std::max(g.mega_grid, 1) * 32);
  g.mg_amax_i = A.alloc<int>((size_t)std::max(g.mega_grid, 1) * 32);
  g.mg_sync = A.alloc<int>((size_t)B * c.llm_kv_heads + 8);
}

// the tokens of the current output column into new_tok (scored: also the column's scores), then their recording; every kernel reads
// the column from *st.step, as the captured decode step does.  `advance`: the column came from a decode step (not the prefill)
static int decode_column(const GenerateCall& q, const DecodeBufs& g, int B, int V, int advance, cudaStream_t s) {
  const ColumnSink& k = q.k;
  const DecodeState& st = k.st;
  const fo1_score_desc* sc = q.sc;
  if (q.mode == DEC_BEAM) return beam_column(q.beam, g.logits, st, advance, s);
  // the logits processors edit the rows first (scored: after storing the raw rows, which score_rows then leaves alone)
  float* raw_out = q.mode == DEC_SCORED ? sc->logits : nullptr;
  if (q.proc.tab != nullptr) {
    FO1_TRY(logits_process(q.proc, g.logits, B, V, k.col != nullptr ? k.col : st.step, k.col != nullptr ? 1 : 0, nullptr, st.finished, k.max_new,
                           k.out_tokens, raw_out, s));
    raw_out = nullptr;
  }
  if (q.mode == DEC_SCORED) {
    FO1_TRY(score_rows(g.logits, V, B, V, g.samp, st.step, st.new_tok, true, st.finished, k.max_new, sc->logprobs, k.max_new, sc->scores,
                       raw_out, V, s));
  } else if (q.mode == DEC_SAMPLED) {
    // the Philox step is read from *st.step, or (slot pool) from each slot's own column
    FO1_TRY(sample_rows(g.logits, V, B, V, g.samp, k.col != nullptr ? k.col : st.step, k.col != nullptr ? 1 : 0, st.new_tok, s));
  } else {
    launch_k(argmax_kernel, dim3(B), dim3(1024), 0, s, g.logits, V, st.new_tok);
    FO1_LAUNCH_CHECK();
  }
  const int threads = std::min(1024, std::max(32, (B + 31) / 32 * 32));
  launch_k(k.stream.progress != nullptr ? decode_update_kernel<true> : decode_update_kernel<false>, dim3(1), dim3(threads), 0, s, k, B, advance);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

// slot pool admission, after the prefill of its n sequences: column 0 from the prefill's last rows (the Philox step is 0), then the
// admitted slots' state (slots_admit_kernel).  The slot list and limits were uploaded to the pool's admission ints by slots_admit.
static int slots_admit_column(const GenerateCall& q, const DecodeBufs& g, int V, const int* d_lens, const int* d_deltas, cudaStream_t s) {
  const SlotPool& p = *q.pool;
  const int n = q.d->n_seqs, N = p.n_slots;
  const int* adm = p.ints + 2 * N;        // slots [N], max_new [N], 0
  if (q.pr != nullptr) FO1_TRY(logits_process(p.proc, g.logits, n, V, adm + 2 * N, 0, adm, nullptr, p.k.max_new, p.k.out_tokens, nullptr, s));
  if (p.mode == DEC_SAMPLED) {
    FO1_TRY(sample_rows(g.logits, V, n, V, g.samp, adm + 2 * N, 0, p.k.st.new_tok, s));
  } else {
    launch_k(argmax_kernel, dim3(n), dim3(1024), 0, s, (const float*)g.logits, V, p.k.st.new_tok);
    FO1_LAUNCH_CHECK();
  }
  slots_admit_kernel<<<1, 256, 0, s>>>(p.k, N, n, adm, adm + N, d_lens, d_deltas, p.k.st.new_tok,
                                       p.mode == DEC_SAMPLED ? g.samp : nullptr, p.prm);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

// the own rows of sequence b in a shared-prefix prefill (L_b without a group)
static int prefix_of(const fo1_prefix_desc* px, int b) { return px && px->seq_group[b] >= 0 ? px->prefix_lens[px->seq_group[b]] : 0; }

// the prefill's attention plan over T packed rows (b: the layer buffers it reads and writes) and the last packed row of every sequence,
// from integer tables cached per shape.  The packed rows are one causal segment per sequence, or with a shared prefix the groups' prefix
// rows (one segment per group) followed by every sequence's own rows.  The cache-write map has one group per sequence with its slot as
// the member; beam search gives each prompt its N slots; a shared prefix puts the prefix groups with their members first, then one
// group per sequence for its own rows at positions P_b + i.
static int prefill_plan(Model* m, const GenerateCall& q, const LayerBuf& b, int T, PrefillAttn& p, const int** d_last, cudaStream_t s) {
  const fo1_model_config& c = m->cfg;
  const fo1_generate_desc* d = q.d;
  const fo1_prefix_desc* px = q.px;
  const int B = d->n_seqs, G = px ? px->n_groups : 0, N = q.bmd ? q.beam.N : 1;
  const int hd = c.llm_head_dim, QD = c.llm_heads * hd, KD = c.llm_kv_heads * hd, ldq = QD + 2 * KD;
  std::vector<int> cu(1, 0), row_gt, grp_off(1, 0), members, last, pre(B), own(B), tiles, rowseg;
  std::string key = "llm:" + std::to_string(N) + ":" + std::to_string(px ? m->kv_cap : 0);
  for (int g = 0; g < G; ++g) {
    cu.push_back(cu.back() + px->prefix_lens[g]);
    for (int t = 0; t < px->prefix_lens[g]; ++t) { row_gt.push_back(g); row_gt.push_back(t); }
    for (int i = 0; i < B; ++i) if (px->seq_group[i] == g) members.push_back(i);
    grp_off.push_back((int)members.size());
    key += ":" + std::to_string(px->prefix_lens[g]);
  }
  int r = cu.back();
  for (int i = 0; i < B; ++i) {
    pre[i] = prefix_of(px, i); own[i] = d->seq_lens[i] - pre[i];
    for (int t = 0; t < own[i]; ++t) { row_gt.push_back(G + i); row_gt.push_back(pre[i] + t); }
    for (int j = 0; j < N; ++j) members.push_back(q.slots ? q.slots[i] : i * N + j);
    grp_off.push_back((int)members.size());
    r += own[i];
    last.push_back(r - 1);
    if (!px) cu.push_back(r);
    key += "/" + std::to_string(px ? px->seq_group[i] : -1) + ":" + std::to_string(d->seq_lens[i]);
    if (q.slots) key += "@" + std::to_string(q.slots[i]);
  }
  const int* gt = nullptr;
  FO1_TRY(cached_ints(m, key + ":gt", row_gt, &gt, s));
  p.row_gt = reinterpret_cast<const int2*>(gt);
  FO1_TRY(cached_ints(m, key + ":go", grp_off, &p.grp_off, s));
  FO1_TRY(cached_ints(m, key + ":mem", members, &p.members, s));
  FO1_TRY(cached_ints(m, key + ":last", last, d_last, s));

  AttnArgs& a = p.causal;
  a = AttnArgs();
  a.q = b.qkv; a.k = b.qkv + QD; a.v = b.qkv + QD + KD; a.o = b.att;
  a.ldq = a.ldk = a.ldv = ldq; a.ldo = QD;
  a.n_seqs = (int)cu.size() - 1; a.total_rows = cu.back(); a.max_seqlen = 0; a.rowseg = b.rowseg;
  for (int i = 0; i < a.n_seqs; ++i) {
    const int len = cu[i + 1] - cu[i];
    a.max_seqlen = std::max(a.max_seqlen, len);
    a.flops += 2.0 * (double)len * len * QD;   // causal: half of 4 L^2 d
  }
  a.q_heads = c.llm_heads; a.kv_heads = c.llm_kv_heads; a.head_dim = hd;
  a.scale = 1.0f / sqrtf((float)hd); a.causal = 1;
  FO1_TRY(cached_ints(m, key + ":cu", cu, &a.cu_seqlens, s));
  attention_tile_table(cu, tiles);        // query tiles restart at every segment
  a.n_tiles = (int)tiles.size() / 2;
  FO1_TRY(cached_ints(m, key + ":til", tiles, &a.tiles, s));

  AttnArgs& o = p.own;
  o = a;
  o.total_rows = 0;
  if (px) {
    const int np = a.total_rows;
    o.q = b.qkv + (size_t)np * ldq; o.o = b.att + (size_t)np * QD;
    o.ldk = o.ldv = KD;
    o.cu_seqlens = nullptr; o.n_seqs = m->kv_batch; o.total_rows = T - np; o.max_seqlen = 0; o.flops = 0.0;
    o.causal = 0; o.kv_rows = m->kv_batch * m->kv_cap;
    prefix_attention_tables(pre.data(), own.data(), B, m->kv_cap, rowseg, tiles);
    o.n_tiles = (int)tiles.size() / 2;
    FO1_TRY(cached_ints(m, key + ":ors", rowseg, &o.rowseg, s));
    FO1_TRY(cached_ints(m, key + ":otil", tiles, &o.tiles, s));
  }
  return FO1_OK;
}

// the prefill's layer stack over T packed rows (with a shared prefix: the n_pre prefix rows, then the own rows), from the caller's
// embeddings and positions through every layer; *x_out: the last layer's output (g.xa or g.xb).  d_lens: the sequences' lengths on
// the device; pos_all: [3][T] scratch of a prefix call.
static int prefill_layers(Model* m, const GenerateCall& q, const PrefillAttn& pa, DecodeBufs& g, long long T, int n_pre, float* cs_pre,
                          int* pos_all, const int* d_lens, cudaStream_t s, bool dry, const bf16** x_out) {
  const fo1_model_config& c = m->cfg;
  const fo1_generate_desc* d = q.d;
  const fo1_prefix_desc* px = q.px;
  const int B = d->n_seqs, H = c.llm_hidden, hd = c.llm_head_dim, KD = c.llm_kv_heads * hd;
  LayerBuf& buf = g.layer;
  const bf16* x = static_cast<const bf16*>(d->inputs_embeds);
  const int* pos = d->position_ids;
  FO1_RUN(attention_rowseg(pa.causal.cu_seqlens, pa.causal.n_seqs, pa.causal.total_rows, buf.rowseg, s));
  if (px) {   // one packed matrix (prefix rows, then own rows) and one position table
    const size_t no = (size_t)T - n_pre;
    if (!dry) {
      FO1_CUDA(cudaMemcpyAsync(g.xb, px->prefix_embeds, (size_t)n_pre * H * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
      FO1_CUDA(cudaMemcpyAsync(g.xb + (size_t)n_pre * H, d->inputs_embeds, no * H * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
      FO1_CUDA(cudaMemcpy2DAsync(pos_all, (size_t)T * sizeof(int), px->prefix_position_ids, (size_t)n_pre * sizeof(int), (size_t)n_pre * sizeof(int),
                                 3, cudaMemcpyDeviceToDevice, s));
      FO1_CUDA(cudaMemcpy2DAsync(pos_all + n_pre, (size_t)T * sizeof(int), d->position_ids, no * sizeof(int), no * sizeof(int), 3,
                                 cudaMemcpyDeviceToDevice, s));
      const size_t layer_stride = (size_t)m->kv_batch * m->kv_cap * KD;
      kv_zero_tail_kernel<<<dim3(B, c.llm_layers), 128, 0, s>>>(static_cast<bf16*>(m->kv_cache) + (size_t)c.llm_layers * layer_stride,
                                                                 (long long)layer_stride, d_lens, m->kv_cap, KD);
      FO1_LAUNCH_CHECK();
    }
    x = g.xb;
    pos = pos_all;
  }
  FO1_RUN(mrope_table(pos, cs_pre, (int)T, hd, c.mrope_section[0], c.mrope_section[1], c.mrope_section[2], c.rope_theta, s));
  for (int li = 0; li < c.llm_layers; ++li) {
    bf16* xo = (li & 1) ? g.xb : g.xa;
    FO1_TRY(llm_layer(m, li, x, xo, buf, (int)T, cs_pre, pa, s, dry));
    x = xo;
  }
  *x_out = x;
  return FO1_OK;
}

// buffer plan, integer tables and the prefill; then (unless `dry`, the pass that sizes the arena) the decode state and column 0
static int llm_prefill(Model* m, GenerateCall& q, cudaStream_t s, bool dry, DecodeBufs& g) {
  const fo1_model_config& c = m->cfg;
  Arena& A = m->arena;
  fo1_generate_desc* d = q.d;
  const fo1_prefix_desc* px = q.px;
  const bool beam = q.bmd != nullptr, lookup = q.lkd != nullptr;
  const int B = d->n_seqs, H = c.llm_hidden, hd = c.llm_head_dim, V = c.llm_vocab;
  long long T = 0;      // packed rows through the layers: every sequence's rows, or (px) the prefix rows then the own rows
  int n_pre = 0;
  for (int b = 0; b < B; ++b) T += d->seq_lens[b] - prefix_of(px, b);
  for (int gi = 0; px && gi < px->n_groups; ++gi) n_pre += px->prefix_lens[gi];
  T += n_pre;
  const int RD = beam ? B * q.beam.N : lookup ? B * (q.lookup.K + 1) : B;   // rows of a decode step: one per sequence, beam or verify row
  const int R = (int)std::max<long long>(T, RD);

  g = DecodeBufs();
  LayerBuf& buf = g.layer;
  // persistent decode kernel (decode_mega.cu): per-CTA slots + the grid barrier
  g.mega_grid = !beam && !lookup ? mega_grid_for(m, B) : 0;
  decode_bufs_alloc(m, g, R, RD, B);
  float* cs_pre = A.alloc<float>((size_t)R * hd);
  buf.rowseg = A.alloc<int>((size_t)R * 2);
  bf16* last = A.alloc<bf16>((size_t)B * H);
  bf16* alln = d->all_logits ? A.alloc<bf16>((size_t)T * H) : nullptr;
  int* d_lens = A.alloc<int>(B);
  int* d_deltas = A.alloc<int>(B);
  int* pos_all = px ? A.alloc<int>((size_t)3 * T) : nullptr;      // prefix positions, then the own rows'
  // sampled or scored decoding: the per-sequence parameters and the tokens the persistent kernel's CTA b drew
  g.samp = q.mode == DEC_SAMPLED || q.mode == DEC_SCORED ? A.alloc<SampleRowParams>(B) : nullptr;
  g.samp_tok = q.mode == DEC_SAMPLED || q.mode == DEC_SCORED ? A.alloc<int>(B) : nullptr;
  if (beam) beam_alloc(A, q.beam);   // beam search: its state and scratch (sized by the dry run like everything else)
  if (lookup) lookup_alloc(A, q.lookup, q.lkd);
  if (q.pr != nullptr && !q.pool) {
    int* pi = A.alloc<int>(q.proc_ints.size());
    q.proc.tab = pi; q.proc.set_of = pi + q.proc_tab_n; q.proc.plen = pi + q.proc_tab_n + B; q.proc.prompt = pi + q.proc_tab_n + 2 * B;
    q.proc.bias = A.alloc<float>(q.proc_bias.size());
  }

  // ---- integer tables and inputs ----
  PrefillAttn pa = {};
  const int* d_last = nullptr;
  if (!dry) {
    FO1_TRY(prefill_plan(m, q, buf, (int)T, pa, &d_last, s));
    FO1_CUDA(cudaMemcpyAsync(d_lens, d->seq_lens, B * sizeof(int), cudaMemcpyHostToDevice, s));
    if (d->rope_deltas_device != nullptr) FO1_CUDA(cudaMemcpyAsync(d_deltas, d->rope_deltas_device, B * sizeof(int), cudaMemcpyDeviceToDevice, s));
    else FO1_CUDA(cudaMemcpyAsync(d_deltas, d->rope_deltas, B * sizeof(int), cudaMemcpyHostToDevice, s));
    if (d->n_stop_ids > 0) FO1_CUDA(cudaMemcpyAsync(q.k.st.stop_ids, d->stop_ids, d->n_stop_ids * sizeof(int), cudaMemcpyHostToDevice, s));
    if (beam) {
      FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(q.beam.prompt_len), d->seq_lens, B * sizeof(int), cudaMemcpyHostToDevice, s));
      FO1_CUDA(cudaMemcpyAsync(const_cast<float*>(q.beam.lp_div), q.lp_div.data(), q.lp_div.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    if (lookup) FO1_TRY(lookup_upload(q.lookup, q.lkd, s));
    if (q.pr != nullptr && !q.pool) {    // (pageable sources: each copy returns once staged)
      FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(q.proc.tab), q.proc_ints.data(), q.proc_ints.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      FO1_CUDA(cudaMemcpyAsync(const_cast<float*>(q.proc.bias), q.proc_bias.data(), q.proc_bias.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    if (q.mode == DEC_SAMPLED || q.mode == DEC_SCORED) {
      // a scored greedy call samples with top_k 1 (bit-identical to greedy) so that both paths score in the sampler's per-row pass
      std::vector<SampleRowParams> h(B);
      for (int b = 0; b < B; ++b) h[b] = score_row_params(q.sp, q.sc ? q.sc->raw_rows : nullptr, b);
      FO1_CUDA(cudaMemcpyAsync(g.samp, h.data(), B * sizeof(SampleRowParams), cudaMemcpyHostToDevice, s));
    }
  }

  // ---- prefill ----
  const bf16* x = nullptr;
  FO1_TRY(prefill_layers(m, q, pa, g, T, n_pre, cs_pre, pos_all, d_lens, s, dry, &x));
  if (d->all_logits) {
    FO1_RUN(rmsnorm(x, H, m->llm.norm, alln, H, (int)T, H, c.rms_eps, NORM_WARP, s));
    FO1_RUN(linear(alln, H, m->llm.lm_head, H, d->all_logits, V, FO1_F32, (int)T, V, H, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
  }
  FO1_RUN(gather_rows_bf16(x, H, d_last, last, H, B, H, s));
  FO1_RUN(rmsnorm(last, H, m->llm.norm, g.lastn, H, B, H, c.rms_eps, seq_norm_kernel(H), s));
  {
    SplitKScope sk(true);       // M = number of sequences: weight streaming
    FO1_RUN(linear(g.lastn, H, m->llm.lm_head, H, g.logits, V, FO1_F32, B, V, H, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
  }
  if (dry) return FO1_OK;
  if (q.pool) return slots_admit_column(q, g, V, d_lens, d_deltas, s);
  if (d->prefill_logits) FO1_CUDA(cudaMemcpyAsync(d->prefill_logits, g.logits, (size_t)B * V * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (beam) {
    FO1_TRY(beam_init(q.beam, q.k.st, d_lens, d_deltas, s));
  } else {
    decode_init_kernel<<<ceil_div(B, 128), 128, 0, s>>>(q.k.st, d_lens, d_deltas, B);
    FO1_LAUNCH_CHECK();
  }
  if (d->max_new_tokens <= 0) return FO1_OK;
  return decode_column(q, g, B, V, 0, s);
}

// the rest of the decode loop as ONE cooperative launch of the persistent kernel
static int decode_persistent(Model* m, const GenerateCall& q, const DecodeBufs& g, cudaStream_t s) {
  const fo1_model_config& c = m->cfg;
  fo1_generate_desc* d = q.d;
  const int B = d->n_seqs;
  MegaArgs a;
  memset(&a, 0, sizeof(a));
  a.B = B; a.layers = c.llm_layers; a.H = c.llm_hidden; a.hd = c.llm_head_dim; a.QD = c.llm_heads * a.hd; a.KD = c.llm_kv_heads * a.hd;
  a.q_heads = c.llm_heads; a.kv_heads = c.llm_kv_heads; a.I = c.llm_inter; a.V = c.llm_vocab; a.eps = c.rms_eps; a.theta = c.rope_theta; a.sec_t = c.mrope_section[0]; a.sec_h = c.mrope_section[1];
  a.layer = static_cast<const MegaLayer*>(m->llm.mega_layers);
  a.head_w = m->llm.head_dec; a.embed = m->llm.embed;
  a.kv_layer_stride = (long long)m->kv_batch * m->kv_cap * a.KD;
  a.kc = static_cast<bf16*>(m->kv_cache); a.vc = a.kc + (size_t)c.llm_layers * a.kv_layer_stride; a.cap = m->kv_cap;
  a.x = g.xa; a.x_mid = g.layer.x_mid; a.qkv = g.layer.qkv; a.att = g.layer.att; a.h = g.layer.h;
  a.ssq = g.mg_ssq; a.cs = g.cs_dec; a.att_part = g.layer.dec_part; a.att_count = g.mg_sync + 8;
  a.amax_val = g.mg_amax_v; a.amax_idx = g.mg_amax_i; a.sink = q.k;
  a.logits = g.logits; a.samp = g.samp; a.samp_tok = g.samp_tok;
  if (q.sc) { a.sc_logprobs = q.sc->logprobs; a.sc_scores = q.sc->scores; a.sc_logits = q.sc->logits; }
  a.proc = q.proc;
  a.n_steps = d->max_new_tokens - 1; a.exit_at = q.exit_at; a.bar = reinterpret_cast<unsigned*>(g.mg_sync);
  const int pairs = B * c.llm_kv_heads;
  a.n_splits = std::max(1, std::min(kMgMaxSplits, g.mega_grid / std::max(1, pairs)));
  FO1_CUDA(cudaMemsetAsync(g.mg_sync, 0, ((size_t)pairs + 8) * sizeof(int), s));
  FO1_TRY(decode_mega_run(a, q.mode, s));
  m->last_decode_path = 1;
  d->steps_run = d->max_new_tokens - 1;
  return FO1_OK;
}

// one decode forward over R rows: the embedding of tok, the M-RoPE table of pos3 ([3][R]), the layers with attention `at`, the final
// norm and the LM head into g.logits
static int decode_forward(Model* m, const DecodeBufs& g, const int* tok, const int* pos3, int R, const DecodeAttn& at, cudaStream_t s) {
  const fo1_model_config& c = m->cfg;
  const int H = c.llm_hidden, V = c.llm_vocab;
  launch_k(embed_tokens_kernel, dim3(R), dim3(256), 0, s, tok, m->llm.embed, g.xa, H);
  FO1_LAUNCH_CHECK();
  FO1_TRY(mrope_table(pos3, g.cs_dec, R, c.llm_head_dim, c.mrope_section[0], c.mrope_section[1], c.mrope_section[2], c.rope_theta, s));
  const bf16* xin = g.xa;
  for (int li = 0; li < c.llm_layers; ++li) {
    bf16* xo = (li & 1) ? g.xa : g.xb;
    FO1_TRY(llm_layer(m, li, xin, xo, g.layer, R, g.cs_dec, at, s, false));
    xin = xo;
  }
  FO1_TRY(rmsnorm(xin, H, m->llm.norm, g.lastn, H, R, H, c.rms_eps, seq_norm_kernel(H), s));
  return linear(g.lastn, H, m->llm.lm_head, H, g.logits, V, FO1_F32, R, V, H, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s);
}

// the rest of the decode loop, per kernel: every step is the SAME launch sequence reading its state from device memory; the first step
// runs eagerly (warms every kernel), the second is captured into a CUDA graph that is replayed afterwards
static int decode_per_kernel(Model* m, const GenerateCall& q, const DecodeBufs& g, cudaStream_t s) {
  const fo1_model_config& c = m->cfg;
  fo1_generate_desc* d = q.d;
  const ColumnSink& k = q.k;
  const bool lookup = q.lkd != nullptr;
  const int B = q.bmd ? q.beam.S * q.beam.N : d->n_seqs, V = c.llm_vocab;
  LlmState* ls = static_cast<LlmState*>(m->llm_state);
  const int R = lookup ? B * (q.lookup.K + 1) : B;     // rows of a step
  const int32_t* h_progress = q.stm ? q.stm->progress : nullptr;
  // programmatic dependent launch: each kernel of the step starts (prologue, weight prefetch) while its predecessor drains
  const bool use_pdl = getenv("FO1_NO_PDL") == nullptr;
  auto enqueue_step = [&]() -> int {
    PdlScope pdl(use_pdl);
    SplitKScope sk(true);       // M = number of sequences in every GEMM of a decode step
    FO1_TRY(decode_forward(m, g, k.st.cur_tok, k.st.pos3, B, DecodeAttn{k.st.cache_len, nullptr, B}, s));
    return decode_column(q, g, B, V, 1, s);
  };
  // prompt lookup: drafts, then ONE verify step over R = B * (K + 1) rows, each computing the plain step's bits for its position
  // (block norms, GEMMs with the M = B choice, the K/V append and attention through the row map), then the acceptance
  auto enqueue_verify = [&]() -> int {
    const LookupArgs& a = q.lookup;
    PdlScope pdl(use_pdl);
    SplitKScope sk(true);
    GemmChoiceScope gc(B);
    FO1_TRY(lookup_drafts(a.corpus, a.ld, a.corpus_len, B, a.K, a.max_ngram, k.st.stop_ids, k.n_stop, a.col, k.max_new, a.drafts, a.n_draft, s));
    FO1_TRY(lookup_rows(a, k.st, s));
    FO1_TRY(decode_forward(m, g, a.row_tok, a.row_pos, R, DecodeAttn{a.row_idx, a.row_slot, B}, s));
    if (q.mode == DEC_SCORED) {
      FO1_TRY(score_rows_lookup(g.logits, V, R, a.K + 1, V, g.samp, a.row_col, a.row_out, a.row_lp, k.st.finished, k.max_new, B, q.sc->scores,
                                q.sc->logits, s));
    } else if (q.mode == DEC_SAMPLED) {
      FO1_TRY(sample_rows(g.logits, V, R, V, a.row_prm, a.row_col, 1, a.row_out, s));   // each row's Philox step is its own column
    } else {
      launch_k(argmax_kernel, dim3(R), dim3(1024), 0, s, (const float*)g.logits, V, a.row_out);
      FO1_LAUNCH_CHECK();
    }
    return lookup_accept(a, k, s);
  };
  auto enqueue = [&]() -> int { return lookup ? enqueue_verify() : enqueue_step(); };
  cudaGraphExec_t gexec = nullptr;
  m->last_decode_path = 0;
  const bool want_graph = !g_prof_on && d->max_new_tokens > 3 && getenv("FO1_NO_GRAPH") == nullptr;
  d->steps_run = 0;
  int rc = FO1_OK;
  cudaEvent_t poll_ev[2] = {nullptr, nullptr};
  if (lookup && d->early_exit_interval > 0)
    for (cudaEvent_t& e : poll_ev) FO1_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (int step = 1; step < d->max_new_tokens; ++step) {
    if (gexec != nullptr) {
      if (cudaGraphLaunch(gexec, s) != cudaSuccess) { set_error("cudaGraphLaunch failed: %s", cudaGetErrorString(cudaGetLastError())); rc = FO1_ERR_CUDA; break; }
      count_launch((uint64_t)c.llm_layers * 9 + (lookup ? 8 : 6) + (q.proc.tab != nullptr ? 1 : 0));
    } else if (want_graph && step == 2) {
      cudaGraph_t graph = nullptr;
      if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        const int erc = enqueue();
        const cudaError_t ce = cudaStreamEndCapture(s, &graph);
        if (erc == FO1_OK && ce == cudaSuccess && graph != nullptr && cudaGraphInstantiate(&gexec, graph, 0) == cudaSuccess) {
          cudaGraphDestroy(graph);
          if (cudaGraphLaunch(gexec, s) != cudaSuccess) { set_error("cudaGraphLaunch failed"); rc = FO1_ERR_CUDA; break; }
        } else {  // capture unavailable: fall back to eager launches (still the same kernels)
          if (graph) cudaGraphDestroy(graph);
          cudaGetLastError();
          gexec = nullptr;
          if ((rc = enqueue()) != FO1_OK) break;
        }
      } else {
        cudaGetLastError();
        if ((rc = enqueue()) != FO1_OK) break;
      }
    } else {
      if ((rc = enqueue()) != FO1_OK) break;
    }
    d->steps_run = step;
    // streamed: `done` is in host memory, so the host loop stops enqueueing without a sync once the device has published it
    if (h_progress != nullptr && (__atomic_load_n(h_progress, __ATOMIC_ACQUIRE) & FO1_STREAM_DONE)) break;
    // prompt lookup: sequences end after a varying number of steps, so the loop polls after every step, one step behind: it waits for
    // the previous step's n_active while this step runs, so the device never waits for the host and at most one step runs past the
    // end of the last sequence
    if (lookup && d->early_exit_interval > 0) {
      const int slot = step & 1;
      if (cudaMemcpyAsync(ls->h_flag + slot, k.st.n_active, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
          cudaEventRecord(poll_ev[slot], s) != cudaSuccess) {
        set_error("early-exit poll failed"); rc = FO1_ERR_CUDA; break;
      }
      if (step > 1) {
        if (cudaEventSynchronize(poll_ev[slot ^ 1]) != cudaSuccess) { set_error("early-exit poll failed"); rc = FO1_ERR_CUDA; break; }
        if (ls->h_flag[slot ^ 1] <= 0) break;
      }
    } else if (d->early_exit_interval > 0 && step % d->early_exit_interval == 0) {
      if (cudaMemcpyAsync(ls->h_flag, k.st.n_active, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
        set_error("early-exit poll failed"); rc = FO1_ERR_CUDA; break;
      }
      if (*ls->h_flag <= q.exit_at) break;  // (exit_at 0: every sequence has emitted a stop id; the tail is already pad_id)
    }
  }
  if (gexec != nullptr) {
    cudaStreamSynchronize(s);   // the exec must outlive its in-flight launches
    cudaGraphExecDestroy(gexec);
  }
  for (cudaEvent_t e : poll_ev)
    if (e != nullptr) cudaEventDestroy(e);
  return rc;
}

// the device aliases of the caller's stream buffers; each must be pinned host memory mapped into the device's address space
static int stream_resolve(const fo1_stream_desc* h, StreamArgs* sa) {
  const char* names[4] = {"tokens", "lens", "progress", "cancel"};
  const void* hp[4] = {h->tokens, h->lens, h->progress, h->cancel};
  void* dp[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int i = 0; i < 4; ++i) {
    if (hp[i] == nullptr) continue;          // (only cancel may be NULL: checked by the caller)
    cudaPointerAttributes at;
    const bool host = cudaPointerGetAttributes(&at, hp[i]) == cudaSuccess && at.type == cudaMemoryTypeHost;
    if (!host || cudaHostGetDevicePointer(&dp[i], const_cast<void*>(hp[i]), 0) != cudaSuccess || dp[i] == nullptr) {
      cudaGetLastError();
      set_error("fo1_llm_generate: stream: stream buffer `%s` is not pinned host memory mapped for the device (cudaHostAlloc, "
                "or cudaHostRegister with cudaHostRegisterMapped)", names[i]);
      return FO1_ERR_INVALID_ARG;
    }
  }
  sa->tokens = static_cast<int*>(dp[0]); sa->lens = static_cast<int*>(dp[1]); sa->progress = static_cast<int*>(dp[2]);
  sa->cancel = static_cast<const int*>(dp[3]);
  return FO1_OK;
}

// host checks of a shared-prefix call: before the model or the device is touched.  who: the entry point named in the messages
static int prefix_check(const fo1_generate_desc* d, const fo1_prefix_desc* px, const char* who = "fo1_llm_generate") {
  FO1_CHECK_ARG(px->n_groups > 0 && px->prefix_lens && px->prefix_embeds && px->prefix_position_ids && px->seq_group,
                "%s: prefix: null prefix argument", who);
  FO1_CHECK_ARG(d->n_seqs > 0 && d->seq_lens, "%s: prefix: null argument", who);
  FO1_CHECK_ARG(d->all_logits == nullptr, "%s: prefix: all_logits is not available with a shared prefix", who);
  std::vector<int> members(px->n_groups, 0);
  for (int b = 0; b < d->n_seqs; ++b) {
    const int g = px->seq_group[b];
    FO1_CHECK_ARG(g >= -1 && g < px->n_groups, "%s: prefix: sequence %d: group %d out of range [-1, %d)", who, b, g, px->n_groups);
    if (g < 0) continue;
    ++members[g];
    FO1_CHECK_ARG(px->prefix_lens[g] >= 1 && px->prefix_lens[g] < d->seq_lens[b],
                  "%s: prefix: sequence %d: prefix %d rows, length %d (1 <= P < L)", who, b, px->prefix_lens[g], d->seq_lens[b]);
  }
  for (int g = 0; g < px->n_groups; ++g)
    FO1_CHECK_ARG(members[g] >= 2, "%s: prefix: group %d has %d member(s) (at least 2)", who, g, members[g]);
  return FO1_OK;
}

// the option pointers of d into q, normalised (an option that asks for nothing is the call without it), then the combination table
// of include/fo1.h, then each option's checks: all before anything is enqueued.  Only the beam and processor checks read the model
// (its vocabulary); the per-sequence host arrays are the caller's, and need neither the model nor the device.
static int generate_check(Model* m, fo1_generate_desc* d, GenerateCall& q) {
  q.d = d; q.sp = d->sampling; q.sc = d->scores; q.stm = d->stream; q.px = d->prefix; q.pr = d->processors; q.lkd = d->lookup;
  q.bmd = d->beam;
  if (q.sc != nullptr && q.sc->logprobs == nullptr && q.sc->scores == nullptr && q.sc->logits == nullptr) q.sc = nullptr;
  if (q.px != nullptr && q.px->n_groups == 0) q.px = nullptr;
  if (q.pr != nullptr) {
    FO1_CHECK_ARG(q.pr->seq_set != nullptr, "fo1_llm_generate: processors: null seq_set");
    bool any = false;
    for (int b = 0; b < d->n_seqs; ++b) any |= q.pr->seq_set[b] >= 0;
    if (!any) q.pr = nullptr;
  }
  const struct { const void* a; const char* an; const void* b; const char* bn; } refused[] = {
      {q.bmd, "beam", q.sp, "sampling"}, {q.bmd, "beam", q.sc, "scores"}, {q.bmd, "beam", q.stm, "stream"},
      {q.bmd, "beam", q.px, "prefix"}, {q.bmd, "beam", q.pr, "processors"}, {q.bmd, "beam", q.lkd, "lookup"},
      {q.lkd, "lookup", q.stm, "stream"}, {q.lkd, "lookup", q.pr, "processors"}};
  for (const auto& r : refused)
    if (r.a != nullptr && r.b != nullptr) {
      set_error("fo1_llm_generate: %s does not combine with %s", r.an, r.bn);
      return FO1_ERR_UNSUPPORTED;
    }
  FO1_CHECK_ARG(q.stm == nullptr || (q.stm->tokens && q.stm->lens && q.stm->progress), "fo1_llm_generate: stream: null stream buffer "
                "(tokens, lens and progress are required; cancel may be NULL)");
  if (q.lkd) FO1_TRY(lookup_check(d, q.lkd));
  if (q.px) FO1_TRY(prefix_check(d, q.px));
  if (q.bmd) FO1_TRY(beam_check(d, q.bmd, m->cfg.llm_vocab));
  if (q.pr) FO1_TRY(proc_check(q.pr, d->n_seqs, m->cfg.llm_vocab, "fo1_llm_generate"));
  if (q.sp) FO1_TRY(sampling_check(q.sp, d->n_seqs, "fo1_llm_generate: sampling"));
  if (q.sc) FO1_TRY(raw_rows_check(q.sp, q.sc->raw_rows, d->n_seqs, "fo1_llm_generate: scores"));
  return FO1_OK;
}

static int llm_generate(Model* m, fo1_generate_desc* d, cudaStream_t s) {
  GenerateCall q{};
  FO1_TRY(generate_check(m, d, q));
  const fo1_stream_desc* stm = q.stm;
  const fo1_beam_desc* bmd = q.bmd;
  const fo1_lookup_desc* lkd = q.lkd;
  const fo1_processor_desc* pr = q.pr;
  const fo1_score_desc* sc = q.sc;
  FO1_CHECK_ARG(m->llm.ok, "fo1_llm_generate: model not finalized (LLM weights unresolved)");
  FO1_CHECK_ARG(m->slot_pool == nullptr, "fo1_llm_generate: a slot pool is open on this model (it owns the K/V cache); fo1_slots_close first");
  const fo1_model_config& c = m->cfg;
  FO1_CHECK_ARG(d->n_seqs > 0 && d->seq_lens && d->inputs_embeds && d->position_ids && (d->rope_deltas || d->rope_deltas_device),
                "fo1_llm_generate: null argument");
  FO1_CHECK_ARG(d->max_new_tokens == 0 || (d->out_tokens && d->out_lens), "fo1_llm_generate: null outputs");
  FO1_CHECK_ARG(c.llm_head_dim == 128, "fo1_llm_generate: head_dim %d unsupported (128)", c.llm_head_dim);
  int max_len = 0;
  for (int b = 0; b < d->n_seqs; ++b) {
    FO1_CHECK_ARG(d->seq_lens[b] > 0, "fo1_llm_generate: sequence %d is empty", b);
    max_len = std::max(max_len, d->seq_lens[b]);
  }
  ColumnSink& k = q.k;
  if (stm) {
    FO1_TRY(stream_resolve(stm, &k.stream));
    __atomic_store_n(stm->progress, d->max_new_tokens > 0 ? 0 : FO1_STREAM_DONE, __ATOMIC_RELEASE);   // before anything is enqueued
  }
  const int rows = bmd ? d->n_seqs * bmd->num_beams : d->n_seqs;     // decode rows / cache slots
  FO1_TRY(ensure_state(m, rows, d->n_stop_ids, &k.st));
  k.n_stop = d->n_stop_ids; k.pad_id = d->pad_id; k.max_new = d->max_new_tokens;
  k.out_tokens = d->out_tokens; k.out_lens = d->out_lens;
  // a greedy call with logits processors draws with top_k 1 (bit-identical to the arg-max) from the stored, processed rows
  q.mode = bmd ? DEC_BEAM : sc ? DEC_SCORED : q.sp || pr ? DEC_SAMPLED : DEC_GREEDY;
  if (pr) {
    std::vector<int> tab;
    proc_table(proc_sets(pr), tab, q.proc_bias);
    const int B = d->n_seqs;
    long long ld = 1;
    for (int b = 0; b < B; ++b) ld = std::max<long long>(ld, pr->prompt_offsets[b + 1] - pr->prompt_offsets[b]);
    q.proc_tab_n = tab.size();
    q.proc_ints = std::move(tab);
    q.proc_ints.resize(q.proc_tab_n + 2 * B + (size_t)B * ld, 0);
    for (int b = 0; b < B; ++b) {
      const int o = pr->prompt_offsets[b], n = pr->prompt_offsets[b + 1] - o;
      q.proc_ints[q.proc_tab_n + b] = pr->seq_set[b];
      q.proc_ints[q.proc_tab_n + B + b] = n;
      std::copy(pr->prompt + o, pr->prompt + o + n, q.proc_ints.begin() + q.proc_tab_n + 2 * B + (size_t)b * ld);
    }
    q.proc.ld = ld;
  }
  // a shared-prefix call rounds the slot up to 64 rows: the cache-reading attention's last key tile stays inside the slot; a lookup
  // call's verify rows write up to K rows past the sequence's last position
  const int n_drafts = lkd ? std::min(lkd->num_tokens, kLookupMaxDrafts) : 0;
  const int cap = max_len + std::max(d->max_new_tokens, 1) + n_drafts;
  FO1_TRY(ensure_kv(m, rows, q.px ? (cap + 63) / 64 * 64 : cap));
  FO1_TRY(int_cache_trim(m));
  if (bmd) {
    BeamArgs& a = q.beam;
    a.S = d->n_seqs; a.N = bmd->num_beams; a.K = bmd->n_keep; a.V = c.llm_vocab; a.max_new = d->max_new_tokens;
    a.num_return = bmd->num_return; a.early_stopping = bmd->early_stopping; a.lp_positive = bmd->length_penalty > 0.0 ? 1 : 0;
    a.n_stop = d->n_stop_ids; a.pad_id = d->pad_id; a.stop_ids = k.st.stop_ids;
    const size_t layer_stride = (size_t)m->kv_batch * m->kv_cap * c.llm_kv_heads * c.llm_head_dim;
    a.kc = static_cast<bf16*>(m->kv_cache); a.vc = a.kc + (size_t)c.llm_layers * layer_stride; a.layer_stride = (long long)layer_stride;
    a.layers = c.llm_layers; a.cap = m->kv_cap; a.kv_dim = c.llm_kv_heads * c.llm_head_dim;
    a.steps_run = bmd->steps_run; a.out_tokens = d->out_tokens; a.out_lens = d->out_lens; a.beam_indices = bmd->beam_indices;
    a.seq_scores = bmd->sequence_scores; a.out_logprobs = bmd->logprobs; a.scores = bmd->scores; a.logits = bmd->logits;
    // HF divides by (len ** length_penalty), a Python float that torch rounds to fp32
    for (int i = 0; i <= a.max_new; ++i) q.lp_div.push_back((float)std::pow((double)i, bmd->length_penalty));
  }
  if (lkd) {
    LookupArgs& a = q.lookup;
    a.B = d->n_seqs; a.K = n_drafts; a.max_ngram = lkd->max_ngram; a.max_new = d->max_new_tokens;
    int longest = 0;
    for (int b = 0; b < d->n_seqs; ++b) longest = std::max(longest, lkd->corpus_offsets[b + 1] - lkd->corpus_offsets[b]);
    a.ld = (long long)longest + std::max(d->max_new_tokens, 1);
    a.logprobs = sc ? sc->logprobs : nullptr;
  }
  m->arena.reset(true);
  DecodeBufs g;
  FO1_TRY(llm_prefill(m, q, s, true, g));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  if (d->max_new_tokens > 0 && !bmd) {  // out_tokens pre-filled with pad so an early exit leaves a clean tail
    const long long n = (long long)d->n_seqs * d->max_new_tokens;
    fill_int_kernel<<<(int)std::min<long long>((n + 255) / 256, 1024), 256, 0, s>>>(d->out_tokens, d->pad_id, n);
    FO1_LAUNCH_CHECK();
    FO1_CUDA(cudaMemsetAsync(d->out_lens, 0, d->n_seqs * sizeof(int), s));
    if (sc && sc->logprobs) FO1_CUDA(cudaMemsetAsync(sc->logprobs, 0, (size_t)n * sizeof(float), s));      // 0 past out_lens
  }
  FO1_TRY(llm_prefill(m, q, s, false, g));
  if (d->max_new_tokens <= 0) return FO1_OK;
  if (lkd) FO1_TRY(lookup_init(q.lookup, k.st, g.samp, s));
  if (g.mega_grid > 0 && d->max_new_tokens > 1) return decode_persistent(m, q, g, s);
  FO1_TRY(decode_per_kernel(m, q, g, s));
  return bmd ? beam_finalize(q.beam, s) : FO1_OK;
}

// -------------------------------------------------------------------------------- teacher-forced scoring
// the generate descriptor of a scoring call's prefill (no decoding), and every host check of include/fo1.h, before anything is enqueued
static int loglik_check(Model* m, const fo1_loglik_desc* d, fo1_generate_desc* gd, const fo1_prefix_desc** px_out) {
  FO1_CHECK_ARG(d->n_seqs > 0 && d->seq_lens && d->inputs_embeds && d->position_ids && d->targets, "fo1_llm_loglik: null argument");
  FO1_CHECK_ARG(d->logprobs && d->seq_logprob && d->seq_count, "fo1_llm_loglik: null output (logprobs, seq_logprob and seq_count are required)");
  *gd = fo1_generate_desc{};
  gd->n_seqs = d->n_seqs; gd->seq_lens = d->seq_lens; gd->inputs_embeds = d->inputs_embeds; gd->position_ids = d->position_ids;
  gd->all_logits = d->all_logits;
  const fo1_prefix_desc* px = d->prefix != nullptr && d->prefix->n_groups > 0 ? d->prefix : nullptr;
  for (int b = 0; b < d->n_seqs; ++b) FO1_CHECK_ARG(d->seq_lens[b] > 0, "fo1_llm_loglik: sequence %d is empty", b);
  if (px) FO1_TRY(prefix_check(gd, px, "fo1_llm_loglik"));
  const int V = m->cfg.llm_vocab;
  long long r = 0;
  for (int b = 0; b < d->n_seqs; ++b) {
    const int L = d->seq_lens[b], P = prefix_of(px, b);
    for (int t = 0; t < L; ++t, ++r) {
      const int tg = d->targets[r];
      if (tg == -100) continue;
      FO1_CHECK_ARG(tg >= 0 && tg < V, "fo1_llm_loglik: sequence %d row %d: target %d is outside [0, %d) and not -100", b, t, tg, V);
      FO1_CHECK_ARG(t < L - 1, "fo1_llm_loglik: sequence %d: its last row (%d) is scored; it has no next token", b, t);
      FO1_CHECK_ARG(t >= P, "fo1_llm_loglik: sequence %d row %d is scored inside its shared prefix of %d rows", b, t, P);
    }
  }
  FO1_CHECK_ARG(m->slot_pool == nullptr, "fo1_llm_loglik: a slot pool is open on this model (it owns the K/V cache); fo1_slots_close first");
  *px_out = px;
  return FO1_OK;
}

// the prefill of fo1_llm_generate (prefill_plan, prefill_layers), then the scored rows only: gathered, normed with the all_logits
// path's kernel, the log-likelihood head and the merge; `dry` sizes the arena
static int llm_loglik_run(Model* m, const fo1_loglik_desc* ld, GenerateCall& q, const std::vector<int>& ints, int n_scored, cudaStream_t s,
                          bool dry) {
  const fo1_model_config& c = m->cfg;
  Arena& A = m->arena;
  const fo1_generate_desc* d = q.d;
  const fo1_prefix_desc* px = q.px;
  const int B = d->n_seqs, H = c.llm_hidden, hd = c.llm_head_dim, V = c.llm_vocab, Ms = n_scored;
  const int n_parts = ceil_div(V, kLoglikTile);
  long long T = 0, rows = 0;
  int n_pre = 0;
  for (int b = 0; b < B; ++b) { T += d->seq_lens[b] - prefix_of(px, b); rows += d->seq_lens[b]; }
  for (int gi = 0; px && gi < px->n_groups; ++gi) n_pre += px->prefix_lens[gi];
  T += n_pre;
  DecodeBufs g{};
  decode_bufs_alloc(m, g, (int)T, 1, B);
  float* cs_pre = A.alloc<float>((size_t)T * hd);
  g.layer.rowseg = A.alloc<int>((size_t)T * 2);
  int* d_lens = A.alloc<int>(B);
  int* pos_all = px ? A.alloc<int>((size_t)3 * T) : nullptr;
  bf16* alln = d->all_logits ? A.alloc<bf16>((size_t)T * H) : nullptr;
  bf16* xs = A.alloc<bf16>((size_t)std::max(Ms, 1) * H);
  bf16* xn = A.alloc<bf16>((size_t)std::max(Ms, 1) * H);
  float4* part = A.alloc<float4>((size_t)std::max(Ms, 1) * n_parts);
  float* xt = A.alloc<float>(std::max(Ms, 1));
  int* di = A.alloc<int>(ints.size());     // packed rows [Ms], full rows [Ms], targets [Ms], sequence offsets [B + 1], counts [B]
  const int *d_pack = di, *d_full = di + Ms, *d_tgt = di + 2 * Ms, *d_off = di + 3 * Ms, *d_cnt = di + 3 * Ms + B + 1;
  PrefillAttn pa = {};
  const int* d_last = nullptr;
  if (!dry) {
    FO1_TRY(prefill_plan(m, q, g.layer, (int)T, pa, &d_last, s));
    FO1_CUDA(cudaMemcpyAsync(d_lens, d->seq_lens, B * sizeof(int), cudaMemcpyHostToDevice, s));
    FO1_CUDA(cudaMemcpyAsync(di, ints.data(), ints.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: returns once staged)
  }
  const bf16* x = nullptr;
  FO1_TRY(prefill_layers(m, q, pa, g, T, n_pre, cs_pre, pos_all, d_lens, s, dry, &x));
  if (d->all_logits) {
    FO1_RUN(rmsnorm(x, H, m->llm.norm, alln, H, (int)T, H, c.rms_eps, NORM_WARP, s));
    FO1_RUN(linear(alln, H, m->llm.lm_head, H, d->all_logits, V, FO1_F32, (int)T, V, H, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
  }
  if (dry) return FO1_OK;
  FO1_CUDA(cudaMemsetAsync(ld->logprobs, 0, (size_t)rows * sizeof(float), s));
  if (ld->greedy) FO1_CUDA(cudaMemsetAsync(ld->greedy, 0, (size_t)rows * sizeof(int), s));
  if (Ms > 0) {
    FO1_TRY(gather_rows_bf16(x, H, d_pack, xs, H, Ms, H, s));
    FO1_TRY(rmsnorm(xs, H, m->llm.norm, xn, H, Ms, H, c.rms_eps, NORM_WARP, s));   // the all_logits rows' kernel: the same bits
    FO1_TRY(loglik_head(xn, m->llm.lm_head, Ms, V, H, d_tgt, part, xt, s));
    FO1_TRY(loglik_merge(part, n_parts, Ms, d_tgt, xt, d_full, ld->logprobs, ld->greedy, ld->lse, ld->target_logits, s));
  }
  FO1_TRY(loglik_seq_sum(ld->logprobs, d_off, B, ld->seq_logprob, s));
  FO1_CUDA(cudaMemcpyAsync(ld->seq_count, d_cnt, B * sizeof(int), cudaMemcpyDeviceToDevice, s));
  return FO1_OK;
}

static int llm_loglik(Model* m, const fo1_loglik_desc* ld, cudaStream_t s) {
  fo1_generate_desc gd;
  GenerateCall q{};
  FO1_TRY(loglik_check(m, ld, &gd, &q.px));
  q.d = &gd;
  FO1_CHECK_ARG(m->llm.ok, "fo1_llm_loglik: model not finalized (LLM weights unresolved)");
  const fo1_model_config& c = m->cfg;
  FO1_CHECK_ARG(c.llm_head_dim == 128, "fo1_llm_loglik: head_dim %d unsupported (128)", c.llm_head_dim);
  const int B = gd.n_seqs;
  // scored rows in row order: their packed row (prefix rows first with a shared prefix), their row over the full sequences, target
  std::vector<int> pack, full, tgt, off(1, 0), cnt(B, 0);
  int n_pre = 0, max_len = 0;
  for (int gi = 0; q.px && gi < q.px->n_groups; ++gi) n_pre += q.px->prefix_lens[gi];
  int own0 = n_pre;
  for (int b = 0; b < B; ++b) {
    const int L = gd.seq_lens[b], P = prefix_of(q.px, b);
    max_len = std::max(max_len, L);
    for (int t = 0; t < L; ++t) {
      const int r = off.back() + t;
      if (ld->targets[r] == -100) continue;
      pack.push_back(q.px ? own0 + t - P : r); full.push_back(r); tgt.push_back(ld->targets[r]);
      ++cnt[b];
    }
    own0 += L - P;
    off.push_back(off.back() + L);
  }
  const int Ms = (int)pack.size();
  std::vector<int> ints(pack);
  ints.insert(ints.end(), full.begin(), full.end());
  ints.insert(ints.end(), tgt.begin(), tgt.end());
  ints.insert(ints.end(), off.begin(), off.end());
  ints.insert(ints.end(), cnt.begin(), cnt.end());
  // the cache the prefill of fo1_llm_generate with max_new_tokens 0 uses (a shared prefix rounds the slot up to 64 rows)
  FO1_TRY(ensure_kv(m, B, q.px ? (max_len + 1 + 63) / 64 * 64 : max_len + 1));
  FO1_TRY(int_cache_trim(m));
  m->arena.reset(true);
  FO1_TRY(llm_loglik_run(m, ld, q, ints, Ms, s, true));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  return llm_loglik_run(m, ld, q, ints, Ms, s, false);
}

// -------------------------------------------------------------------------------- slot pool
static void slots_free(Model* m) {
  SlotPool* p = static_cast<SlotPool*>(m->slot_pool);
  if (!p) return;
  if (p->ints) cudaFree(p->ints);
  if (p->prm) cudaFree(p->prm);
  if (p->proc_ints) cudaFree(p->proc_ints);
  if (p->proc.tab) cudaFree(const_cast<int*>(p->proc.tab));
  if (p->proc.bias) cudaFree(const_cast<float*>(p->proc.bias));
  delete p;
  m->slot_pool = nullptr;
}

// the device state of a freshly registered pool (its caller frees the pool if this fails)
static int slots_init(SlotPool* p, const fo1_slots_desc* o, const DecodeState& st, cudaStream_t s) {
  const int N = o->n_slots;
  p->n_slots = N; p->interval = o->early_exit_interval; p->mode = o->sampled ? DEC_SAMPLED : DEC_GREEDY;
  p->busy.assign(N, 0);
  ColumnSink& k = p->k;
  k = ColumnSink();
  k.st = st;
  k.st.finished = o->finished;
  k.n_stop = o->n_stop_ids; k.pad_id = o->pad_id; k.max_new = o->max_new_tokens;
  k.out_tokens = o->out_tokens; k.out_lens = o->out_lens;
  if (cudaMalloc(reinterpret_cast<void**>(&p->ints), ((size_t)4 * N + 1) * sizeof(int)) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&p->prm), (size_t)N * sizeof(SampleRowParams)) != cudaSuccess) {
    cudaGetLastError();
    set_error("fo1_slots_open: out of device memory for %d slots", N);
    return FO1_ERR_CUDA;
  }
  k.col = p->ints; k.max_new_row = p->ints + N;
  // every slot starts idle (finished, nothing running): an idle slot's rows still run in each step, so its state must be valid
  FO1_CUDA(cudaMemsetAsync(p->ints, 0, ((size_t)4 * N + 1) * sizeof(int), s));
  FO1_CUDA(cudaMemsetAsync(st.cache_len, 0, (size_t)N * sizeof(int), s));
  for (int a = 0; a < 3; ++a) FO1_CUDA(cudaMemsetAsync(st.pos3 + (size_t)a * N, 0, (size_t)N * sizeof(int), s));
  FO1_CUDA(cudaMemsetAsync(st.cur_tok, 0, (size_t)N * sizeof(int), s));
  FO1_CUDA(cudaMemsetAsync(st.n_active, 0, sizeof(int), s));
  FO1_CUDA(cudaMemsetAsync(st.step, 0, sizeof(int), s));
  FO1_CUDA(cudaMemsetAsync(o->out_lens, 0, (size_t)N * sizeof(int), s));
  fill_int_kernel<<<ceil_div(N, 256), 256, 0, s>>>(o->finished, 1, N);
  FO1_LAUNCH_CHECK();
  if (o->n_stop_ids > 0) FO1_CUDA(cudaMemcpyAsync(st.stop_ids, o->stop_ids, o->n_stop_ids * sizeof(int), cudaMemcpyHostToDevice, s));
  const std::vector<SampleRowParams> greedy(N, SampleRowParams{1.0f, 1.0f, 1, 0, 0ull});
  FO1_CUDA(cudaMemcpyAsync(p->prm, greedy.data(), greedy.size() * sizeof(SampleRowParams), cudaMemcpyHostToDevice, s));
  return cudaStreamSynchronize(s) == cudaSuccess ? FO1_OK : (set_error("fo1_slots_open: %s", cudaGetErrorString(cudaGetLastError())), FO1_ERR_CUDA);
}

static int slots_open(Model* m, const fo1_slots_desc* o, cudaStream_t s) {
  FO1_CHECK_ARG(m->llm.ok, "fo1_slots_open: model not finalized (LLM weights unresolved)");
  FO1_CHECK_ARG(m->slot_pool == nullptr, "fo1_slots_open: a slot pool is already open on this model");
  FO1_CHECK_ARG(m->cfg.llm_head_dim == 128, "fo1_slots_open: head_dim %d unsupported (128)", m->cfg.llm_head_dim);
  FO1_CHECK_ARG(o->n_slots >= 1 && o->n_slots <= 65535, "fo1_slots_open: n_slots %d out of range [1, 65535]", o->n_slots);
  FO1_CHECK_ARG(o->max_new_tokens >= 1 && o->cap > o->max_new_tokens, "fo1_slots_open: max_new_tokens %d / cap %d (1 <= max_new_tokens < cap)",
                o->max_new_tokens, o->cap);
  FO1_CHECK_ARG(o->early_exit_interval >= 1, "fo1_slots_open: early_exit_interval %d must be >= 1", o->early_exit_interval);
  FO1_CHECK_ARG(o->n_stop_ids >= 0 && (o->n_stop_ids == 0 || o->stop_ids), "fo1_slots_open: null stop_ids");
  FO1_CHECK_ARG(o->out_tokens && o->out_lens && o->finished, "fo1_slots_open: null outputs");
  const int N = o->n_slots;
  DecodeState st;
  FO1_TRY(ensure_state(m, N, o->n_stop_ids, &st));
  FO1_TRY(ensure_kv(m, N, o->cap));
  SlotPool* p = new SlotPool();
  m->slot_pool = p;
  const int rc = slots_init(p, o, st, s);
  if (rc != FO1_OK) slots_free(m);      // a pool that failed to open is not left registered: generate calls stay possible
  return rc;
}

// an admission's processors: its sets join the pool's distinct sets (the device table is rebuilt when one is new), and each admitted
// slot gets its set and prompt ids
static int slots_proc_admit(SlotPool* p, const fo1_processor_desc* pr, const int* slots, int n, int cap, cudaStream_t s) {
  const int N = p->n_slots;
  if (p->proc_ints == nullptr) {
    if (cudaMalloc(reinterpret_cast<void**>(&p->proc_ints), ((size_t)2 * N + (size_t)N * cap) * sizeof(int)) != cudaSuccess) {
      cudaGetLastError();
      set_error("fo1_slots_admit: out of device memory for the processors' prompt rows");
      return FO1_ERR_CUDA;
    }
    p->slot_set.assign(N, -1);
    p->proc.set_of = p->proc_ints; p->proc.plen = p->proc_ints + N; p->proc.prompt = p->proc_ints + 2 * N; p->proc.ld = cap;
  }
  const std::vector<ProcSet> sets = proc_sets(pr);
  std::vector<std::vector<int>> keys;
  bool fresh = p->proc.tab == nullptr;
  for (const ProcSet& ps : sets) {
    keys.push_back(ps.key());
    fresh |= p->proc_index.count(keys.back()) == 0;
  }
  for (int i = 0; i < n; ++i) p->slot_set[slots[i]] = -1;
  if (fresh) {
    // keep the sets of the running slots (renumbered), then add the new ones
    std::vector<int> remap(p->proc_sets.size(), -1);
    std::vector<ProcSet> kept;
    std::map<std::vector<int>, int> index;
    for (int b = 0; b < N; ++b) {
      int& g = p->slot_set[b];
      if (g < 0 || !p->busy[b]) { g = -1; continue; }
      if (remap[g] < 0) {
        remap[g] = (int)kept.size();
        index.emplace(p->proc_sets[g].key(), remap[g]);
        kept.push_back(p->proc_sets[g]);
      }
      g = remap[g];
    }
    p->proc_sets = std::move(kept);
    p->proc_index = std::move(index);
  }
  std::vector<int> global(sets.size());
  for (size_t i = 0; i < sets.size(); ++i) {
    auto it = p->proc_index.emplace(keys[i], (int)p->proc_sets.size());
    if (it.second) p->proc_sets.push_back(sets[i]);
    global[i] = it.first->second;
  }
  if (fresh) {
    std::vector<int> tab;
    std::vector<float> bias;
    proc_table(p->proc_sets, tab, bias);
    if (tab.size() > p->proc_tab_cap || bias.size() > p->proc_bias_cap) {
      FO1_CUDA(cudaStreamSynchronize(s));       // an earlier admission's launches may still read the old table
      if (p->proc.tab) cudaFree(const_cast<int*>(p->proc.tab));
      if (p->proc.bias) cudaFree(const_cast<float*>(p->proc.bias));
      p->proc.tab = nullptr; p->proc.bias = nullptr;
      p->proc_tab_cap = std::max(tab.size(), 2 * p->proc_tab_cap);
      p->proc_bias_cap = std::max(bias.size(), 2 * p->proc_bias_cap);
      int* t = nullptr;
      float* bb = nullptr;
      FO1_CUDA(cudaMalloc(reinterpret_cast<void**>(&t), p->proc_tab_cap * sizeof(int)));
      p->proc.tab = t;
      FO1_CUDA(cudaMalloc(reinterpret_cast<void**>(&bb), p->proc_bias_cap * sizeof(float)));
      p->proc.bias = bb;
    }
    FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(p->proc.tab), tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    FO1_CUDA(cudaMemcpyAsync(const_cast<float*>(p->proc.bias), bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  for (int i = 0; i < n; ++i) {
    const int b = slots[i], o = pr->prompt_offsets[i], len = pr->prompt_offsets[i + 1] - o;
    p->slot_set[b] = pr->seq_set[i] >= 0 ? global[pr->seq_set[i]] : -1;
    FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(p->proc.plen) + b, &len, sizeof(int), cudaMemcpyHostToDevice, s));
    if (len > 0)
      FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(p->proc.prompt) + (size_t)b * cap, pr->prompt + o, len * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  // (pageable source: the copy returns once staged)
  FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(p->proc.set_of), p->slot_set.data(), N * sizeof(int), cudaMemcpyHostToDevice, s));
  return FO1_OK;
}

// an admission without processors into a pool that has them: its slots get no set
static int slots_proc_clear(SlotPool* p, const int* slots, int n, cudaStream_t s) {
  for (int i = 0; i < n; ++i) p->slot_set[slots[i]] = -1;
  FO1_CUDA(cudaMemcpyAsync(const_cast<int*>(p->proc.set_of), p->slot_set.data(), p->n_slots * sizeof(int), cudaMemcpyHostToDevice, s));
  return FO1_OK;
}

static int slots_admit(Model* m, const fo1_slots_admit_desc* a, cudaStream_t s) {
  SlotPool* p = static_cast<SlotPool*>(m->slot_pool);
  FO1_CHECK_ARG(p != nullptr, "fo1_slots_admit: no slot pool is open");
  const int N = p->n_slots, n = a->n;
  FO1_CHECK_ARG(n >= 1 && n <= N, "fo1_slots_admit: %d sequences for %d slots", n, N);
  FO1_CHECK_ARG(a->slots && a->seq_lens && a->max_new_tokens && a->inputs_embeds && a->position_ids && a->rope_deltas_device,
                "fo1_slots_admit: null argument");
  if (a->sampling) {
    FO1_CHECK_ARG(p->mode == DEC_SAMPLED, "fo1_slots_admit: sampling parameters for a pool opened without sampling");
    FO1_TRY(sampling_check(a->sampling, n, "fo1_slots_admit"));
  }
  std::vector<char> seen(N, 0);
  for (int i = 0; i < n; ++i) {
    const int b = a->slots[i];
    FO1_CHECK_ARG(b >= 0 && b < N, "fo1_slots_admit: sequence %d: slot %d out of range [0, %d)", i, b, N);
    FO1_CHECK_ARG(!p->busy[b] && !seen[b], "fo1_slots_admit: sequence %d: slot %d is occupied", i, b);
    seen[b] = 1;
    FO1_CHECK_ARG(a->max_new_tokens[i] >= 1 && a->max_new_tokens[i] <= p->k.max_new,
                  "fo1_slots_admit: sequence %d: max_new_tokens %d out of range [1, %d]", i, a->max_new_tokens[i], p->k.max_new);
    FO1_CHECK_ARG(a->seq_lens[i] >= 1 && a->seq_lens[i] + a->max_new_tokens[i] <= m->kv_cap,
                  "fo1_slots_admit: sequence %d: %d prompt rows + %d new tokens exceed the slot capacity %d", i, a->seq_lens[i],
                  a->max_new_tokens[i], m->kv_cap);
  }
  const fo1_processor_desc* pr = a->processors;
  if (pr) {
    FO1_TRY(proc_check(pr, n, m->cfg.llm_vocab, "fo1_slots_admit"));
    for (int i = 0; i < n; ++i)
      FO1_CHECK_ARG(pr->prompt_offsets[i + 1] - pr->prompt_offsets[i] <= m->kv_cap, "fo1_slots_admit: sequence %d: %d prompt ids exceed the slot "
                    "capacity %d", i, pr->prompt_offsets[i + 1] - pr->prompt_offsets[i], m->kv_cap);
    FO1_TRY(slots_proc_admit(p, pr, a->slots, n, m->kv_cap, s));
  } else if (p->proc.tab != nullptr) {
    FO1_TRY(slots_proc_clear(p, a->slots, n, s));
  }
  fo1_generate_desc d{};
  d.n_seqs = n; d.seq_lens = a->seq_lens; d.inputs_embeds = a->inputs_embeds; d.position_ids = a->position_ids;
  d.rope_deltas_device = a->rope_deltas_device; d.max_new_tokens = 1; d.pad_id = p->k.pad_id;
  GenerateCall q{};
  q.d = &d; q.sp = a->sampling; q.mode = p->mode; q.k = p->k; q.pool = p; q.slots = a->slots; q.pr = pr;
  FO1_TRY(int_cache_trim(m));
  FO1_CUDA(cudaMemcpyAsync(p->ints + 2 * N, a->slots, n * sizeof(int), cudaMemcpyHostToDevice, s));
  FO1_CUDA(cudaMemcpyAsync(p->ints + 3 * N, a->max_new_tokens, n * sizeof(int), cudaMemcpyHostToDevice, s));
  m->arena.reset(true);
  DecodeBufs g;
  FO1_TRY(llm_prefill(m, q, s, true, g));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  FO1_TRY(llm_prefill(m, q, s, false, g));
  for (int i = 0; i < n; ++i) p->busy[a->slots[i]] = 1;
  return FO1_OK;
}

// the decode buffers of n_slots rows: only per-step scratch, so each segment carves them anew
static void slots_decode_bufs(Model* m, const SlotPool& p, DecodeBufs& g) {
  g = DecodeBufs();
  g.mega_grid = mega_grid_for(m, p.n_slots);
  decode_bufs_alloc(m, g, p.n_slots, p.n_slots, p.n_slots);
  g.samp = pool_mode(p) == DEC_SAMPLED ? p.prm : nullptr;
  g.samp_tok = m->arena.alloc<int>(p.n_slots);
}

static int slots_decode(Model* m, int exit_at, int* steps_run, cudaStream_t s) {
  SlotPool* p = static_cast<SlotPool*>(m->slot_pool);
  FO1_CHECK_ARG(p != nullptr, "fo1_slots_decode: no slot pool is open");
  FO1_CHECK_ARG(exit_at >= 0, "fo1_slots_decode: exit_at %d must be >= 0", exit_at);
  LlmState* ls = static_cast<LlmState*>(m->llm_state);
  const DecodeState& st = p->k.st;
  const int N = p->n_slots;
  // h_flag: [0] n_active, [1] the step counter before the segment, [2] after it
  FO1_CUDA(cudaMemcpyAsync(ls->h_flag, st.n_active, sizeof(int), cudaMemcpyDeviceToHost, s));
  FO1_CUDA(cudaMemcpyAsync(ls->h_flag + 1, st.step, sizeof(int), cudaMemcpyDeviceToHost, s));
  FO1_CUDA(cudaStreamSynchronize(s));
  const int step0 = ls->h_flag[1];
  if (ls->h_flag[0] > exit_at) {
    // a running slot finishes within max_new steps (its own limit), so a segment needs at most that many
    fo1_generate_desc d{};
    d.n_seqs = N; d.max_new_tokens = p->k.max_new + 1; d.early_exit_interval = p->interval; d.pad_id = p->k.pad_id;
    GenerateCall q{};
    q.d = &d; q.mode = pool_mode(*p); q.k = p->k; q.pool = p; q.exit_at = exit_at; q.proc = p->proc;
    DecodeBufs g;
    m->arena.reset(true);
    slots_decode_bufs(m, *p, g);
    FO1_TRY(arena_ensure(m, m->arena.peak));
    m->arena.reset(false);
    slots_decode_bufs(m, *p, g);
    if (g.mega_grid > 0) FO1_TRY(decode_persistent(m, q, g, s));
    else FO1_TRY(decode_per_kernel(m, q, g, s));
  }
  std::vector<int> fin(N);
  FO1_CUDA(cudaMemcpyAsync(ls->h_flag + 2, st.step, sizeof(int), cudaMemcpyDeviceToHost, s));
  FO1_CUDA(cudaMemcpyAsync(fin.data(), st.finished, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, s));
  FO1_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < N; ++b)
    if (fin[b]) p->busy[b] = 0;
  *steps_run = ls->h_flag[2] - step0;
  return FO1_OK;
}

// -------------------------------------------------------------------------------- splice plan (host, integer)
static int splice_plan(const int64_t* ids, int n_ids, const int32_t* grid_hw, int n_images, int n_regions, const fo1_splice_cfg& cf,
                       std::vector<int64_t>& new_ids, std::vector<int>& kind, std::vector<int>& index, std::vector<int>& pos,
                       int* rope_delta) {
  // ---- omchat_qwen2_5_vl.py:318-368: walk the ids, expand image placeholders, keep one slot per region ----
  int cur_img = 0, cur_reg = 0, img_row = 0;
  const int unit = cf.merge * cf.merge;
  for (int i = 0; i < n_ids; ++i) {
    const int64_t t = ids[i];
    if (t == cf.image_placeholder) {
      if (cur_img >= n_images) { set_error("fo1_splice_plan: more image placeholders than images (%d)", n_images); return FO1_ERR_INVALID_ARG; }
      const int n = grid_hw[2 * cur_img] * grid_hw[2 * cur_img + 1] / unit;
      for (int k = 0; k < n; ++k) { new_ids.push_back(cf.image_token_id); kind.push_back(1); index.push_back(img_row + k); }
      img_row += n;
      ++cur_img;
    } else if (t == cf.region_placeholder) {
      if (cur_reg >= n_regions) { set_error("fo1_splice_plan: more region placeholders than region features (%d)", n_regions); return FO1_ERR_INVALID_ARG; }
      new_ids.push_back(cf.region_placeholder); kind.push_back(2); index.push_back(cur_reg++);
    } else {
      new_ids.push_back(t); kind.push_back(0); index.push_back((int)t);
    }
  }
  // ---- get_rope_index (modeling_qwen2_5_vl.py:1625-1699) on the spliced ids, attention mask all ones ----
  const int L = (int)new_ids.size();
  pos.assign((size_t)3 * L, 0);
  int image_nums = 0;
  for (int i = 0; i + 1 < L; ++i)
    if (new_ids[i] == cf.vision_start_token_id && new_ids[i + 1] == cf.image_token_id) ++image_nums;
  // (a vision_start in the last position indexes out of range in the reference; treated as "no image" here)
  int st = 0, image_index = 0;
  long long next_base = 0;   // llm_pos_ids_list[-1].max() + 1
  bool have_any = false;
  auto emit_text = [&](int from, int len, long long base) {
    for (int k = 0; k < len; ++k)
      for (int a = 0; a < 3; ++a) pos[(size_t)a * L + from + k] = (int)(base + k);
  };
  for (int it = 0; it < image_nums; ++it) {
    int ed = -1;
    for (int i = st; i < L; ++i) if (new_ids[i] == cf.image_token_id) { ed = i; break; }
    if (ed < 0 || image_index >= n_images) { set_error("fo1_splice_plan: image token bookkeeping mismatch"); return FO1_ERR_INVALID_ARG; }
    const int lh = grid_hw[2 * image_index] / cf.merge, lw = grid_hw[2 * image_index + 1] / cf.merge;
    ++image_index;
    const int text_len = ed - st;
    const long long st_idx = have_any ? next_base : 0;
    emit_text(st, text_len, st_idx);
    const long long vb = st_idx + text_len;
    for (int y = 0; y < lh; ++y)
      for (int x = 0; x < lw; ++x) {
        const size_t p = (size_t)ed + (size_t)y * lw + x;
        if (p >= (size_t)L) { set_error("fo1_splice_plan: image tokens overrun the sequence"); return FO1_ERR_INVALID_ARG; }
        pos[p] = (int)vb;                     // t index = 0 for an image
        pos[(size_t)L + p] = (int)(vb + y);
        pos[(size_t)2 * L + p] = (int)(vb + x);
      }
    long long mx = vb + std::max(lh, lw) - 1;
    if (text_len > 0) mx = std::max(mx, st_idx + text_len - 1);
    next_base = mx + 1;
    have_any = true;
    st = ed + lh * lw;
  }
  long long maxpos = have_any ? next_base - 1 : -1;
  if (st < L) {
    const long long st_idx = have_any ? next_base : 0;
    emit_text(st, L - st, st_idx);
    maxpos = st_idx + (L - st) - 1;
  }
  *rope_delta = (int)(maxpos + 1 - L);
  return FO1_OK;
}

}  // namespace fo1

using namespace fo1;

extern "C" int fo1_splice_plan(const int64_t* input_ids, int32_t n_ids, const int32_t* image_grid_hw, int32_t n_images,
                               int32_t n_regions, const fo1_splice_cfg* cfg, int64_t* new_ids, int32_t* src_kind,
                               int32_t* src_index, int32_t* position_ids, int32_t* rope_delta, int32_t* out_len, int32_t capacity) {
  FO1_CHECK_ARG(input_ids && cfg && out_len && rope_delta && n_ids >= 0 && (n_images == 0 || image_grid_hw), "fo1_splice_plan: null argument");
  FO1_CHECK_ARG(cfg->merge > 0, "fo1_splice_plan: merge must be positive");
  std::vector<int64_t> ids;
  std::vector<int> kind, index, pos;
  FO1_TRY(splice_plan(input_ids, n_ids, image_grid_hw, n_images, n_regions, *cfg, ids, kind, index, pos, rope_delta));
  const int L = (int)ids.size();
  *out_len = L;
  if (L > capacity || !new_ids || !src_kind || !src_index || !position_ids) {
    set_error("fo1_splice_plan: capacity %d < required %d", capacity, L);
    return FO1_ERR_WORKSPACE;
  }
  memcpy(new_ids, ids.data(), (size_t)L * sizeof(int64_t));
  memcpy(src_kind, kind.data(), (size_t)L * sizeof(int));
  memcpy(src_index, index.data(), (size_t)L * sizeof(int));
  for (int a = 0; a < 3; ++a) memcpy(position_ids + (size_t)a * capacity, pos.data() + (size_t)a * L, (size_t)L * sizeof(int));
  return FO1_OK;
}

extern "C" int fo1_llm_build_embeds(fo1_model* m, const int32_t* src_kind, const int32_t* src_index, int32_t n_rows,
                                    const void* img_feats, const void* region_feats, void* inputs_embeds, void* stream) {
  FO1_CHECK_ARG(m && src_kind && src_index && inputs_embeds, "fo1_llm_build_embeds: null argument");
  FO1_CHECK_ARG(m->llm.ok, "fo1_llm_build_embeds: model not finalized");
  if (n_rows <= 0) return FO1_OK;
  FO1_CHECK_ARG(m->cfg.llm_hidden % 8 == 0, "fo1_llm_build_embeds: hidden %% 8");
  build_embeds_kernel<<<n_rows, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src_kind, src_index, m->llm.embed, static_cast<const bf16*>(img_feats), static_cast<const bf16*>(region_feats),
      static_cast<bf16*>(inputs_embeds), m->cfg.llm_hidden);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

extern "C" int fo1_llm_generate(fo1_model* m, fo1_generate_desc* d, void* stream) {
  FO1_CHECK_ARG(m && d, "fo1_llm_generate: null argument");
  return llm_generate(m, d, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_llm_loglik(fo1_model* m, const fo1_loglik_desc* d, void* stream) {
  FO1_CHECK_ARG(m && d, "fo1_llm_loglik: null argument");
  return llm_loglik(m, d, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_slots_open(fo1_model* m, const fo1_slots_desc* o, void* stream) {
  FO1_CHECK_ARG(m && o, "fo1_slots_open: null argument");
  return slots_open(m, o, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_slots_admit(fo1_model* m, const fo1_slots_admit_desc* a, void* stream) {
  FO1_CHECK_ARG(m && a, "fo1_slots_admit: null argument");
  return slots_admit(m, a, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_slots_decode(fo1_model* m, int32_t exit_at, int32_t* steps_run, void* stream) {
  FO1_CHECK_ARG(m && steps_run, "fo1_slots_decode: null argument");
  return slots_decode(m, exit_at, steps_run, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_slots_close(fo1_model* m) {
  FO1_CHECK_ARG(m, "fo1_slots_close: null argument");
  FO1_CHECK_ARG(m->slot_pool != nullptr, "fo1_slots_close: no slot pool is open");
  FO1_CUDA(cudaDeviceSynchronize());
  slots_free(m);
  return FO1_OK;
}

extern "C" int32_t fo1_stream_progress(const int32_t* progress) { return __atomic_load_n(progress, __ATOMIC_ACQUIRE); }

extern "C" void fo1_stream_cancel(int32_t* cancel) { __atomic_store_n(cancel, 1, __ATOMIC_RELEASE); }

extern "C" size_t fo1_decode_attention_workspace_bytes(int32_t n_seqs, int32_t q_heads) {
  return (size_t)(n_seqs > 0 ? n_seqs : 0) * (q_heads > 0 ? q_heads : 0) * fo1::kDecSplits * (128 + 4) * sizeof(float);
}

extern "C" int fo1_decode_attention(const fo1_decode_attn_desc* d, void* stream) {
  using namespace fo1;
  FO1_CHECK_ARG(d != nullptr, "fo1_decode_attention: null descriptor");
  FO1_CHECK_ARG(d->n_seqs >= 0 && d->cap > 0, "fo1_decode_attention: bad n_seqs / cap");
  if (d->n_seqs == 0) return FO1_OK;
  FO1_CHECK_ARG(d->q && d->k_cache && d->v_cache && d->cache_len && d->out, "fo1_decode_attention: null pointer");
  FO1_CHECK_ARG(d->n_seqs <= 65535, "fo1_decode_attention: n_seqs %d exceeds the grid limit", d->n_seqs);
  FO1_CHECK_ARG((d->ldq % 2) == 0 && (d->ldo % 8) == 0 && (reinterpret_cast<uintptr_t>(d->k_cache) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->v_cache) & 15) == 0,
                "fo1_decode_attention: pitches / cache pointers misaligned");
  const size_t need = fo1_decode_attention_workspace_bytes(d->n_seqs, d->q_heads);
  if (d->workspace == nullptr || d->workspace_bytes < need) { set_error("fo1_decode_attention: workspace %zu B < required %zu B", d->workspace_bytes, need); return FO1_ERR_WORKSPACE; }
  return decode_attention(static_cast<const bf16*>(d->q), d->ldq, static_cast<const bf16*>(d->k_cache), static_cast<const bf16*>(d->v_cache), d->cache_len,
                          nullptr, d->n_seqs, d->n_seqs, d->cap, d->q_heads, d->kv_heads, d->head_dim, d->scale, static_cast<bf16*>(d->out), d->ldo,
                          static_cast<float*>(d->workspace), static_cast<cudaStream_t>(stream));
}
