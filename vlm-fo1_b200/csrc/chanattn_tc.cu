// chanattn_tc.cu -- DaViT channel-group attention (modeling_davit.py:151-172) as two wgmma contractions.
//
// Per image and group of 32 channels the reference computes, over the N tokens of the map,
//     A = softmax_c2( (q * N^-0.5)^T k )   [32 x 32]          out = (A v^T)^T   [N x 32]
// i.e. a Gram matrix over the TOKEN axis followed by a 32-wide mixing of v.  Both are dense contractions with almost no
// arithmetic per byte (the pass over q, k and the pass over v are what cost), so the kernels are built to stream:
//
//   chan_gram_tc_kernel  : CTA = (token chunk, 128-channel quad = 4 groups, image).  TMA brings q and k tiles of 128 tokens
//                          x 128 channels ([token][channel] rows, 128-byte swizzle) through a 3-stage ring; each of the two
//                          consumer warpgroups owns one 64-channel half (two groups) and accumulates
//                          G[c1][c2] += sum_tok q[tok][c1] k[tok][c2] for its 64 x 64 block in registers with ONE wgmma
//                          chain, both operands MN-major straight from the TMA tiles (the token axis is the contraction
//                          axis, so no transposition is needed).  Only the two 32 x 32 diagonal blocks are kept.  Partial
//                          Grams of the token chunks are written side by side and summed in a FIXED order by the consumer
//                          (no atomics: the result is bit-reproducible and independent of the batch slot).
//   chan_apply_tc_kernel : same CTA shape.  Prologue: sum the partial Grams, scale, softmax over c2 (fp32), and lay the
//                          quad's block-diagonal [128 x 128] bf16 matrix out as a K-major swizzled B operand in shared
//                          memory.  Main loop: v tiles by TMA, out[tok][c1] = sum_c2 v[tok][c2] A[c1][c2] as wgmma
//                          m64n128k16 steps (64 tokens per warpgroup), the warps convert and write 256-byte rows.
// The arithmetic waste of multiplying the off-diagonal blocks is free: the tensor pipe is far from busy at HBM speed.
#include <cuda.h>

#include <algorithm>

#include "kernels.cuh"
#include "ptx.cuh"

namespace fo1 {

int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                      uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2);

constexpr int kCaTok = 128;               // tokens per tile
constexpr int kCaQuad = 128;              // channels per CTA (4 groups of 32)
constexpr int kCaConsumers = 256;         // warps 0-7: two consumer warpgroups
constexpr int kCaThreads = kCaConsumers + 32;   // warp 8: TMA producer
constexpr int kCaStages = 3;
constexpr int kCaBoxBytes = kCaTok * 128; // one [128 tokens][64 channels] box
constexpr int kCaMaxChunks = 32;

__device__ __forceinline__ void ca_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t b = ptx::smem_u32(bar);
  uint32_t spins = 0;
  while (!ptx::mbar_try_wait(b, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

struct ChanArgs {
  int N, C, groups, n_chunks, tiles_per_chunk, B;
  float* part;          // [n_chunks][B][groups][32][32] partial Grams
  bf16* out;            // [B][N][C]
  float scale;
};

// ------------------------------------------------------------------------------------------------------ Gram
constexpr int kGramSmem = kCaStages * 4 * kCaBoxBytes + 1024 + 128;

__global__ void __launch_bounds__(kCaThreads, 1)
chan_gram_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const ChanArgs a) {
  extern __shared__ uint8_t ca_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ca_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kCaStages * 4 * kCaBoxBytes);
  uint64_t* full = bars;                 // [stages]
  uint64_t* empty = bars + kCaStages;    // [stages]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x, quad = blockIdx.y, b = blockIdx.z;
  const int tile0 = chunk * a.tiles_per_chunk;
  const int n_tiles = max(0, min(a.tiles_per_chunk, (a.N + kCaTok - 1) / kCaTok - tile0));

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ);
    ptx::prefetch_tmap(&tmK);
    for (int s = 0; s < kCaStages; ++s) { ptx::mbar_init(ptx::smem_u32(full + s), 1); ptx::mbar_init(ptx::smem_u32(empty + s), kCaConsumers / 32); }
    ptx::mbar_fence_init();
  }
  __syncthreads();

  if (warp == kCaConsumers / 32) {
    if (ptx::elect_one()) {
      for (int t = 0; t < n_tiles; ++t) {
        const int st = t % kCaStages;
        if (t >= kCaStages) ca_wait(empty + st, ((t / kCaStages) - 1) & 1);
        const uint32_t fb = ptx::smem_u32(full + st);
        uint8_t* base = smem + st * 4 * kCaBoxBytes;
        ptx::mbar_expect_tx(fb, 4 * kCaBoxBytes);
        const int tok = (tile0 + t) * kCaTok;
        ptx::tma_load_3d(ptx::smem_u32(base), &tmQ, fb, quad * kCaQuad, tok, b);
        ptx::tma_load_3d(ptx::smem_u32(base + kCaBoxBytes), &tmQ, fb, quad * kCaQuad + 64, tok, b);
        ptx::tma_load_3d(ptx::smem_u32(base + 2 * kCaBoxBytes), &tmK, fb, quad * kCaQuad, tok, b);
        ptx::tma_load_3d(ptx::smem_u32(base + 3 * kCaBoxBytes), &tmK, fb, quad * kCaQuad + 64, tok, b);
      }
    }
  } else {
    const int wg = warp >> 2;               // 64-channel half of the quad: its q box and its k box
    float acc[32];                          // G[64 x 64] fragment of this warpgroup
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int t = 0; t < n_tiles; ++t) {
      const int st = t % kCaStages;
      ca_wait(full + st, (t / kCaStages) & 1);
      const uint32_t qa = ptx::smem_u32(smem + st * 4 * kCaBoxBytes) + wg * kCaBoxBytes, ka = qa + 2 * kCaBoxBytes;
      ptx::wgmma_fence_regs(acc);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kCaTok / 16; ++kk)      // 16 tokens per step: 16 rows x 128 B = 2048 B into each box
        ptx::Wgmma<64>::template ss<1, 1>(acc, ptx::wgmma_desc_mn_sw128(qa + kk * 2048, kCaBoxBytes), ptx::wgmma_desc_mn_sw128(ka + kk * 2048, kCaBoxBytes),
                                          (t > 0 || kk > 0) ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_regs(acc);
      if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(empty + st));
    }
    // this warp's 16 rows lie in group (warp / 2) of the quad; of their 64 columns only that group's 32 are kept
    const int gsel = (warp >> 1) & 1;                 // group inside the warpgroup's half
    const int g = quad * 4 + (warp >> 1);
    const int fr = lane >> 2, fq2 = (lane & 3) * 2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = (warp & 1) * 16 + fr + 8 * h;   // row inside the group
      if (g * 32 + row >= a.C) continue;
      float* dst = a.part + ((((long long)chunk * a.B + b) * a.groups + g) * 32 + row) * 32;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const float v0 = gsel ? acc[4 * (4 + cc) + 2 * h] : acc[4 * cc + 2 * h];
        const float v1 = gsel ? acc[4 * (4 + cc) + 2 * h + 1] : acc[4 * cc + 2 * h + 1];
        *reinterpret_cast<float2*>(dst + cc * 8 + fq2) = make_float2(v0, v1);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------- apply
constexpr int kApplyB = 2 * kCaBoxBytes;                       // block-diagonal A as the B operand: two K blocks of [128][64]
constexpr int kApplyStage = 2 * kCaBoxBytes;                   // v tile: two K blocks of [128 tokens][64 channels]
constexpr int kApplyStaging = (kCaConsumers / 32) * kFragStageBytes;   // per consumer warp: 16 rows x 256 B
constexpr int kApplySmem = kApplyB + kCaStages * kApplyStage + kApplyStaging + 1024 + 128;

__global__ void __launch_bounds__(kCaThreads, 1)
chan_apply_tc_kernel(const __grid_constant__ CUtensorMap tmV, const ChanArgs a) {
  extern __shared__ uint8_t ca_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ca_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;
  uint8_t* sV = sB + kApplyB;
  uint8_t* sStg = sV + kCaStages * kApplyStage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStg + kApplyStaging);
  uint64_t* full = bars;                      // [stages]
  uint64_t* empty = bars + kCaStages;         // [stages]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x, quad = blockIdx.y, b = blockIdx.z;
  const int tile0 = chunk * a.tiles_per_chunk;
  const int n_tiles = max(0, min(a.tiles_per_chunk, (a.N + kCaTok - 1) / kCaTok - tile0));

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmV);
    for (int s = 0; s < kCaStages; ++s) { ptx::mbar_init(ptx::smem_u32(full + s), 1); ptx::mbar_init(ptx::smem_u32(empty + s), kCaConsumers / 32); }
    ptx::mbar_fence_init();
  }
  // ---- the quad's block-diagonal softmax matrix as a K-major, 128B-swizzled B operand: row c1, 128 columns c2 ----
  if (threadIdx.x < 128) {
    const int c1 = threadIdx.x, grp = c1 >> 5;
    const int g = quad * 4 + grp;
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
    if (quad * kCaQuad + c1 < a.C) {
      for (int ch = 0; ch < a.n_chunks; ++ch) {         // fixed order: bit-reproducible
        const float4* src = reinterpret_cast<const float4*>(a.part + ((((long long)ch * a.B + b) * a.groups + g) * 32 + (c1 & 31)) * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 t = __ldg(src + q);
          v[4 * q] += t.x; v[4 * q + 1] += t.y; v[4 * q + 2] += t.z; v[4 * q + 3] += t.w;
        }
      }
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < 32; ++j) { v[j] *= a.scale; m = fmaxf(m, v[j]); }
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) { v[j] = __expf(v[j] - m); sum += v[j]; }
      const float inv = 1.0f / sum;
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= inv;
    }
    // row c1: K block kb = grp / 2 holds this group's 32 columns at column offset (grp & 1) * 32; everything else is zero
#pragma unroll
    for (int kb = 0; kb < 2; ++kb) {
      uint8_t* row = sB + kb * kCaBoxBytes + c1 * 128;
#pragma unroll
      for (int ch16 = 0; ch16 < 8; ++ch16) {
        uint4 w = make_uint4(0u, 0u, 0u, 0u);
        if (kb == (grp >> 1) && (ch16 >> 2) == (grp & 1)) {
          const int j = (ch16 & 3) * 8;
          w = make_uint4(pack_bf16(v[j], v[j + 1]), pack_bf16(v[j + 2], v[j + 3]), pack_bf16(v[j + 4], v[j + 5]), pack_bf16(v[j + 6], v[j + 7]));
        }
        *reinterpret_cast<uint4*>(row + ((ch16 ^ (c1 & 7)) << 4)) = w;
      }
    }
    ptx::fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp == kCaConsumers / 32) {
    if (ptx::elect_one()) {
      for (int t = 0; t < n_tiles; ++t) {
        const int st = t % kCaStages;
        if (t >= kCaStages) ca_wait(empty + st, ((t / kCaStages) - 1) & 1);
        const uint32_t fb = ptx::smem_u32(full + st);
        uint8_t* base = sV + st * kApplyStage;
        ptx::mbar_expect_tx(fb, kApplyStage);
        const int tok = (tile0 + t) * kCaTok;
        ptx::tma_load_3d(ptx::smem_u32(base), &tmV, fb, quad * kCaQuad, tok, b);
        ptx::tma_load_3d(ptx::smem_u32(base + kCaBoxBytes), &tmV, fb, quad * kCaQuad + 64, tok, b);
      }
    }
  } else {
    const int wg = warp >> 2;                                        // tokens [64 wg, 64 wg + 64) of the tile
    const int fr = lane >> 2, fq = lane & 3;
    uint8_t* stg = sStg + warp * kFragStageBytes;
    const int cols_live = min(kCaQuad, a.C - quad * kCaQuad);        // channels of this quad that exist
    const uint32_t ba = ptx::smem_u32(sB);
    for (int t = 0; t < n_tiles; ++t) {
      const int st = t % kCaStages;
      ca_wait(full + st, (t / kCaStages) & 1);
      const uint32_t va = ptx::smem_u32(sV + st * kApplyStage) + wg * (64 * 128);
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      ptx::wgmma_fence_regs(acc);
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)                 // K = 128 channels: two 64-wide K blocks x four 16-wide steps
        ptx::Wgmma<128>::template ss<0, 0>(acc, ptx::wgmma_desc_k_sw128(va + (kk >> 2) * kCaBoxBytes + (kk & 3) * 32),
                                           ptx::wgmma_desc_k_sw128(ba + (kk >> 2) * kCaBoxBytes + (kk & 3) * 32), kk > 0 ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_regs(acc);
      if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(empty + st));     // the v tile has been read: the producer may refill the slot
#pragma unroll
      for (int c8 = 0; c8 < 16; ++c8) {
        *frag_stage_word(stg, fr, c8 * 4 + fq) = pack_bf16(acc[4 * c8], acc[4 * c8 + 1]);
        *frag_stage_word(stg, fr + 8, c8 * 4 + fq) = pack_bf16(acc[4 * c8 + 2], acc[4 * c8 + 3]);
      }
      __syncwarp();
      const int tok0 = (tile0 + t) * kCaTok + warp * 16;
      const int chunks = cols_live / 8;
      bf16* op = a.out + ((long long)b * a.N + tok0) * a.C + quad * kCaQuad;
      const int slot = lane & 15;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = 2 * it + (lane >> 4);
        if (slot < chunks && tok0 + rr < a.N)
          *reinterpret_cast<uint4*>(op + (long long)rr * a.C + slot * 8) = frag_stage_slot(stg, rr, slot);
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------------------ host
// The token chunking fixes the summation order of the Gram: it must NOT depend on the batch size, or an image's features would
// depend on how many neighbours it was batched with (tests/test_gpu_eval_drivers.py: generate_batch == one-by-one generate).
static void chan_plan(int /*B*/, int N, int C, int* n_chunks, int* tiles_per_chunk) {
  const int quads = ceil_div(C, kCaQuad), tiles = ceil_div(N, kCaTok);
  int n = ceil_div(2 * 132, std::max(1, quads));     // about two CTAs' worth of work per SM for ONE image; a batch only adds CTAs
  n = std::max(1, std::min(n, std::min(tiles, kCaMaxChunks)));
  *tiles_per_chunk = ceil_div(tiles, n);
  *n_chunks = ceil_div(tiles, *tiles_per_chunk);
}

size_t channel_attention_ws_floats(int B, int N, int C) {
  int nc = 1, tpc = 1;
  chan_plan(B, N, C, &nc, &tpc);
  return (size_t)nc * B * (C / 32) * 1024;
}

int channel_attention(const bf16* qkv, float* ws, bf16* out, int B, int N, int C, int groups, cudaStream_t s) {
  FO1_CHECK_ARG(groups * 32 == C, "channel_attention: needs 32 channels per group (C=%d groups=%d)", C, groups);
  FO1_CHECK_ARG(C % 8 == 0, "channel_attention: C=%d must be a multiple of 8", C);
  if (B == 0 || N == 0) return FO1_OK;
  static bool attr_set = false;
  if (!attr_set) {
    FO1_CUDA(cudaFuncSetAttribute(chan_gram_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGramSmem));
    FO1_CUDA(cudaFuncSetAttribute(chan_apply_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kApplySmem));
    attr_set = true;
  }
  ChanArgs a;
  a.N = N; a.C = C; a.groups = groups; a.B = B; a.part = ws; a.out = out; a.scale = 1.0f / sqrtf((float)N);
  chan_plan(B, N, C, &a.n_chunks, &a.tiles_per_chunk);
  CUtensorMap tmQ, tmK, tmV;
  const uint64_t row = (uint64_t)3 * C * 2, img = (uint64_t)N * row;
  FO1_TRY(make_tmap_3d_bf16(&tmQ, qkv, C, N, B, row, img, 64, kCaTok, 1));
  FO1_TRY(make_tmap_3d_bf16(&tmK, qkv + C, C, N, B, row, img, 64, kCaTok, 1));
  FO1_TRY(make_tmap_3d_bf16(&tmV, qkv + 2 * C, C, N, B, row, img, 64, kCaTok, 1));
  dim3 grid(a.n_chunks, ceil_div(C, kCaQuad), B);
  {
    ProfScope prof("chanattn", 4.0 * B * (double)N * C * 32, 4.0 * B * (double)N * C * 2, s);
    chan_gram_tc_kernel<<<grid, kCaThreads, kGramSmem, s>>>(tmQ, tmK, a);
    FO1_LAUNCH_CHECK();
    chan_apply_tc_kernel<<<grid, kCaThreads, kApplySmem, s>>>(tmV, a);
    FO1_LAUNCH_CHECK();
  }
  return FO1_OK;
}

}  // namespace fo1

extern "C" size_t fo1_channel_attention_workspace_bytes(int32_t n_images, int32_t n_tokens, int32_t channels) {
  if (n_images <= 0 || n_tokens <= 0 || channels <= 0) return 0;
  return fo1::channel_attention_ws_floats(n_images, n_tokens, channels) * sizeof(float);
}

extern "C" int fo1_channel_attention(const void* qkv, int32_t n_images, int32_t n_tokens, int32_t channels, int32_t groups, void* out,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  using namespace fo1;
  FO1_CHECK_ARG(qkv && out && n_images >= 0 && n_tokens >= 0 && channels > 0, "fo1_channel_attention: bad argument");
  FO1_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "fo1_channel_attention: pointers must be 16-byte aligned");
  const size_t need = fo1_channel_attention_workspace_bytes(n_images, n_tokens, channels);
  if (need > 0 && (workspace == nullptr || workspace_bytes < need)) {
    set_error("fo1_channel_attention: workspace %zu B < required %zu B", workspace_bytes, need);
    return FO1_ERR_WORKSPACE;
  }
  return channel_attention(static_cast<const bf16*>(qkv), static_cast<float*>(workspace), static_cast<bf16*>(out), n_images, n_tokens, channels,
                           groups, static_cast<cudaStream_t>(stream));
}
