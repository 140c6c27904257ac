// attention_tc.cu -- variable-length softmax attention on the Hopper tensor cores (wgmma + TMA).
//
// One kernel serves the ViT's windowed / full attention (head_dim 80; modeling_qwen2_5_vl.py:172-209, the
// flash_attn_varlen_func call at :205), DaViT's 12x12 window attention (head_dim 32; modeling_davit.py:225-282) and the
// LLM's causal GQA prefill (head_dim 128, 16 q / 2 kv heads; modeling_qwen2_5_vl.py:822-913, _flash_attention_forward
// at :895).
//
// Formulation: the packed token rows are cut into query tiles of up to 128 rows REGARDLESS of the segment boundaries; a
// row attends the keys [lo, hi) of its own segment (hi clipped to row + 1 when causal), so a tile's key range is
// [lo(first row), hi(last row)) and the per-row mask is two integer compares.  That makes 64-token ViT windows, ragged
// edge windows (46x46 grids), 144-token DaViT windows, whole images and ragged causal prompts the same code path.
// The engines pass a tile table whose tiling restarts at every image / prompt, so a sample's result does not depend on
// its position in the batch (bit-identical across batch compositions and rank counts).
//
// CTA = one (query tile, head), 288 threads:
//   warp 8   : TMA producer -- Q once, then K and V 64-key tiles through two 2-stage rings (3-D tensor maps over
//              (head_dim, head, row), 64-wide boxes, 128-byte swizzle; head_dim 80 / 32 are zero-filled to the box by
//              the TMA out-of-bounds rule, so every operand has 128-byte rows);
//   warps 0-7: two consumer warpgroups, 64 query rows each -- S_j = Q.K_j^T (wgmma m64n64k16, K-major operands) into
//              registers; softmax on the accumulator fragment (a row lives in the four lanes of a quad): mask, running
//              max / sum, P = exp2(S*scale - m) packed to bf16 in place as the A fragments of the next wgmma; O += P_j.V_j
//              with V taken MN-major straight from its TMA tile (no transposition pass).  O stays in registers for the
//              whole key loop; it is rescaled only when a row's max has grown by more than 2^8 since the last rescale
//              (stale maxima are exact: the factor cancels in O / l).  While one warpgroup is in its softmax the other
//              one's wgmma keeps the tensor cores busy.
// Warps whose 16 rows cannot see a key tile at all (the other window of the tile) skip the exponentials.
#include <cuda.h>

#include <algorithm>
#include <map>
#include <mutex>

#include "kernels.cuh"
#include "ptx.cuh"

namespace fo1 {

int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                      uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2);

constexpr int kAtM = 128;          // query rows per CTA
constexpr int kAtN = 64;           // keys per iteration
constexpr int kAtConsumers = 256;  // two warpgroups, 64 query rows each
constexpr int kAtThreads = kAtConsumers + 32;
constexpr float kAtRescale = 8.0f; // log2 units a row maximum may lag behind before O is rescaled

template <int HD>
struct AtCfg {
  static constexpr int HDP = HD <= 64 ? 64 : 128;      // head_dim as staged (zero-filled)
  static constexpr int NDB = HDP / 64;                 // 64-wide boxes per row
  static constexpr int N0 = NDB == 1 ? HD : 64;        // live dims of the first box
  static constexpr int N1 = NDB == 2 ? HD - 64 : 16;   // live dims of the second box (16 for head_dim 80; unused with one box)
  static constexpr int kQBytes = NDB * kAtM * 128;
  static constexpr int kKBytes = NDB * kAtN * 128;
  static constexpr int kVBytes = NDB * kAtN * 128;
  static constexpr int kTileBytes = kQBytes + 2 * kKBytes + 2 * kVBytes;
  // the dynamic window is at least 128-byte aligned: aligning it to 1024 costs at most 896 B; 128 B of barriers follow the tiles
  static constexpr int kSmemBytes = kTileBytes + 896 + 128;
  static_assert(HD % 16 == 0 && HD <= 128, "head_dim must be a multiple of 16, at most 128");
};

struct AttnTcArgs {
  bf16* o; long long ldo;
  const int2* rowseg;   // [T]: keys [lo, hi) of the segment every packed row belongs to
  const int2* tiles;    // optional [n_tiles] (first row, rows <= 128) of every query tile; null: tile i = rows [128 i, 128 i + 128)
  int T, q_heads, kv_heads;
  int n_work;           // query tiles x heads
  float sl2;            // softmax scale * log2(e)
};

// a wait that turns a protocol bug into a trap instead of a hung GPU
__device__ __forceinline__ void at_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t b = ptx::smem_u32(bar);
  uint32_t spins = 0;
  while (!ptx::mbar_try_wait(b, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// (lo, hi) of every packed row from cu_seqlens
__global__ void __launch_bounds__(256) attn_rowseg_kernel(const int* __restrict__ cu, int n_seqs, int T, int2* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T) return;
  int a = 0, b = n_seqs;   // largest s with cu[s] <= r
  while (b - a > 1) {
    const int mid = (a + b) >> 1;
    if (__ldg(cu + mid) <= r) a = mid; else b = mid;
  }
  const int lo = __ldg(cu + a), hi = __ldg(cu + a + 1);
  out[r] = (r >= lo && r < hi) ? make_int2(lo, hi) : make_int2(r, r + 1);   // rows outside every segment see themselves only
}

template <int HD, bool CAUSAL>
__global__ void __launch_bounds__(kAtThreads, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
               const AttnTcArgs a) {
  using Cfg = AtCfg<HD>;
  constexpr int NDB = Cfg::NDB, N0 = Cfg::N0, N1 = Cfg::N1;
  extern __shared__ uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::kQBytes;
  uint8_t* sV = sK + 2 * Cfg::kKBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * Cfg::kVBytes);
  uint64_t* q_full = bars;            // [1]
  uint64_t* k_full = bars + 1;        // [2]
  uint64_t* k_empty = bars + 3;       // [2]
  uint64_t* v_full = bars + 5;        // [2]
  uint64_t* v_empty = bars + 7;       // [2]
  uint64_t* q_empty = bars + 9;       // [1] the consumers are done with the Q tile (their output staging)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ);
    ptx::prefetch_tmap(&tmK);
    ptx::prefetch_tmap(&tmV);
    ptx::mbar_init(ptx::smem_u32(q_full), 1);
    ptx::mbar_init(ptx::smem_u32(q_empty), kAtConsumers);
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(ptx::smem_u32(k_full + s), 1);
      ptx::mbar_init(ptx::smem_u32(k_empty + s), kAtConsumers / 32);   // one arrive per consumer warp
      ptx::mbar_init(ptx::smem_u32(v_full + s), 1);
      ptx::mbar_init(ptx::smem_u32(v_empty + s), kAtConsumers / 32);
    }
    ptx::mbar_fence_init();
  }
  __syncthreads();

  // Persistent CTA: work items (query tile, head), head fastest, static round robin.  Barriers and the tensor-map prefetch are set up
  // once; every role walks the same item list and carries ONE running key-tile counter g across items (ring stage = g & 1, phase =
  // (g >> 1) & 1), so the K/V ring keeps streaming across item boundaries.  The Q tile is single-buffered: the producer reloads it
  // only after the consumers released it (q_empty).
  const int n_work = a.n_work;
  auto item_geom = [&](int work, int& head, int& kvh, int& row0, int& rows_valid, int& kv_begin, int& n_kv) {
    head = work % a.q_heads;
    const int tile = work / a.q_heads;
    kvh = head / (a.q_heads / a.kv_heads);
    row0 = tile * kAtM; rows_valid = min(kAtM, a.T - row0);
    if (a.tiles != nullptr) {
      const int2 tl = __ldg(a.tiles + tile);
      row0 = tl.x; rows_valid = tl.y;
    }
    // key range of the tile (segments are ordered, so first row's lo / last row's hi bound every row's range)
    kv_begin = __ldg(&a.rowseg[row0].x);
    int kv_end = __ldg(&a.rowseg[row0 + rows_valid - 1].y);
    if (CAUSAL) kv_end = min(kv_end, row0 + rows_valid);
    n_kv = (kv_end - kv_begin + kAtN - 1) / kAtN;
  };

  if (warp == kAtConsumers / 32) {
    // ================================================ TMA producer ================================================
    if (ptx::elect_one()) {
      uint32_t g = 0, item = 0;
      for (int work = blockIdx.x; work < n_work; work += gridDim.x, ++item) {
        int head, kvh, row0, rows_valid, kv_begin, n_kv;
        item_geom(work, head, kvh, row0, rows_valid, kv_begin, n_kv);
        if (item > 0) at_wait(q_empty, (item - 1) & 1);
        ptx::mbar_expect_tx(ptx::smem_u32(q_full), Cfg::kQBytes);
#pragma unroll
        for (int b = 0; b < NDB; ++b) ptx::tma_load_3d(ptx::smem_u32(sQ + b * kAtM * 128), &tmQ, ptx::smem_u32(q_full), b * 64, head, row0);
        for (int j = 0; j < n_kv; ++j, ++g) {
          const uint32_t st = g & 1;
          const int key0 = kv_begin + j * kAtN;
          if (g >= 2) at_wait(k_empty + st, ((g >> 1) - 1) & 1);
          ptx::mbar_expect_tx(ptx::smem_u32(k_full + st), Cfg::kKBytes);
#pragma unroll
          for (int b = 0; b < NDB; ++b)
            ptx::tma_load_3d(ptx::smem_u32(sK + st * Cfg::kKBytes + b * kAtN * 128), &tmK, ptx::smem_u32(k_full + st), b * 64, kvh, key0);
          if (g >= 2) at_wait(v_empty + st, ((g >> 1) - 1) & 1);
          ptx::mbar_expect_tx(ptx::smem_u32(v_full + st), Cfg::kVBytes);
#pragma unroll
          for (int b = 0; b < NDB; ++b)
            ptx::tma_load_3d(ptx::smem_u32(sV + st * Cfg::kVBytes + b * kAtN * 128), &tmV, ptx::smem_u32(v_full + st), b * 64, kvh, key0);
        }
      }
    }
  } else {
    // ========================================= consumers: S = Q.K^T, softmax, O += P.V =========================================
    const int wg = warp >> 2;
    const int fr = lane >> 2, fq2 = (lane & 3) * 2;
    const int r_lo = warp * 16 + fr;                    // this thread's rows inside the tile: r_lo and r_lo + 8
    const uint32_t q_addr = ptx::smem_u32(sQ) + wg * (64 * 128);
    uint32_t gbase = 0, item = 0;
    for (int work = blockIdx.x; work < n_work; work += gridDim.x, ++item) {
      int head, kvh, row0, rows_valid, kv_begin, n_kv;
      item_geom(work, head, kvh, row0, rows_valid, kv_begin, n_kv);
      int lo[2], hi[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h, row = row0 + r;
        lo[h] = 0; hi[h] = 0;                             // rows beyond the tile: empty key range
        if (r < rows_valid) {
          const int2 rs = __ldg(a.rowseg + row);
          lo[h] = rs.x; hi[h] = rs.y;
          if (CAUSAL) hi[h] = min(hi[h], row + 1);
        }
      }
      int wlo_min = min(lo[0], lo[1]), wlo_max = max(lo[0], lo[1]), whi_min = min(hi[0], hi[1]), whi_max = max(hi[0], hi[1]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        wlo_min = min(wlo_min, __shfl_xor_sync(0xffffffffu, wlo_min, o));
        wlo_max = max(wlo_max, __shfl_xor_sync(0xffffffffu, wlo_max, o));
        whi_min = min(whi_min, __shfl_xor_sync(0xffffffffu, whi_min, o));
        whi_max = max(whi_max, __shfl_xor_sync(0xffffffffu, whi_max, o));
      }
      const uint32_t span[2] = {(uint32_t)(hi[0] - lo[0]), (uint32_t)(hi[1] - lo[1])};
      float m_run[2] = {-INFINITY, -INFINITY};            // running maxima (scaled, log2 units) of the two rows
      float l_run[2] = {0.f, 0.f};                        // this thread's share of the two row sums (quad-reduced at the end)
      float o0[N0 / 2], o1[N1 / 2];
#pragma unroll
      for (int i = 0; i < N0 / 2; ++i) o0[i] = 0.f;
#pragma unroll
      for (int i = 0; i < N1 / 2; ++i) o1[i] = 0.f;

      at_wait(q_full, item & 1);
      for (int j = 0; j < n_kv; ++j) {
        const uint32_t g = gbase + j, st = g & 1;
        const int k0 = kv_begin + j * kAtN;
        const bool dead = (k0 >= whi_max) || (k0 + kAtN <= wlo_min);          // no row of this warp sees the tile
        const bool interior = (k0 >= wlo_max) && (k0 + kAtN <= whi_min);      // every row sees every key
        // ---- S_j = Q . K_j^T (64 x 64 per warpgroup, K-major operands) ----
        at_wait(k_full + st, (g >> 1) & 1);
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        const uint32_t k_addr = ptx::smem_u32(sK + st * Cfg::kKBytes);
        ptx::wgmma_fence_regs(s);
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk)
          ptx::Wgmma<64>::template ss<0, 0>(s, ptx::wgmma_desc_k_sw128(q_addr + (kk >> 2) * (kAtM * 128) + (kk & 3) * 32),
                                            ptx::wgmma_desc_k_sw128(k_addr + (kk >> 2) * (kAtN * 128) + (kk & 3) * 32), kk > 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::wgmma_fence_regs(s);
        if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(k_empty + st));
        // ---- softmax on the fragment: a row lives in the four lanes of a quad, two rows per thread ----
        uint32_t p[4][4];                                   // P as the A fragments of the four 16-key steps
        if (dead) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) { p[kk][0] = 0u; p[kk][1] = 0u; p[kk][2] = 0u; p[kk][3] = 0u; }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float mt = -INFINITY;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int idx = 4 * c8 + 2 * h + e;
                if (!interior) {
                  const bool ok = (uint32_t)(k0 + c8 * 8 + fq2 + e - lo[h]) < span[h];
                  s[idx] = ok ? s[idx] : -INFINITY;
                }
                mt = fmaxf(mt, s[idx]);
              }
            }
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
            const float m_new = fmaxf(m_run[h], mt * a.sl2);
            // lazy rescale: keep a stale maximum until it lags by 2^8 (stale maxima are exact: the factor cancels in O / l);
            // a row without any live key so far has O == 0 exactly
            if (m_new > m_run[h] + kAtRescale) {
              if (m_run[h] != -INFINITY) {
                const float alpha = ex2_approx(m_run[h] - m_new);
                l_run[h] *= alpha;
#pragma unroll
                for (int c8 = 0; c8 < N0 / 8; ++c8) { o0[4 * c8 + 2 * h] *= alpha; o0[4 * c8 + 2 * h + 1] *= alpha; }
                if constexpr (NDB == 2) {
#pragma unroll
                  for (int c8 = 0; c8 < N1 / 8; ++c8) { o1[4 * c8 + 2 * h] *= alpha; o1[4 * c8 + 2 * h + 1] *= alpha; }
                }
              }
              m_run[h] = m_new;
            }
            const float m_use = (m_run[h] == -INFINITY) ? 0.f : m_run[h];
            float sum = 0.f;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int idx = 4 * c8 + 2 * h + e;
                s[idx] = ex2_approx(fmaf(s[idx], a.sl2, -m_use));
                sum += s[idx];
              }
            }
            l_run[h] += sum;
          }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            p[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
            p[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
            p[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
            p[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
          }
        }
        // ---- O += P_j . V_j: P from registers, V MN-major straight from its TMA tile (no transposition pass) ----
        at_wait(v_full + st, (g >> 1) & 1);
        const uint32_t v_addr = ptx::smem_u32(sV + st * Cfg::kVBytes);
        ptx::wgmma_fence_regs(o0);
        ptx::wgmma_fence_regs(o1);
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kAtN / 16; ++kk) {
          ptx::Wgmma<N0>::template rs<1>(o0, p[kk], ptx::wgmma_desc_mn_sw128(v_addr + kk * 2048, kAtN * 128), 1u);
          if constexpr (NDB == 2)
            ptx::Wgmma<N1>::template rs<1>(o1, p[kk], ptx::wgmma_desc_mn_sw128(v_addr + kAtN * 128 + kk * 2048, kAtN * 128), 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::wgmma_fence_regs(o0);
        ptx::wgmma_fence_regs(o1);
        if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(v_empty + st));
      }
      gbase += (uint32_t)n_kv;

      // ---- O / l -> bf16, staged through the (dead) Q tile, row-contiguous 16-byte stores ----
      float inv[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[h] = l > 0.f ? 1.0f / l : 0.f;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");      // both warpgroups have read Q for the last time
      constexpr int PITCH = Cfg::HDP * 2;
      uint8_t* stg = sQ + warp * 16 * PITCH;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rr = fr + 8 * h;
#pragma unroll
        for (int c8 = 0; c8 < N0 / 8; ++c8)
          *reinterpret_cast<uint32_t*>(stg + rr * PITCH + (((c8 & ~7) | ((c8 ^ rr) & 7)) << 4) + (lane & 3) * 4) =
              pack_bf16(o0[4 * c8 + 2 * h] * inv[h], o0[4 * c8 + 2 * h + 1] * inv[h]);
        if constexpr (NDB == 2) {
#pragma unroll
          for (int c8 = 0; c8 < N1 / 8; ++c8) {
            const int ch = 8 + c8;
            *reinterpret_cast<uint32_t*>(stg + rr * PITCH + (((ch & ~7) | ((ch ^ rr) & 7)) << 4) + (lane & 3) * 4) =
                pack_bf16(o1[4 * c8 + 2 * h] * inv[h], o1[4 * c8 + 2 * h + 1] * inv[h]);
          }
        }
      }
      __syncwarp();
      constexpr int CH = HD / 8;
      bf16* op = a.o + (long long)(row0 + warp * 16) * a.ldo + (long long)head * HD;
      for (int i = lane; i < 16 * CH; i += 32) {
        const int rr = i / CH, ch = i - rr * CH;
        if (warp * 16 + rr < rows_valid)
          *reinterpret_cast<uint4*>(op + (long long)rr * a.ldo + ch * 8) =
              *reinterpret_cast<const uint4*>(stg + rr * PITCH + (((ch & ~7) | ((ch ^ rr) & 7)) << 4));
      }
      __syncwarp();
      ptx::fence_proxy_async_smem();                       // the next Q tile arrives through the async proxy
      ptx::mbar_arrive(ptx::smem_u32(q_empty));            // the Q tile (staging) is free for the next item
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- host
// (lo, hi) table scratch: one grow-only buffer per stream (attention calls on one stream are ordered)
static int rowseg_scratch(cudaStream_t stream, size_t rows, int2** out) {
  struct Buf { int2* p = nullptr; size_t rows = 0; };
  static std::map<cudaStream_t, Buf> pool;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  Buf& b = pool[stream];
  if (rows > b.rows) {
    FO1_CUDA(cudaStreamSynchronize(stream));
    if (b.p) FO1_CUDA(cudaFree(b.p));
    b.p = nullptr; b.rows = 0;
    const size_t want = std::max<size_t>(rows, 1 << 17);
    FO1_CUDA(cudaMalloc(reinterpret_cast<void**>(&b.p), want * sizeof(int2)));
    b.rows = want;
  }
  *out = b.p;
  return FO1_OK;
}

void attention_tile_table(const std::vector<int>& group_cu, std::vector<int>& tiles) {
  tiles.clear();
  for (size_t g = 0; g + 1 < group_cu.size(); ++g)
    for (int r = group_cu[g]; r < group_cu[g + 1]; r += kAtM) {
      tiles.push_back(r);
      tiles.push_back(std::min(kAtM, group_cu[g + 1] - r));
    }
}

int attention_rowseg(const int* cu_seqlens, int n_seqs, int T, int* rowseg /*[T][2]*/, cudaStream_t s) {
  if (T <= 0) return FO1_OK;
  attn_rowseg_kernel<<<ceil_div(T, 256), 256, 0, s>>>(cu_seqlens, n_seqs, T, reinterpret_cast<int2*>(rowseg));
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

template <int HD, bool CAUSAL>
static int launch_attn_tc(const AttnArgs& a, const int2* rowseg, cudaStream_t s) {
  using Cfg = AtCfg<HD>;
  static bool attr_set = false;
  if (!attr_set) {
    FO1_CUDA(cudaFuncSetAttribute(attn_tc_kernel<HD, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  const int T = a.total_rows;
  CUtensorMap tmQ, tmK, tmV;
  FO1_TRY(make_tmap_3d_bf16(&tmQ, a.q, HD, a.q_heads, T, (uint64_t)HD * 2, (uint64_t)a.ldq * 2, 64, 1, kAtM));
  FO1_TRY(make_tmap_3d_bf16(&tmK, a.k, HD, a.kv_heads, T, (uint64_t)HD * 2, (uint64_t)a.ldk * 2, 64, 1, kAtN));
  FO1_TRY(make_tmap_3d_bf16(&tmV, a.v, HD, a.kv_heads, T, (uint64_t)HD * 2, (uint64_t)a.ldv * 2, 64, 1, kAtN));
  AttnTcArgs g;
  g.o = a.o; g.ldo = a.ldo; g.rowseg = rowseg; g.T = T; g.q_heads = a.q_heads; g.kv_heads = a.kv_heads;
  g.tiles = reinterpret_cast<const int2*>(a.tiles);
  g.sl2 = a.scale * 1.4426950408889634f;
  const long long blocks = (long long)(a.tiles != nullptr ? a.n_tiles : ceil_div(T, kAtM)) * a.q_heads;
  FO1_CHECK_ARG(blocks < (1ll << 31), "attention: grid too large (%lld blocks)", blocks);
  g.n_work = (int)blocks;
  ProfScope prof(CAUSAL ? "attn_causal" : "attn", a.flops, 0.0, s);
  // persistent for the non-causal shapes (equal-cost items): one CTA per SM walks the item list.  Causal prompts have items of very
  // different cost, which a static round robin balances badly, so they keep one CTA per item (the same kernel with a one-item
  // list) and leave the balancing to the hardware block scheduler.  FO1_ATTN_ONE_ITEM: A/B knob.
  const long long resident = device_sm_count();
  const unsigned grid = (unsigned)((CAUSAL || getenv("FO1_ATTN_ONE_ITEM") != nullptr || blocks < resident) ? blocks : resident);
  attn_tc_kernel<HD, CAUSAL><<<grid, kAtThreads, Cfg::kSmemBytes, s>>>(tmQ, tmK, tmV, g);
  FO1_LAUNCH_CHECK();
  return FO1_OK;
}

int attention_varlen(const AttnArgs& a, cudaStream_t s) {
  FO1_CHECK_ARG(a.q && a.k && a.v && a.o && (a.cu_seqlens || a.rowseg), "attention: null pointer");
  FO1_CHECK_ARG(a.q_heads > 0 && a.kv_heads > 0 && a.q_heads % a.kv_heads == 0, "attention: heads %d/%d", a.q_heads, a.kv_heads);
  FO1_CHECK_ARG((a.ldq % 8) == 0 && (a.ldk % 8) == 0 && (a.ldv % 8) == 0 && (a.ldo % 8) == 0, "attention: pitches must be multiples of 8");
  FO1_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) |
                  reinterpret_cast<uintptr_t>(a.o)) & 15) == 0, "attention: q / k / v / o must be 16-byte aligned");
  if (a.n_seqs == 0 || a.total_rows <= 0) return FO1_OK;
  const int2* rowseg = reinterpret_cast<const int2*>(a.rowseg);
  if (rowseg == nullptr) {
    int2* scratch = nullptr;
    FO1_TRY(rowseg_scratch(s, (size_t)a.total_rows, &scratch));
    FO1_TRY(attention_rowseg(a.cu_seqlens, a.n_seqs, a.total_rows, reinterpret_cast<int*>(scratch), s));
    rowseg = scratch;
  }
  switch (a.head_dim) {
    case 32: return a.causal ? launch_attn_tc<32, true>(a, rowseg, s) : launch_attn_tc<32, false>(a, rowseg, s);
    case 64: return a.causal ? launch_attn_tc<64, true>(a, rowseg, s) : launch_attn_tc<64, false>(a, rowseg, s);
    case 80: return a.causal ? launch_attn_tc<80, true>(a, rowseg, s) : launch_attn_tc<80, false>(a, rowseg, s);
    case 128: return a.causal ? launch_attn_tc<128, true>(a, rowseg, s) : launch_attn_tc<128, false>(a, rowseg, s);
    default:
      set_error("attention: head_dim %d unsupported (32, 64, 80, 128)", a.head_dim);
      return FO1_ERR_UNSUPPORTED;
  }
}

}  // namespace fo1

extern "C" int fo1_attention_varlen(const fo1_attn_desc* d, void* stream) {
  using namespace fo1;
  FO1_CHECK_ARG(d != nullptr, "fo1_attention_varlen: null descriptor");
  FO1_CHECK_ARG(d->total_rows >= 0, "fo1_attention_varlen: total_rows %d", d->total_rows);
  AttnArgs a;
  a.q = static_cast<const bf16*>(d->q); a.k = static_cast<const bf16*>(d->k); a.v = static_cast<const bf16*>(d->v);
  a.o = static_cast<bf16*>(d->o);
  a.ldq = d->ldq; a.ldk = d->ldk; a.ldv = d->ldv; a.ldo = d->ldo;
  a.cu_seqlens = d->cu_seqlens; a.rowseg = nullptr; a.n_seqs = d->n_seqs; a.total_rows = d->total_rows; a.max_seqlen = d->max_seqlen;
  a.q_heads = d->q_heads; a.kv_heads = d->kv_heads; a.head_dim = d->head_dim;
  a.scale = d->scale; a.causal = d->causal; a.flops = 0.0;
  return attention_varlen(a, static_cast<cudaStream_t>(stream));
}
