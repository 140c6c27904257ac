// decode_mega.cu -- the greedy decode loop of the Qwen2.5 decoder as ONE persistent kernel (one CTA per SM, all decode steps).
//
// Why: a decode step at batch <= 32 is pure weight streaming (6.2 GB of bf16 weights + the live K/V per step, SURVEY.md section 8d);
// as 330 dependent kernel launches per step (9 per layer) it ran at a third of the HBM roofline because every launch pays
// ramp-up, drain and a dependency bubble of several microseconds for a few microseconds of streaming.  Here the whole step
// -- and the whole greedy loop (modeling_qwen2_5_vl.py:1126-1242, 1848-1876; HF generate's greedy search; KeywordsStoppingCriteria
// mm_utils.py:137-181) -- is one cooperative launch: the CTAs walk the same phase list, separated by grid barriers, and each
// warp keeps a private cp.async ring of weight chunks that is refilled ACROSS tile and phase boundaries (weights depend on
// nothing, so the next phase's first chunks are already in flight while the barrier is crossed).
//
// Per layer (5 barriers):   x -> [qkv] -> [attention + combine] -> [o-proj + residual] -> [gate/up + SiLU*up] -> [down + residual]
//   * every matrix phase is out[b, n] = epi(sum_k A[b, k] W[n, k]) with b < 32 rows: a CTA owns 16-column tiles of N (static
//     round robin), its 8 warps split K (64-wide chunks, chunk c to warp c mod 8), multiply with mma.sync m16n8k16 out of the
//     ring (W) and a shared-memory copy of A (bulk-copied once per phase; streamed in 1024-wide halves for K = 11008), and
//     reduce their partial sums through shared memory in a fixed order.  HBM-bound byte streaming: the tensor path only has to
//     keep up with 64 FLOP per weight byte pair (SURVEY: "do not reshape to reach the tensor cores" -- M is the batch).
//   * RMSNorm is folded: W' = W diag(g) is prepared once (weights.py), the row factor rsqrt(mean(x^2) + eps) multiplies the
//     accumulator in the epilogue.  The row sums of squares of the residual stream are produced by the phase that writes it
//     (per-CTA partial slots, summed by every consumer in the same fixed order -> bit-reproducible).
//   * attention: items (sequence, kv head, key split); M-RoPE of q and of the new k, the cache append and the split-KV
//     flash-decoding tile loop (the 8 query heads of a GQA group are the rows of the m16 tile) run in one phase; the last
//     split to finish merges the partials of its (sequence, kv head).
//   * the LM head streams the (norm-folded) vocabulary matrix, every CTA keeps the running arg-max of its columns, CTA 0 merges
//     them, records the token, tests the stop ids and advances the loop state; the next step starts after one more barrier.
#include <cooperative_groups.h>

#include <algorithm>

#include "decode_mega.cuh"

namespace fo1 {

constexpr int kMgThreads = 256;
constexpr int kMgWarps = 8;
constexpr int kMgRows = 32;                 // batch rows at most (MT = 1: 16, MT = 2: 32 -- one or two m16 tiles)
constexpr int kMgTileN = 16;                // output columns per tile
constexpr int kMgChunkK = 64;               // k per ring stage
constexpr int kMgWBytes = kMgTileN * kMgChunkK * 2;                // 2 KB of weights per stage
constexpr int kMgAK = 2048;                 // widest A kept resident in shared memory; wider A (down-proj) travels in the ring stages
constexpr int kMgAPitch = kMgAK * 2 + 16;   // bytes per resident A row (+16: ldmatrix rows fall on different banks)
constexpr int kMgSmemBytes = 232448 - 1024; // the 227 KB a CTA may opt into minus the kernel's few static words; laid out per MT below
constexpr int kMgMiscBytes = 1024;          // rs[32], ssq[32], mbarriers
constexpr int kMgAttnWarps = 8, kMgAttnStages = 3, kMgAttnTileBytes = 16 * 256 * 2;
// split merge: staging area behind the warp-merge buffers ([8 warps][8 heads][128] floats + m, l), 16-byte loads per thread
constexpr int kMgCombineOff = 40960, kMgCombineLoads = (8 * kMgMaxSplits * 33 + kMgThreads - 1) / kMgThreads;

// shared-memory layout: [ weight ring | resident A | per-warp partial tiles | misc ].  With 16 batch rows the A tile is half as
// large and the ring twice as deep: the ring depth (bytes in flight per SM) is what bounds the streaming rate.
template <int MT>
struct MgLay {
  static constexpr int kMisc = kMgSmemBytes - kMgMiscBytes;
  static constexpr int kRedBytes = kMgWarps * 16 * MT * kMgTileN * 4;
  static constexpr int kRed = kMisc - kRedBytes;
  static constexpr int kABytes = 16 * MT * kMgAPitch;
  static constexpr int kA = kRed - kABytes;                               // ring region of the resident-A phases: [0, kA)
  static constexpr int kStagesRes = kA / (kMgWarps * kMgWBytes);          // MT 1: 9, MT 2: 5
  static constexpr int kSelfStage = kMgWBytes + 16 * MT * 128;            // down-proj: the stage carries its A chunk too
  static constexpr int kStagesSelf = kRed / (kMgWarps * kSelfStage);      // MT 1: 6, MT 2: 4 (the A tile is not live in that phase)
  static_assert(kStagesRes >= 3 && kStagesSelf >= 3 && kStagesRes <= 9, "ring depth");
  static_assert(kMgAttnWarps * kMgAttnStages * kMgAttnTileBytes <= kMisc, "the attention ring aliases ring + A + partials");
};

// ------------------------------------------------------------------------------------------------ small device helpers
__device__ __forceinline__ void mg_cp16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void mg_cp16z(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void mg_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void mg_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void mg_ldsm(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mg_ldsm_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mg_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mg_mma_half(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {   // rows 8..15 of A are zero
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%5}, {%7,%8}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(0u), "r"(a2), "r"(b0), "r"(b1));
}
__device__ __forceinline__ unsigned mg_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long mg_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// optional phase profile (FO1_MEGA_PROF=1): every CTA stamps the nanosecond timer when it ENTERS a barrier and when it LEAVES it,
// for the first decode iteration: prof[(cta * slots + slot) * 2 + {0, 1}]
#define MG_STAMP(slot, which) do { if (a.prof != nullptr && it == 0 && threadIdx.x == 0) a.prof[((long long)blockIdx.x * a.prof_slots + (slot)) * 2 + (which)] = mg_now(); } while (0)

// grid-wide barrier: monotonically increasing arrival counter (zeroed by the host), generation g completes at g * gridDim.x.
// Thread 0 brackets the arrive / spin with __threadfence() (MEMBAR.SC.GPU), the cooperative-groups pattern.  A variant relying on
// red.release / ld.acquire alone is lighter; the conservative form is kept until the lighter one has been soaked.
__device__ __forceinline__ void mg_grid_sync(unsigned* bar, unsigned& gen) {
  __syncthreads();
  gen += 1;
  if (threadIdx.x == 0) {
    __threadfence();
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");     // arrive (no return value to wait for)
    const unsigned target = gen * gridDim.x;
    unsigned spins = 0;
    while (mg_ld_acquire(bar) < target) {
      if (++spins > (1u << 28)) __trap();    // a protocol bug must not hang the GPU
    }
    __threadfence();
  }
  __syncthreads();
}
// bulk copy of one contiguous row global -> shared, completion on an mbarrier
__device__ __forceinline__ void mg_bulk_row(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mg_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0, spins = 0;
  while (!ok) {
    asm volatile("{\n.reg .pred P;\nmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\nselp.u32 %0, 1, 0, P;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (!ok && ++spins > (1u << 26)) __trap();
  }
}

// ---------------------------------------------------------------------------------------------------- weight ring
// One warp's view of a matrix phase: the (tile, chunk) pairs it multiplies, in order.  The ring is issued from this
// iterator and consumed in the same order; `issue` may run ahead into the NEXT phase's list before the barrier.
struct MgWork {
  const bf16* W; int K, n_tiles, chunks;      // chunks = K / 64
  int tile, kc;                               // next (tile, chunk) to ISSUE for this warp
  const bf16* A; int lda, B, a_rows;          // self-contained stages (down-proj): the activation matrix the chunk slices come from
  __device__ void begin(const bf16* w, int k, int n, int warp, const bf16* a = nullptr, int lda_ = 0, int b = 0, int rows = 0) {
    W = w; K = k; n_tiles = n / kMgTileN; chunks = k / kMgChunkK; tile = blockIdx.x; kc = warp;
    A = a; lda = lda_; B = b; a_rows = rows;
    if (kc >= chunks) { tile = n_tiles; }      // (never: chunks >= 8)
  }
  __device__ bool done() const { return tile >= n_tiles; }
  __device__ void advance() {
    kc += kMgWarps;
    if (kc >= chunks) { kc = (threadIdx.x >> 5); tile += gridDim.x; }
  }
};

// Per-warp cp.async ring.  (A ring of cp.async.bulk copies from a tile-contiguous weight image was tried too: faster in an empty
// streaming loop (scripts/probes/stream_probe.cu) but slower here, because expect_tx + the bulk issue + the
// mbarrier wait cost this latency-bound loop ~500 cycles more per 2-4 KB stage than four cp.async per lane and a wait_group.)
// Also measured and rejected: the A fragments of the K <= 2048 phases kept in registers to free the 128 KB activation tile for the ring
// (spills at the 255-register cap, step time doubled).
struct MgRing {
  uint32_t base;            // shared address of this warp's stages
  int stage_bytes, n_stages;
  int head, tail;           // stages issued / consumed
  int inflight;
  // (re)configure: only when nothing is in flight.  `self`: the stage also carries the A chunk (rows x 128 B after the 2 KB of W)
  __device__ void mode(uint32_t smem0, int warp, int stage_b, int stages) {
    stage_bytes = stage_b; n_stages = stages; base = smem0 + warp * stages * stage_b; head = tail = 0; inflight = 0;
  }
  // one stage = 16 weight rows x 64 k (128 B per row, 16-byte chunks XOR-swizzled by row): 4 x 16 B per lane
  __device__ void issue(MgWork& w, int lane) {
    const uint32_t st = base + (head % n_stages) * stage_bytes;
    const bf16* src = w.W + ((long long)w.tile * kMgTileN) * w.K + (long long)w.kc * kMgChunkK;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = i * 4 + (lane >> 3), c16 = lane & 7;
      mg_cp16(st + row * 128 + ((c16 ^ (row & 7)) << 4), src + (long long)row * w.K + c16 * 8);
    }
    if (w.A != nullptr) {     // self-contained stage: this chunk's slice of A (rows beyond the batch read as zero)
      const bf16* asrc = w.A + (long long)w.kc * kMgChunkK;
      for (int i = lane; i < w.a_rows * 8; i += 32) {
        const int row = i >> 3, c16 = i & 7;
        mg_cp16z(st + kMgWBytes + row * 128 + ((c16 ^ (row & 7)) << 4), asrc + (long long)(row < w.B ? row : 0) * w.lda + c16 * 8, row < w.B);
      }
    }
    mg_commit();
    ++head; ++inflight;
    w.advance();
  }
  __device__ void fill(MgWork& w, int lane) {
    while (inflight < n_stages - 1 && !w.done()) issue(w, lane);
  }
  // wait until the OLDEST group in flight has landed (at most inflight - 1 newer groups may stay pending)
  __device__ void wait_oldest() {
    switch (inflight - 1) {
      case 0: mg_wait<0>(); break; case 1: mg_wait<1>(); break; case 2: mg_wait<2>(); break; case 3: mg_wait<3>(); break;
      case 4: mg_wait<4>(); break; case 5: mg_wait<5>(); break; case 6: mg_wait<6>(); break; default: mg_wait<7>(); break;
    }
  }
};

// -------------------------------------------------------------------------------------------------------- epilogues
enum { MG_EPI_QKV = 0, MG_EPI_RESID = 1, MG_EPI_GATEUP = 2, MG_EPI_HEAD = 3, MG_EPI_LOGITS = 4 };

struct MgEpi {
  bf16* out; int ldo;                 // QKV / RESID / GATEUP
  const bf16* bias;                   // QKV
  const bf16* resid;                  // RESID (same pitch as out)
  float* ssq_slot;                    // RESID: this CTA's [32] slot of partial row sums of squares (nullptr: none)
  bool scale_rows;                    // multiply by rs[row] (folded RMSNorm)
};

// SELF = false: A [B][K <= 2048] is bulk-copied once per phase into the resident tile and shared by the 8 warps.
// SELF = true (down-proj, K = 11008): every ring stage carries its own [rows][64] slice of A next to the 16 x 64 weight chunk, so a
// warp never waits for anybody else inside the phase.
template <int EPI, int MT, bool SELF>
__device__ __forceinline__ void mg_gemm_phase(const MegaArgs& a, uint8_t* smem, const bf16* A, int lda, int K, int N, MgWork& work, MgRing& ring,
                                             const MgEpi& e, uint32_t& a_parity, float* best_val, int* best_idx) {
  using Lay = MgLay<MT>;
  constexpr int ROWS = 16 * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* sA = smem + Lay::kA;
  float* sRed = reinterpret_cast<float*>(smem + Lay::kRed);
  float* sRs = reinterpret_cast<float*>(smem + Lay::kMisc);      // [32]
  float* sSsq = sRs + 32;                                        // [32]
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(sSsq + 32);
  const int n_tiles = N / kMgTileN, chunks = K / kMgChunkK;
  const bool has_work = (int)blockIdx.x < n_tiles;
  if (threadIdx.x < 32) sSsq[threadIdx.x] = 0.f;
  if (!SELF && has_work && threadIdx.x == 0) {
    asm volatile("fence.proxy.async;" ::: "memory");      // rows were written with ordinary stores by other CTAs (ordered by the grid barrier)
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar0), "r"((uint32_t)(a.B * K * 2)) : "memory");
    for (int r = 0; r < a.B; ++r)
      mg_bulk_row((uint32_t)__cvta_generic_to_shared(sA + r * kMgAPitch), A + (long long)r * lda, K * 2, bar0);
  }
  __syncthreads();
  if (!SELF && has_work) {
    mg_mbar_wait(bar0, a_parity);
    a_parity ^= 1;
  }
  const uint32_t a_base = (uint32_t)__cvta_generic_to_shared(sA);

  float acc[MT][2][4];
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int n = 0; n < 2; ++n) acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.f;
    for (int kc = warp; kc < chunks; kc += kMgWarps) {
      ring.fill(work, lane);
      ring.wait_oldest();
      __syncwarp();
      const uint32_t st = ring.base + (ring.tail % ring.n_stages) * ring.stage_bytes;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t af[MT][4], bf[4];
        const int jm = lane >> 3, r = lane & 7;
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const int row = m * 16 + (jm & 1) * 8 + r;
          if (SELF) mg_ldsm(af[m], st + kMgWBytes + row * 128 + (((ks * 2 + (jm >> 1)) ^ (row & 7)) << 4));
          else mg_ldsm(af[m], a_base + row * kMgAPitch + (kc * kMgChunkK + ks * 16 + (jm >> 1) * 8) * 2);
        }
        const int nrow = (jm >> 1) * 8 + r, c16 = ks * 2 + (jm & 1);
        mg_ldsm(bf, st + nrow * 128 + ((c16 ^ (nrow & 7)) << 4));
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          mg_mma(acc[m][0], af[m], bf[0], bf[1]);
          mg_mma(acc[m][1], af[m], bf[2], bf[3]);
        }
      }
      __syncwarp();
      ++ring.tail; --ring.inflight;
    }
    // ---- cross-warp reduction (fixed order) + epilogue ----
    {
      const int g = lane >> 2, t = lane & 3;
      float* mine = sRed + warp * (ROWS * kMgTileN);
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < 2; ++n) {
          *reinterpret_cast<float2*>(mine + (m * 16 + g) * kMgTileN + n * 8 + 2 * t) = make_float2(acc[m][n][0], acc[m][n][1]);
          *reinterpret_cast<float2*>(mine + (m * 16 + g + 8) * kMgTileN + n * 8 + 2 * t) = make_float2(acc[m][n][2], acc[m][n][3]);
        }
    }
    __syncthreads();
    if ((int)threadIdx.x < ROWS * 8) {
      constexpr int WS = ROWS * kMgTileN;                          // floats per warp partial
      const int row = threadIdx.x >> 3, q = threadIdx.x & 7;      // ROWS rows x 8 threads
      const int n0 = tile * kMgTileN;
      if (EPI == MG_EPI_GATEUP) {
        // tile rows = [8 gate | 8 up]: thread -> output column q
        float gsum = 0.f, usum = 0.f;
#pragma unroll
        for (int w = 0; w < kMgWarps; ++w) { gsum += sRed[w * WS + row * 16 + q]; usum += sRed[w * WS + row * 16 + 8 + q]; }
        if (row < a.B) {
          const float rs = sRs[row];
          e.out[(long long)row * e.ldo + tile * 8 + q] = __float2bfloat16_rn(silu(gsum * rs) * (usum * rs));
        }
      } else {
        float v0 = 0.f, v1 = 0.f;
#pragma unroll
        for (int w = 0; w < kMgWarps; ++w) { v0 += sRed[w * WS + row * 16 + 2 * q]; v1 += sRed[w * WS + row * 16 + 2 * q + 1]; }
        const int c = n0 + 2 * q;
        if (EPI == MG_EPI_QKV) {
          if (row < a.B) {
            const float rs = sRs[row];
            const float y0 = v0 * rs + __bfloat162float(e.bias[c]), y1 = v1 * rs + __bfloat162float(e.bias[c + 1]);
            *reinterpret_cast<uint32_t*>(e.out + (long long)row * e.ldo + c) = pack_bf16(y0, y1);
          }
        } else if (EPI == MG_EPI_RESID) {
          float sq = 0.f;
          if (row < a.B) {
            const uint32_t rr = *reinterpret_cast<const uint32_t*>(e.resid + (long long)row * e.ldo + c);
            const uint32_t o = pack_bf16(v0 + bf16_lo(rr), v1 + bf16_hi(rr));
            *reinterpret_cast<uint32_t*>(e.out + (long long)row * e.ldo + c) = o;
            sq = bf16_lo(o) * bf16_lo(o) + bf16_hi(o) * bf16_hi(o);          // of the values as stored
          }
          sq += __shfl_xor_sync(0xffffffffu, sq, 1);
          sq += __shfl_xor_sync(0xffffffffu, sq, 2);
          sq += __shfl_xor_sync(0xffffffffu, sq, 4);
          if (q == 0) sSsq[row] += sq;                                        // one writer per row, tiles in order
        } else if (EPI == MG_EPI_HEAD) {   // running arg-max of this thread's two columns (lowest index wins ties)
          if (row < a.B) {
            const float rs = sRs[row];
            const float y0 = v0 * rs, y1 = v1 * rs;
            if (y0 > *best_val) { *best_val = y0; *best_idx = c; }
            if (y1 > *best_val) { *best_val = y1; *best_idx = c + 1; }
          }
        } else {   // MG_EPI_LOGITS: the same fp32 values, stored for the sampler
          if (row < a.B) {
            const float rs = sRs[row];
            *reinterpret_cast<float2*>(a.logits + (long long)row * a.V + c) = make_float2(v0 * rs, v1 * rs);
          }
        }
      }
    }
    __syncthreads();
  }
  if (EPI == MG_EPI_RESID && e.ssq_slot != nullptr) {
    __syncthreads();
    if (threadIdx.x < 32) e.ssq_slot[threadIdx.x] = sSsq[threadIdx.x];
  }
}

// rs[row] = rsqrt(mean(x^2) + eps) from the per-CTA partial slots, identical in every CTA (fixed summation order)
__device__ __forceinline__ void mg_row_scale(const MegaArgs& a, uint8_t* smem, const float* slots) {
  float* sRs = reinterpret_cast<float*>(smem + kMgSmemBytes - kMgMiscBytes);
  const int row = threadIdx.x >> 3, q = threadIdx.x & 7;
  float s = 0.f;
  for (int c = q; c < (int)gridDim.x; c += 8) s += slots[c * 32 + row];
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (q == 0) sRs[row] = rsqrtf(s / (float)a.H + a.eps);
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------------ attention
// item = (sequence b, kv head, key split): M-RoPE of q (and, in the last split, of the new k + cache append), then the
// split-KV tile loop of llm.cu::decode_attn_kernel with 8 warps; the last split of a (b, kv head) to arrive merges.
__device__ __forceinline__ void mg_attention_phase(const MegaArgs& a, uint8_t* smem, int layer, int it) {
#define MG_ASTAMP(k) do { if (a.prof != nullptr && it == 0 && layer == 1 && threadIdx.x == 0 && item == (int)blockIdx.x && (int)blockIdx.x == a.n_splits - 1) a.prof[((long long)0 * a.prof_slots + a.prof_slots - 8 + (k)) * 2] = mg_now(); } while (0)
  constexpr int HD = 128;
  const int G = a.q_heads / a.kv_heads;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ldq = a.QD + 2 * a.KD;
  bf16* kc = a.kc + (long long)layer * a.kv_layer_stride;
  bf16* vc = a.vc + (long long)layer * a.kv_layer_stride;
  const int n_items = a.B * a.kv_heads * a.n_splits;
  __shared__ int s_last;
  const float sc = rsqrtf((float)HD) * 1.4426950408889634f;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int sp = item % a.n_splits, kvh = (item / a.n_splits) % a.kv_heads, b = item / (a.n_splits * a.kv_heads);
    MG_ASTAMP(0);
    const int n = a.sink.st.cache_len[b] + 1;
    const int chunk = ((n + a.n_splits - 1) / a.n_splits + 15) & ~15;
    const int t_begin = sp * chunk, t_end = min(n, t_begin + chunk);
    const float* cosv = a.cs + (long long)b * (HD / 2);
    const float* sinv = a.cs + (long long)a.B * (HD / 2) + (long long)b * (HD / 2);
    // ---- the split that owns key n-1 rotates the new k and appends k, v to the cache (before it streams its keys) ----
    if (t_begin < n && n - 1 < t_begin + chunk && n - 1 >= t_begin) {
      const bf16* krow = a.qkv + (long long)b * ldq + a.QD + kvh * HD;
      const bf16* vrow = krow + a.KD;
      bf16* kdst = kc + ((long long)b * a.cap + (n - 1)) * a.KD + kvh * HD;
      bf16* vdst = vc + ((long long)b * a.cap + (n - 1)) * a.KD + kvh * HD;
      if (threadIdx.x < HD / 2) {
        const int d = threadIdx.x;
        const float x1 = __bfloat162float(krow[d]), x2 = __bfloat162float(krow[d + HD / 2]);
        const float co = cosv[d], si = sinv[d];
        kdst[d] = __float2bfloat16_rn(x1 * co - x2 * si);
        kdst[d + HD / 2] = __float2bfloat16_rn(x2 * co + x1 * si);
      } else if (threadIdx.x < HD / 2 + HD / 8) {
        const int c = threadIdx.x - HD / 2;
        reinterpret_cast<uint4*>(vdst)[c] = reinterpret_cast<const uint4*>(vrow)[c];
      }
      // the row is read back by THIS CTA's L1-bypassing cp.async right after the bar.sync: every writer fences its own posted stores
      __threadfence();
    }
    __syncthreads();
    MG_ASTAMP(1);
    float m = -INFINITY, l = 0.f, o[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
    const uint32_t ring = (uint32_t)__cvta_generic_to_shared(smem) + w * kMgAttnStages * kMgAttnTileBytes;
    const int cp_key = lane >> 4, cp_chunk = lane & 15;
    const bf16* kbase = kc + (long long)b * a.cap * a.KD + kvh * HD + cp_chunk * 8;
    const bf16* vbase = vc + (long long)b * a.cap * a.KD + kvh * HD + cp_chunk * 8;
    int t_issue = t_begin + w * 16;
    uint32_t st_issue = 0, st_done = 0;
    auto issue_tile = [&]() {
      if (t_issue < t_end) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int key = 2 * i + cp_key, tok = t_issue + key;
          const bool ok = tok < t_end;
          const long long off = (long long)(ok ? tok : t_begin) * a.KD;
          const uint32_t dst = ring + st_issue + key * 256 + ((cp_chunk ^ (key & 7)) << 4);
          mg_cp16z(dst, kbase + off, ok);
          mg_cp16z(dst + 16 * 256, vbase + off, ok);
        }
        t_issue += kMgAttnWarps * 16;
        st_issue = (st_issue == (kMgAttnStages - 1) * kMgAttnTileBytes) ? 0u : st_issue + kMgAttnTileBytes;
      }
      mg_commit();
    };
    issue_tile();
    issue_tile();
    // (the first key tiles are in flight while q is fetched and rotated)
    // ---- Q fragments of the group's heads (rows g < G), rotated: dims d and d + 64 sit in qa[ks] / qa[ks + 4] of the same lane ----
    uint32_t qa[8][2];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) { qa[ks][0] = 0u; qa[ks][1] = 0u; }
    if (g < G) {
      const bf16* qp = a.qkv + (long long)b * ldq + (long long)(kvh * G + g) * HD + 2 * t;
      uint32_t raw[8][2];
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        raw[ks][0] = *reinterpret_cast<const uint32_t*>(qp + ks * 16);
        raw[ks][1] = *reinterpret_cast<const uint32_t*>(qp + ks * 16 + 8);
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int d = ks * 16 + hh * 8 + 2 * t;          // < 64
          const float c0 = cosv[d], c1 = cosv[d + 1], s0 = sinv[d], s1 = sinv[d + 1];
          const float x1l = bf16_lo(raw[ks][hh]), x1h = bf16_hi(raw[ks][hh]), x2l = bf16_lo(raw[ks + 4][hh]), x2h = bf16_hi(raw[ks + 4][hh]);
          qa[ks][hh] = pack_bf16(x1l * c0 - x2l * s0, x1h * c1 - x2h * s1);
          qa[ks + 4][hh] = pack_bf16(x2l * c0 + x1l * s0, x2h * c1 + x1h * s1);
        }
    }
    MG_ASTAMP(2);
    const int lr = lane & 7, lm = lane >> 3;
    for (int t0 = t_begin + w * 16; t0 < t_end; t0 += kMgAttnWarps * 16) {
      issue_tile();
      mg_wait<2>();
      __syncwarp();
      const uint32_t kt = ring + st_done, vt = kt + 16 * 256;
      float s[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        uint32_t bk[4];
        const int key = (lm >> 1) * 8 + lr;
        mg_ldsm(bk, kt + key * 256 + (((2 * ks + (lm & 1)) ^ (key & 7)) << 4));
        mg_mma_half(s[0], qa[ks][0], qa[ks][1], bk[0], bk[1]);
        mg_mma_half(s[1], qa[ks][0], qa[ks][1], bk[2], bk[3]);
      }
      float tmax = -INFINITY;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int ee = 0; ee < 2; ++ee) {
          s[i][ee] = (t0 + i * 8 + 2 * t + ee < t_end) ? s[i][ee] * sc : -INFINITY;
          tmax = fmaxf(tmax, s[i][ee]);
        }
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
      const float mn = fmaxf(m, tmax);
      const float alpha = exp2f(m - mn);
      const float p00 = exp2f(s[0][0] - mn), p01 = exp2f(s[0][1] - mn), p10 = exp2f(s[1][0] - mn), p11 = exp2f(s[1][1] - mn);
      l = l * alpha + (p00 + p01) + (p10 + p11);
      m = mn;
      const uint32_t pa0 = pack_bf16(p00, p01), pa2 = pack_bf16(p10, p11);
#pragma unroll
      for (int c = 0; c < 16; c += 2) {
        uint32_t bv[4];
        const int key = (lm & 1) * 8 + lr;
        mg_ldsm_t(bv, vt + key * 256 + (((c + (lm >> 1)) ^ (key & 7)) << 4));
        o[c][0] *= alpha; o[c][1] *= alpha; o[c + 1][0] *= alpha; o[c + 1][1] *= alpha;
        mg_mma_half(o[c], pa0, pa2, bv[0], bv[1]);
        mg_mma_half(o[c + 1], pa0, pa2, bv[2], bv[3]);
      }
      __syncwarp();
      st_done = (st_done == (kMgAttnStages - 1) * kMgAttnTileBytes) ? 0u : st_done + kMgAttnTileBytes;
    }
    mg_wait<0>();
    MG_ASTAMP(3);
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    __syncthreads();
    MG_ASTAMP(4);
    float* sm_o = reinterpret_cast<float*>(smem);              // [warps][8][HD]
    float* sm_m = sm_o + kMgAttnWarps * 8 * HD;
    float* sm_l = sm_m + kMgAttnWarps * 8;
    if (t == 0) { sm_m[w * 8 + g] = m; sm_l[w * 8 + g] = l; }
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<float2*>(&sm_o[(w * 8 + g) * HD + j * 8 + 2 * t]) = make_float2(o[j][0], o[j][1]);
    __syncthreads();
    // merge the 8 warps: thread -> (head r = tid / 32, dims 4 * (tid % 32) ..), warps in index order
    {
      const int r = threadIdx.x >> 5, d4 = (threadIdx.x & 31) * 4;
      if (r < G) {
        float mm = -INFINITY;
#pragma unroll
        for (int ww = 0; ww < kMgAttnWarps; ++ww) mm = fmaxf(mm, sm_m[ww * 8 + r]);
        float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
        float den = 0.f;
#pragma unroll
        for (int ww = 0; ww < kMgAttnWarps; ++ww) {
          const float f = (sm_m[ww * 8 + r] == -INFINITY) ? 0.f : exp2f(sm_m[ww * 8 + r] - mm);
          const float4 v = *reinterpret_cast<const float4*>(&sm_o[(ww * 8 + r) * HD + d4]);
          num.x += v.x * f; num.y += v.y * f; num.z += v.z * f; num.w += v.w * f;
          den += sm_l[ww * 8 + r] * f;
        }
        float* rec = a.att_part + (((long long)b * a.q_heads + kvh * G + r) * kMgMaxSplits + sp) * (HD + 4);
        if (d4 == 0) { rec[0] = mm; rec[1] = den; }
        *reinterpret_cast<float4*>(rec + 4 + d4) = num;
      }
    }
    // ---- last split of this (b, kv head) to arrive merges the splits in index order ----
    MG_ASTAMP(5);
    __threadfence();                                           // every writer publishes its part of the record before the count
    __syncthreads();
    MG_ASTAMP(6);
    if (threadIdx.x == 0) {
      const int prev = atomicAdd(a.att_count + b * a.kv_heads + kvh, 1);
      s_last = (prev == a.n_splits - 1) ? 1 : 0;
      if (s_last) a.att_count[b * a.kv_heads + kvh] = 0;       // self-cleaning for the next layer
    }
    __syncthreads();
    if (s_last) {
      __threadfence();
      // stage the G x n_splits records in shared memory with independent 16-byte loads (one L2 round trip instead of a
      // dependent chain per head), then merge from there in split order
      constexpr int kRecF4 = (HD + 4) / 4;
      float* st = reinterpret_cast<float*>(smem + kMgCombineOff);
      const int total = G * a.n_splits * kRecF4;
      float4 v[kMgCombineLoads];
#pragma unroll
      for (int k = 0; k < kMgCombineLoads; ++k) {
        const int i = threadIdx.x + k * kMgThreads;
        if (i < total) {
          const int rc = i / kRecF4, c = i - rc * kRecF4;
          const int r = rc / a.n_splits, s2 = rc - r * a.n_splits;
          v[k] = __ldcg(reinterpret_cast<const float4*>(a.att_part + (((long long)b * a.q_heads + kvh * G + r) * kMgMaxSplits + s2) * (HD + 4)) + c);
        }
      }
#pragma unroll
      for (int k = 0; k < kMgCombineLoads; ++k) {
        const int i = threadIdx.x + k * kMgThreads;
        if (i < total) reinterpret_cast<float4*>(st)[i] = v[k];
      }
      __syncthreads();                                           // (s_last is uniform over the block)
      const int r = threadIdx.x >> 5, d4 = (threadIdx.x & 31) * 4;
      if (r < G) {
        const float* rec = st + (long long)r * a.n_splits * (HD + 4);
        float mm = -INFINITY;
        for (int s2 = 0; s2 < a.n_splits; ++s2) mm = fmaxf(mm, rec[s2 * (HD + 4)]);
        float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
        float den = 0.f;
        for (int s2 = 0; s2 < a.n_splits; ++s2) {
          const float ms = rec[s2 * (HD + 4)];
          const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
          const float4 v = *reinterpret_cast<const float4*>(rec + s2 * (HD + 4) + 4 + d4);
          num.x += v.x * f; num.y += v.y * f; num.z += v.z * f; num.w += v.w * f;
          den += rec[s2 * (HD + 4) + 1] * f;
        }
        uint2 o2;
        o2.x = pack_bf16(num.x / den, num.y / den);
        o2.y = pack_bf16(num.z / den, num.w / den);
        *reinterpret_cast<uint2*>(a.att + (long long)b * a.QD + (long long)(kvh * G + r) * HD + d4) = o2;
      }
    }
    __syncthreads();
    MG_ASTAMP(7);
  }
}

// ----------------------------------------------------------------------------------------------------------- kernel
// MODE (DecodeMode) DEC_GREEDY: the greedy loop.  DEC_SAMPLED: the head stores its logits, CTA b < B draws sequence b's token with
// the row routine of sampling.cuh (one more grid barrier per step), CTA 0 records the drawn tokens.  DEC_SCORED: CTA b also scores
// row b in the same phase -- one more pass over the row for Z_kept, the log-probability and the optional scores / logits rows (a
// scored greedy call runs here with top_k = 1, which draws the arg-max).  PROC (logits processors, a.proc): CTA b first edits row b
// (processors.cuh), in both modes; a greedy call with processors runs DEC_SAMPLED with top_k = 1.  PROC is a template parameter so
// that the calls without processors keep the registers and spills of the plain instantiations.  STREAM: CTA 0 also mirrors each recorded column into the
// caller's mapped host buffers and publishes it (a.sink.stream), and honours the host's cancel flag.
template <int MT, int MODE, bool STREAM, bool PROC>
__global__ void __launch_bounds__(kMgThreads, 1) decode_mega_kernel(const MegaArgs a) {
  using Lay = MgLay<MT>;
  extern __shared__ __align__(128) uint8_t mg_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned gen = 0;
  const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(mg_smem);
  uint64_t* sBar = reinterpret_cast<uint64_t*>(mg_smem + Lay::kMisc + 256);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(sBar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  MgRing ring;
  ring.mode(smem0, warp, kMgWBytes, Lay::kStagesRes);
  MgWork work;
  uint32_t a_par = 0;                 // phase parity of the resident-A barrier
  float* ssq_x = a.ssq;                                   // [grid][32]
  float* ssq_mid = a.ssq + (long long)gridDim.x * 32;
  const int ldq = a.QD + 2 * a.KD;
  const int half = a.hd / 2;

  for (int it = 0; it < a.n_steps; ++it) {
    int slot = 0;
    // ---- E: x = embed[cur_tok], its row sums of squares, cos / sin of the current positions ----
    {
      if (threadIdx.x < 32) ssq_x[blockIdx.x * 32 + threadIdx.x] = 0.f;
      __syncthreads();
      for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
        const bf16* src = a.embed + (long long)a.sink.st.cur_tok[b] * a.H;
        float sq = 0.f;
        for (int c = threadIdx.x * 8; c < a.H; c += kMgThreads * 8) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + c);
          *reinterpret_cast<uint4*>(a.x + (long long)b * a.H + c) = v;
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) sq += bf16_lo(u[k]) * bf16_lo(u[k]) + bf16_hi(u[k]) * bf16_hi(u[k]);
        }
        sq = warp_sum(sq);
        __shared__ float s_part[kMgWarps];
        if (lane == 0) s_part[warp] = sq;
        __syncthreads();
        if (threadIdx.x == 0) {
          float tot = 0.f;
          for (int ww = 0; ww < kMgWarps; ++ww) tot += s_part[ww];
          ssq_x[blockIdx.x * 32 + b] = tot;
        }
        for (int j = threadIdx.x; j < half; j += kMgThreads) {
          const int axis = j < a.sec_t ? 0 : (j < a.sec_t + a.sec_h ? 1 : 2);
          const float inv = 1.0f / powf(a.theta, (float)(2 * j) / (float)a.hd);
          const float ang = (float)a.sink.st.pos3[axis * a.B + b] * inv;
          a.cs[(long long)b * half + j] = cosf(ang);
          a.cs[(long long)a.B * half + (long long)b * half + j] = sinf(ang);
        }
        __syncthreads();
      }
    }
    work.begin(a.layer[0].qkv_w, a.H, ldq, warp);
    ring.fill(work, lane);
    MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;

    for (int L = 0; L < a.layers; ++L) {
      const MegaLayer& W = a.layer[L];
      MgEpi e;
      // ---- qkv = rs * (W' x) + b ----
      mg_row_scale(a, mg_smem, ssq_x);
      e.out = a.qkv; e.ldo = ldq; e.bias = W.qkv_b; e.resid = nullptr; e.ssq_slot = nullptr; e.scale_rows = true;
      mg_gemm_phase<MG_EPI_QKV, MT, false>(a, mg_smem, a.x, a.H, a.H, ldq, work, ring, e, a_par, nullptr, nullptr);
      mg_wait<0>();                                          // (nothing is in flight: the attention ring aliases the weight ring)
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
      // ---- attention (rope, cache append, split-KV tiles, combine) ----
      mg_attention_phase(a, mg_smem, L, it);
      __syncthreads();
      ring.mode(smem0, warp, kMgWBytes, Lay::kStagesRes);
      work.begin(W.o_w, a.QD, a.H, warp);
      ring.fill(work, lane);
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
      // ---- x_mid = x + att . Wo^T ----
      e.out = a.x_mid; e.ldo = a.H; e.bias = nullptr; e.resid = a.x; e.ssq_slot = ssq_mid + blockIdx.x * 32; e.scale_rows = false;
      mg_gemm_phase<MG_EPI_RESID, MT, false>(a, mg_smem, a.att, a.QD, a.QD, a.H, work, ring, e, a_par, nullptr, nullptr);
      work.begin(W.gu_w, a.H, 2 * a.I, warp);
      ring.fill(work, lane);
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
      // ---- h = silu(rs * Wg' x_mid) * (rs * Wu' x_mid) ----
      mg_row_scale(a, mg_smem, ssq_mid);
      e.out = a.h; e.ldo = a.I; e.resid = nullptr; e.ssq_slot = nullptr; e.scale_rows = true;
      mg_gemm_phase<MG_EPI_GATEUP, MT, false>(a, mg_smem, a.x_mid, a.H, a.H, 2 * a.I, work, ring, e, a_par, nullptr, nullptr);
      // down-proj: self-contained stages (weights + the A slice); only the WEIGHT half could be prefetched before the barrier, so the
      // ring is re-configured here and filled after it (h is complete only then)
      ring.mode(smem0, warp, Lay::kSelfStage, Lay::kStagesSelf);
      work.begin(W.down_w, a.I, a.H, warp, a.h, a.I, a.B, 16 * MT);
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
      // ---- x = x_mid + h . Wd^T ----
      e.out = a.x; e.ldo = a.H; e.resid = a.x_mid; e.ssq_slot = ssq_x + blockIdx.x * 32; e.scale_rows = false;
      mg_gemm_phase<MG_EPI_RESID, MT, true>(a, mg_smem, a.h, a.I, a.I, a.H, work, ring, e, a_par, nullptr, nullptr);
      ring.mode(smem0, warp, kMgWBytes, Lay::kStagesRes);
      if (L + 1 < a.layers) work.begin(a.layer[L + 1].qkv_w, a.H, ldq, warp);
      else work.begin(a.head_w, a.H, a.V, warp);
      ring.fill(work, lane);
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
    }
    // ---- LM head: running arg-max of this CTA's columns (sampled or scored: the logits rows) ----
    [[maybe_unused]] float best_val = -INFINITY;
    [[maybe_unused]] int best_idx = 0x7fffffff;
    if constexpr (MODE != DEC_GREEDY) {
      MgEpi e;
      e.out = nullptr; e.ldo = 0; e.bias = nullptr; e.resid = nullptr; e.ssq_slot = nullptr; e.scale_rows = true;
      mg_row_scale(a, mg_smem, ssq_x);
      mg_gemm_phase<MG_EPI_LOGITS, MT, false>(a, mg_smem, a.x, a.H, a.H, a.V, work, ring, e, a_par, nullptr, nullptr);
      MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
      // ---- CTA b draws sequence b's token.  Its scratch aliases the weight ring: the head phase consumed every stage it
      // issued and the next step's first fill comes after the barriers below, so no cp.async is in flight here ----
      if ((int)blockIdx.x < a.B) {
        mg_wait<0>();
        SampleSmem<kMgThreads>& sm = *reinterpret_cast<SampleSmem<kMgThreads>*>(mg_smem);
        const int b = blockIdx.x;
        if constexpr (PROC) {    // the logits processors on the row CTA b owns (nothing past the sequence's stop)
          const int col = a.sink.col != nullptr ? __ldcg(a.sink.col + b) : __ldcg(a.sink.st.step);
          if (col < a.sink.max_new && !__ldcg(a.sink.st.finished + b))
            process_row<kMgThreads>(a.proc, b, col, a.logits + (long long)b * a.V, a.V, a.sink.out_tokens + (long long)b * a.sink.max_new,
                                    MODE == DEC_SCORED && a.sc_logits != nullptr ? a.sc_logits + ((long long)col * a.B + b) * a.V : nullptr);
        }
        if constexpr (MODE == DEC_SCORED) {
          const float* row = a.logits + (long long)b * a.V;
          const int step = __ldcg(a.sink.st.step);
          const int tok = sample_row<kMgThreads, SMP_DRAW_KEPT>(row, a.V, a.samp[b], step, sm);
          if (threadIdx.x == 0) a.samp_tok[b] = tok;
          if (step < a.sink.max_new && !__ldcg(a.sink.st.finished + b)) {       // past the sequence's stop nothing is recorded
            const long long o = ((long long)step * a.B + b) * a.V;
            const float lp = score_row<kMgThreads>(row, a.V, a.samp[b].temperature, tok, sm, a.sc_scores ? a.sc_scores + o : nullptr,
                                                   a.sc_logits && !PROC ? a.sc_logits + o : nullptr);
            if (threadIdx.x == 0 && a.sc_logprobs != nullptr) a.sc_logprobs[(long long)b * a.sink.max_new + step] = lp;
          }
        } else {
          // the Philox step is the output column: the call's step counter, or (slot pool) the slot's own column
          const int col = a.sink.col != nullptr ? __ldcg(a.sink.col + b) : __ldcg(a.sink.st.step);
          const int tok = sample_row<kMgThreads>(a.logits + (long long)b * a.V, a.V, a.samp[b], col, sm);
          if (threadIdx.x == 0) a.samp_tok[b] = tok;
        }
      }
    } else {
      MgEpi e;
      e.out = nullptr; e.ldo = 0; e.bias = nullptr; e.resid = nullptr; e.ssq_slot = nullptr; e.scale_rows = true;
      mg_row_scale(a, mg_smem, ssq_x);
      mg_gemm_phase<MG_EPI_HEAD, MT, false>(a, mg_smem, a.x, a.H, a.H, a.V, work, ring, e, a_par, &best_val, &best_idx);
      // the 8 threads of a row hold disjoint columns: merge (lowest index among equal maxima)
#pragma unroll
      for (int o2 = 1; o2 < 8; o2 <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best_val, o2);
        const int oi = __shfl_xor_sync(0xffffffffu, best_idx, o2);
        if (ov > best_val || (ov == best_val && oi < best_idx)) { best_val = ov; best_idx = oi; }
      }
      const int row = threadIdx.x >> 3;
      if ((threadIdx.x & 7) == 0) { a.amax_val[blockIdx.x * 32 + row] = best_val; a.amax_idx[blockIdx.x * 32 + row] = best_idx; }
    }
    MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
    // ---- CTA 0: merge the arg-max slots (a warp per sequence), then record the column as decode_update_kernel does ----
    if (blockIdx.x == 0) {
      const int step = *a.sink.st.step;
      bool publish = false, cancel = false;
      column_prologue<STREAM>(a.sink, step, publish, cancel);
      for (int b = warp; b < a.B; b += kMgWarps) {
        [[maybe_unused]] float bv = -INFINITY; int bi = 0x7fffffff;
        if constexpr (MODE != DEC_GREEDY) {
          bi = __ldcg(a.samp_tok + b);
        } else {
          for (int c = lane; c < (int)gridDim.x; c += 32) {
            const float v = __ldcg(a.amax_val + c * 32 + b); const int i = __ldcg(a.amax_idx + c * 32 + b);
            if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
          }
#pragma unroll
          for (int o2 = 16; o2 > 0; o2 >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o2);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o2);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
          }
        }
        if (lane == 0) record_token<STREAM>(a.sink, a.B, b, step, bi, true, publish, cancel);
      }
      column_epilogue<STREAM>(a.sink, step, publish, cancel);
    }
    MG_STAMP(slot, 0); mg_grid_sync(a.bar, gen); MG_STAMP(slot, 1); ++slot;
    if (__ldcg(a.sink.st.n_active) <= a.exit_at) break;   // (exit_at 0: every sequence has stopped; the tail of out_tokens is pad already)
  }
  mg_wait<0>();
}

}  // namespace fo1

namespace fo1 {

// every instantiation, [MT - 1][DecodeMode][STREAM]
// every instantiation, [MT - 1][DecodeMode][STREAM][PROC]; a greedy call with processors runs DEC_SAMPLED, so the greedy loop has
// no PROC instantiation (its slot repeats the plain one)
#define MG_PAIR(MT, MODE, STREAM, P) {reinterpret_cast<void*>(decode_mega_kernel<MT, MODE, STREAM, false>), \
                                      reinterpret_cast<void*>(decode_mega_kernel<MT, MODE, STREAM, P>)}
#define MG_KERNELS(MT, MODE, P) {MG_PAIR(MT, MODE, false, P), MG_PAIR(MT, MODE, true, P)}
static void* const kMgKernels[2][3][2][2] = {{MG_KERNELS(1, DEC_GREEDY, false), MG_KERNELS(1, DEC_SAMPLED, true), MG_KERNELS(1, DEC_SCORED, true)},
                                             {MG_KERNELS(2, DEC_GREEDY, false), MG_KERNELS(2, DEC_SAMPLED, true), MG_KERNELS(2, DEC_SCORED, true)}};
#undef MG_KERNELS
#undef MG_PAIR

int decode_mega_grid() {
  static int grid = -1;
  if (grid < 0) {
    grid = 0;
    int dev = 0, coop = 0, per_sm = 0;
    bool ok = cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) == cudaSuccess && coop;
    for (const auto& per_mt : kMgKernels)
      for (const auto& per_mode : per_mt)
        for (const auto& per_stream : per_mode)
          for (void* fn : per_stream)
          ok = ok && cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kMgSmemBytes) == cudaSuccess &&
               cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kMgThreads, kMgSmemBytes) == cudaSuccess && per_sm >= 1;
    if (ok)
      grid = device_sm_count();
    else
      fprintf(stderr, "[fo1] decode_mega: cooperative launch with %d B of shared memory is not available (%s); using the per-kernel decode path\n",
              kMgSmemBytes, cudaGetErrorString(cudaGetLastError()));
    cudaGetLastError();
  }
  return grid;
}

// FO1_MEGA_PROF: where the first decode iteration spent its time, from its MG_STAMP / MG_ASTAMP slots, on stderr (after a synchronise)
static int mg_prof_report(const MegaArgs& a, int grid, cudaStream_t s) {
  const int prof_slots = a.prof_slots;
  std::vector<unsigned long long> h((size_t)grid * prof_slots * 2);
  FO1_CUDA(cudaStreamSynchronize(s));
  FO1_CUDA(cudaMemcpy(h.data(), a.prof, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  cudaFree(a.prof);
  // per slot: the last CTA to enter the barrier ends the phase; release = when CTA 0 leaves.  work = last_enter - previous release,
  // skew = last_enter - first_enter, barrier = release - last_enter
  const char* names[5] = {"qkv", "attn", "oproj", "gateup", "down"};
  double tot[5][3] = {{0}}, misc = 0;
  unsigned long long prev_release = 0;
  for (int sl = 0; sl < prof_slots - 8; ++sl) {
    unsigned long long first = ~0ull, last = 0, rel = 0;
    for (int cta = 0; cta < grid; ++cta) {
      const unsigned long long e = h[((size_t)cta * prof_slots + sl) * 2], l = h[((size_t)cta * prof_slots + sl) * 2 + 1];
      if (e < first) first = e;
      if (e > last) last = e;
      if (l > rel) rel = l;
    }
    if (sl >= 1 && sl <= 5 * a.layers) {
      const int ph = (sl - 1) % 5;
      tot[ph][0] += (double)(last - prev_release); tot[ph][1] += (double)(last - first); tot[ph][2] += (double)(rel - last);
    } else if (sl > 0) misc += (double)(rel - prev_release);
    prev_release = rel;
  }
  fprintf(stderr, "[decode_mega profile, first iteration, B=%d, %d CTAs] per layer (us): ", a.B, grid);
  for (int ph = 0; ph < 5; ++ph)
    fprintf(stderr, "%s work %.1f (skew %.1f) barrier %.1f | ", names[ph], tot[ph][0] / a.layers / 1e3, tot[ph][1] / a.layers / 1e3,
            tot[ph][2] / a.layers / 1e3);
  fprintf(stderr, "head+update %.1f us\n", misc / 1e3);
  {   // distribution over CTAs of the time spent in layer 1's attention phase (slot 7: enter of the barrier after it; slot 6: leave before it)
    std::vector<std::pair<double, int>> dur;
    for (int cta = 0; cta < grid; ++cta)
      dur.push_back({(double)(h[((size_t)cta * prof_slots + 7) * 2] - h[((size_t)cta * prof_slots + 6) * 2 + 1]) / 1e3, cta});
    std::sort(dur.begin(), dur.end());
    fprintf(stderr, "[decode_mega profile] attention phase per CTA (us): min %.1f p25 %.1f median %.1f p75 %.1f max %.1f; slowest CTAs:", dur[0].first,
            dur[grid / 4].first, dur[grid / 2].first, dur[3 * grid / 4].first, dur.back().first);
    for (int k = 0; k < 6; ++k) fprintf(stderr, " %d(%.1f)", dur[grid - 1 - k].second, dur[grid - 1 - k].first);
    fprintf(stderr, "\n");
  }
  fprintf(stderr, "[decode_mega profile] attention item of CTA 0, layer 1 (us since its start): ");
  const unsigned long long a0 = h[((size_t)0 * prof_slots + prof_slots - 8) * 2];
  const char* an[8] = {"start", "append+fence", "q rotated", "tiles done", "warps synced", "partials written", "fence+sync", "combined"};
  for (int k = 0; k < 8; ++k) fprintf(stderr, "%s %.1f | ", an[k], (double)(h[((size_t)0 * prof_slots + prof_slots - 8 + k) * 2] - a0) / 1e3);
  fprintf(stderr, "\n");
  return FO1_OK;
}

bool decode_mega_supports(int H, int hd, int q_heads, int kv_heads, int I, int V) {
  const int QD = q_heads * hd, KD = kv_heads * hd;
  // one GQA group (<= 8 query heads of 128) is the row block of an m16 attention tile
  const bool heads = hd == 128 && kv_heads >= 1 && q_heads % kv_heads == 0 && q_heads / kv_heads <= 8;
  // every matrix phase: K in 64-wide chunks over all 8 warps, N in 16-column tiles, A resident up to 2048 wide
  const bool widths = H % kMgChunkK == 0 && QD % kMgChunkK == 0 && I % kMgChunkK == 0 && H <= kMgAK && QD <= kMgAK &&
                      H / kMgChunkK >= kMgWarps && QD / kMgChunkK >= kMgWarps && H % kMgTileN == 0 && (QD + 2 * KD) % kMgTileN == 0 &&
                      (2 * I) % kMgTileN == 0;
  return heads && widths && V % kMgTileN == 0;
}

// One cooperative launch for the whole decode loop.  `a.bar` and `a.att_count` must be zero (the caller memsets them on `s`).
int decode_mega_run(MegaArgs a, DecodeMode mode, cudaStream_t s) {
  const int grid = decode_mega_grid();
  FO1_CHECK_ARG(grid > 0, "decode_mega: cooperative launch of a %d-byte-smem CTA per SM is not available on this device", kMgSmemBytes);
  FO1_CHECK_ARG(a.B >= 1 && a.B <= kMgRows, "decode_mega: %d sequences (1..%d)", a.B, kMgRows);
  FO1_CHECK_ARG(a.QD == a.q_heads * a.hd && a.KD == a.kv_heads * a.hd && decode_mega_supports(a.H, a.hd, a.q_heads, a.kv_heads, a.I, a.V),
                "decode_mega: unsupported shape (H %d, %d q / %d kv heads of %d, I %d, V %d)", a.H, a.q_heads, a.kv_heads, a.hd, a.I, a.V);
  FO1_CHECK_ARG(mode != DEC_SCORED || a.samp != nullptr, "decode_mega: scoring needs the per-row sampling parameters");
  FO1_CHECK_ARG(mode == DEC_GREEDY || (a.samp != nullptr && a.logits != nullptr && a.samp_tok != nullptr && (a.V & 1) == 0),
                "decode_mega: sampling buffers missing");
  FO1_CHECK_ARG(mode != DEC_GREEDY || a.proc.tab == nullptr, "decode_mega: logits processors run in the sampled or scored loop");
  const StreamArgs& sa = a.sink.stream;
  FO1_CHECK_ARG(sa.progress == nullptr || (sa.tokens != nullptr && sa.lens != nullptr), "decode_mega: stream buffers missing");
  const bool prof = getenv("FO1_MEGA_PROF") != nullptr;
  if (prof) {
    // per CTA: one slot per grid barrier (the embedding, 5 per layer, the sampling barrier of the sampled / scored modes, the
    // head, the record), then the 8 sub-stamps of one attention item (CTA 0, layer 1)
    a.prof_slots = 5 * a.layers + 3 + (mode != DEC_GREEDY ? 1 : 0) + 8;
    const size_t bytes = (size_t)grid * a.prof_slots * 2 * sizeof(unsigned long long);
    FO1_CUDA(cudaMalloc(reinterpret_cast<void**>(&a.prof), bytes));
    FO1_CUDA(cudaMemsetAsync(a.prof, 0, bytes, s));
  }
  {
    void* params[] = {&a};
    ProfScope ps("decode_mega", 0.0, 0.0, s);
    FO1_CUDA(cudaLaunchCooperativeKernel(kMgKernels[a.B <= 16 ? 0 : 1][mode][sa.progress != nullptr][a.proc.tab != nullptr], dim3(grid), dim3(kMgThreads), params,
                                         kMgSmemBytes, s));
    count_launch();
  }
  return prof ? mg_prof_report(a, grid, s) : FO1_OK;
}

}  // namespace fo1
