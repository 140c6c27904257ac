// Streaming-pattern probe for the decode weight ring (development tool, not part of the library):
// how fast can 148 CTAs x 8 warps pull a [N][K] bf16 matrix through shared memory with
//   mode 0: per-warp cp.async rings, 16 rows x 128 B per stage from a row-major matrix (the decode_mega v2 pattern)
//   mode 1: mode 0 + two __syncthreads per 4 stages (the cross-warp reduction cadence)
//   mode 2: per-warp rings fed by ONE cp.async.bulk per stage from a tile-contiguous copy (stage bytes = SB)
//   mode 3: mode 2 + the two __syncthreads per tile
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o scripts/probes/stream_probe scripts/probes/stream_probe.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("cuda error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ void cp16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void waitg() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wait_n(int n) {
  switch (n) { case 0: waitg<0>(); break; case 1: waitg<1>(); break; case 2: waitg<2>(); break; case 3: waitg<3>(); break;
    case 4: waitg<4>(); break; case 5: waitg<5>(); break; case 6: waitg<6>(); break; case 7: waitg<7>(); break;
    case 8: waitg<8>(); break; case 9: waitg<9>(); break; case 10: waitg<10>(); break; case 11: waitg<11>(); break;
    case 12: waitg<12>(); break; case 13: waitg<13>(); break; case 14: waitg<14>(); break; default: waitg<15>(); break; }
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) asm volatile("{\n.reg .pred P;\nmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\nselp.u32 %0, 1, 0, P;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// mode 0/1: matrix [N][K] row-major, tile = 16 rows, chunk = 64 k (2 KB per stage), warp w takes chunks w, w+8, ...
__global__ void __launch_bounds__(256, 1) probe_cpasync(const uint16_t* W, int N, int K, int depth, int syncs, unsigned* sink) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(smem) + warp * depth * 2048;
  const int n_tiles = N / 16, chunks = K / 64;
  int it = blockIdx.x, ic = warp;          // issue cursor
  int head = 0, tail = 0, inflight = 0;
  unsigned acc = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int kc = warp; kc < chunks; kc += 8) {
      while (inflight < depth - 1 && it < n_tiles) {
        const uint32_t st = base + (head % depth) * 2048;
        const uint16_t* src = W + (long long)it * 16 * K + ic * 64;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = i * 4 + (lane >> 3), c16 = lane & 7;
          cp16(st + row * 128 + ((c16 ^ (row & 7)) << 4), src + (long long)row * K + c16 * 8);
        }
        commit(); ++head; ++inflight;
        ic += 8; if (ic >= chunks) { ic = warp; it += gridDim.x; }
      }
      wait_n(inflight - 1);
      __syncwarp();
      acc += *reinterpret_cast<const unsigned*>(smem + warp * depth * 2048 + (tail % depth) * 2048 + lane * 64);
      __syncwarp();
      ++tail; --inflight;
    }
    if (syncs) { __syncthreads(); __syncthreads(); }
  }
  if (acc == 0x12345678u) *sink = acc;
}

// mode 2/3: tile-contiguous copy: [tile][chunk group][SB bytes]; warp w takes stages w, w+8, ... of the tile
__global__ void __launch_bounds__(256, 1) probe_bulk(const uint8_t* W, int n_tiles, int tile_bytes, int SB, int depth, int syncs, unsigned* sink) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[8 * 16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(smem) + warp * depth * SB;
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(bars + warp * 16);
  if (lane == 0) for (int i = 0; i < depth; ++i) mbar_init(bar0 + i * 8, 1);
  __syncthreads();
  const int per_tile = tile_bytes / SB;     // stages per tile
  int it = blockIdx.x, ic = warp;
  int head = 0, tail = 0, inflight = 0;
  unsigned acc = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int kc = warp; kc < per_tile; kc += 8) {
      while (inflight < depth - 1 && it < n_tiles) {
        if (lane == 0) {
          const int s = head % depth;
          mbar_expect(bar0 + s * 8, SB);
          bulk(base + s * SB, W + (long long)it * tile_bytes + (long long)ic * SB, SB, bar0 + s * 8);
        }
        ++head; ++inflight;
        ic += 8; if (ic >= per_tile) { ic = warp; it += gridDim.x; }
      }
      const int s = tail % depth;
      mbar_wait(bar0 + s * 8, (tail / depth) & 1);
      acc += *reinterpret_cast<const unsigned*>(smem + warp * depth * SB + s * SB + lane * 64);
      __syncwarp();
      ++tail; --inflight;
    }
    if (syncs) { __syncthreads(); __syncthreads(); }
  }
  if (acc == 0x12345678u) *sink = acc;
}

int main() {
  const int N = 22016, K = 2048, NBUF = 8;
  const size_t bytes = (size_t)N * K * 2;
  uint8_t* buf[NBUF];
  for (int i = 0; i < NBUF; ++i) { CK(cudaMalloc(&buf[i], bytes)); CK(cudaMemset(buf[i], i + 1, bytes)); }
  unsigned* sink; CK(cudaMalloc(&sink, 4));
  CK(cudaFuncSetAttribute(probe_cpasync, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CK(cudaFuncSetAttribute(probe_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto run = [&](const char* name, auto launch) {
    for (int i = 0; i < NBUF; ++i) launch(i);
    CK(cudaDeviceSynchronize());
    const int reps = 4 * NBUF;
    CK(cudaEventRecord(e0));
    for (int r = 0; r < reps; ++r) launch(r % NBUF);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaGetLastError());
    printf("%-44s %7.1f us/pass  %6.2f TB/s\n", name, ms * 1e3 / reps, bytes * reps / (ms * 1e-3) / 1e12);
  };
  char name[128];
  for (int syncs = 0; syncs < 2; ++syncs)
    for (int depth : {5, 9, 12}) {
      snprintf(name, sizeof name, "cp.async 2KB stages depth %d syncs %d (%d KB/SM)", depth, syncs, 8 * (depth - 1) * 2);
      run(name, [&](int i) { probe_cpasync<<<148, 256, 8 * depth * 2048>>>((const uint16_t*)buf[i], N, K, depth, syncs, sink); });
    }
  for (int syncs = 0; syncs < 2; ++syncs)
    for (int SB : {2048, 4096, 8192})
      for (int kb : {64, 128, 184}) {
        int depth = kb * 1024 / 8 / SB + 1;
        if (depth < 2 || depth > 16) continue;
        if (8 * depth * SB > 200 * 1024) continue;
        snprintf(name, sizeof name, "bulk %d B stages depth %d syncs %d (%d KB/SM)", SB, depth, syncs, 8 * (depth - 1) * SB / 1024);
        run(name, [&](int i) { probe_bulk<<<148, 256, 8 * depth * SB>>>(buf[i], N / 16, 16 * K * 2, SB, depth, syncs, sink); });
      }
  // one-shot latency of a short phase: a single pass over 10 MB (the qkv matrix) from a cold start
  return 0;
}
