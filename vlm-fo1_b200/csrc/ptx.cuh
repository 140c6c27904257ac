// ptx.cuh -- thin inline-PTX wrappers for the sm_90a async machinery: mbarrier, TMA, wgmma.
#pragma once
#include <stdint.h>

#include "wgmma.cuh"

namespace fo1 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n.reg .pred P;\n.reg .b32 R;\nelect.sync R|P, 0xffffffff;\nselp.u32 %0, 1, 0, P;\n}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n.reg .pred P;\nmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\nselp.u32 %0, 1, 0, P;\n}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- thread-block clusters ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders the shared-memory (and mbarrier) accesses before it against those after it
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster.  Default (CTA-scope) release: it only signals
// that this warp's wgmma reads of a stage have retired (wgmma.wait_group), and a cluster-scope release would cost a GPU-wide fence
// per k-block.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(rank));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

// ---- TMA (cp.async.bulk.tensor) ----------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// the same box into the same shared-memory offset of every CTA in `cta_mask`, each completing the bytes on its own mbarrier at
// `bar`'s offset
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- wgmma (warpgroup MMA; the instruction wrappers are in wgmma.cuh) ---------------------------
// generic-proxy shared-memory writes (st.shared) -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// orders the warpgroup's register / shared-memory accesses before the wgmma.mma_async that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses to accumulator registers across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128-byte-swizzled shared-memory operand descriptor: rows of 128 B (64 bf16 of K), 8-row swizzle atoms
// 1024 B apart (SBO); LBO is not used for a single 64-element K atom.  A 16-element K step inside the atom advances
// the start address by 32 B.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);          // start address, 16-byte units
  d |= (uint64_t)1 << 16;                              // leading byte offset (ignored)
  d |= (uint64_t)(1024 >> 4) << 32;                    // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                              // SWIZZLE_128B
  return d;
}
// MN-major, 128-byte-swizzled operand (a [K index][64 MN-elements] TMA tile used with the transpose bit, e.g. V[key][dim]
// as the B operand of P.V): rows of 128 B = 64 MN-elements of one K index, 8-row (8 K indices) groups SBO = 1024 B
// apart, 64-element atoms along MN `lbo` bytes apart.  A 16-element K step advances the start address by 2048 B.
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

}  // namespace ptx

// ---- accumulator fragments -> row-contiguous global stores -----------------------------------------------------------
// A warp of a warpgroup owns 16 accumulator rows; lane l holds rows l / 4 and l / 4 + 8, two adjacent columns per
// 8-column chunk.  Storing from there writes 8 rows x 16 B per instruction, so the warp parks 16 rows x 256 B in shared
// memory (16-byte slots XOR-swizzled by row: conflict-free both ways) and writes whole 256-byte rows back.
constexpr int kFragStageBytes = 16 * 256;
// 4-byte word `w` (0..63) of row `row` (0..15) of a warp's staging block
__device__ __forceinline__ uint32_t* frag_stage_word(uint8_t* stg, int row, int w) {
  return reinterpret_cast<uint32_t*>(stg + row * 256 + ((((w >> 2) ^ (row & 7)) << 4) | ((w & 3) << 2)));
}
__device__ __forceinline__ uint4 frag_stage_slot(const uint8_t* stg, int row, int slot) {
  return *reinterpret_cast<const uint4*>(stg + row * 256 + ((slot ^ (row & 7)) << 4));
}

}  // namespace fo1
