// common.cuh -- shared host/device helpers for libfo1 (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "fo1.h"

namespace fo1 {

// ---- error plumbing: never throw / exit across the C ABI --------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define FO1_CHECK_ARG(cond, ...)            \
  do {                                      \
    if (!(cond)) {                          \
      ::fo1::set_error(__VA_ARGS__);        \
      return FO1_ERR_INVALID_ARG;           \
    }                                       \
  } while (0)

#define FO1_CUDA(expr)                                                                    \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::fo1::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return FO1_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define FO1_LAUNCH_CHECK()                                                                \
  do {                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      ::fo1::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return FO1_ERR_CUDA;                                                                \
    }                                                                                     \
    ::fo1::count_launch();                                                                \
  } while (0)

#define FO1_TRY(expr)            \
  do {                           \
    int _s = (expr);             \
    if (_s != FO1_OK) return _s; \
  } while (0)

// ---- optional per-launch profiler (CUDA events on the launching stream; off by default) ----------
extern bool g_prof_on;
struct ProfScope {
  int idx;
  cudaStream_t s;
  ProfScope(const char* tag, double flops, double bytes, cudaStream_t stream);
  ~ProfScope();
};

// ---- programmatic dependent launch (decode loop) ----------------------------------------------------
// Inside a PdlScope every launch_k() carries cudaLaunchAttributeProgrammaticStreamSerialization: the kernel may start
// while its predecessor on the stream is still draining.  Kernels launched this way call griddep_wait() before they
// touch anything a predecessor wrote (and before they write anything a predecessor may still read) and
// griddep_launch() as early as possible; both are no-ops for ordinary launches.
extern thread_local bool t_pdl;
struct PdlScope {
  bool prev;
  explicit PdlScope(bool on) : prev(t_pdl) { t_pdl = on; }
  ~PdlScope() { t_pdl = prev; }
};
// Split-K of skinny GEMMs (gemm_wgmma.cu's automatic choice) is allowed only inside a SplitKScope: the decode steps and the LM head
// (M = number of sequences: weight streaming, where the choice depends on N and K only) and the public fo1_gemm_bf16.  Every other
// linear() of the engine keeps ONE accumulation order whatever its M, so a sample's tower / projector / prefill results do not depend
// on how many neighbours shared its batch (a short prompt alone used to take split-K, the same prompt inside a batch did not).
extern thread_local bool t_splitk_ok;
struct SplitKScope {
  bool prev;
  explicit SplitKScope(bool on) : prev(t_splitk_ok) { t_splitk_ok = on; }
  ~SplitKScope() { t_splitk_ok = prev; }
};
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = t_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device helpers ---------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// exact-erf GELU, x * Phi(x), with ONE special-function op per element (the GEMM epilogues are issue/MUFU-bound on
// erff): erfc(z) = 2^P(z) on z = |x|/sqrt(2) in [0, 4], P the degree-7 Chebyshev fit of log2(erfc) (relative error
// 4.3e-6, clamped beyond z = 4 where erfc < 1.6e-8); Phi(x) = erfc(z)/2 for x < 0, 1 - erfc(z)/2 otherwise.
// |gelu_erf(x) - x*Phi(x)| <= 7e-7 absolute, 4.2e-6 relative over [-8, 8] (fp32 evaluation, checked against scipy).
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fminf(fabsf(x) * 0.70710678118654752440f, 4.0f);
  float p = -2.1777637812192552e-05f;
  p = fmaf(p, z, 0.0005068330792710185f);
  p = fmaf(p, z, -0.005339398048818111f);
  p = fmaf(p, z, 0.03423144668340683f);
  p = fmaf(p, z, -0.15289084613323212f);
  p = fmaf(p, z, -0.9167589545249939f);
  p = fmaf(p, z, -1.6281543970108032f);
  p = fmaf(p, z, 6.178960575198289e-06f);
  const float q = 0.5f * ex2_approx(p);
  return x * (x < 0.f ? q : 1.0f - q);
}
__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
#endif

}  // namespace fo1
