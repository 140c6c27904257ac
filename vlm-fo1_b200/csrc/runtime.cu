// runtime.cu -- error reporting and launch accounting behind the C ABI.
#include <array>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace fo1 {

static thread_local char t_err[1024] = {0};
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
}


// ---- profiler ------------------------------------------------------------------------------------
bool g_prof_on = false;
thread_local bool t_pdl = false;
thread_local bool t_splitk_ok = false;
thread_local int t_gemm_choice_m = 0;
struct ProfRec { cudaEvent_t a, b; std::string tag; double flops, bytes; };
static std::vector<ProfRec> g_recs;
static std::mutex g_prof_mu;

ProfScope::ProfScope(const char* tag, double flops, double bytes, cudaStream_t stream) : idx(-1), s(stream) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfRec r;
  r.tag = tag; r.flops = flops; r.bytes = bytes;
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, stream);
  g_recs.push_back(r);
  idx = (int)g_recs.size() - 1;
}
ProfScope::~ProfScope() {
  if (idx < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_recs[idx].b, s);
}

}  // namespace fo1

extern "C" void fo1_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(fo1::g_prof_mu);
  for (auto& r : fo1::g_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  fo1::g_recs.clear();
  fo1::g_prof_on = on != 0;
}

extern "C" int fo1_profile_collect(char* buf, size_t cap) {
  if (!buf || cap < 64) return FO1_ERR_INVALID_ARG;
  if (cudaDeviceSynchronize() != cudaSuccess) { fo1::set_error("fo1_profile_collect: device sync failed"); return FO1_ERR_CUDA; }
  std::lock_guard<std::mutex> lk(fo1::g_prof_mu);
  std::map<std::string, std::array<double, 5>> agg;  // launches, ms, flops, bytes, max_ms
  for (auto& r : fo1::g_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) continue;
    auto& a = agg[r.tag];
    a[0] += 1; a[1] += ms; a[2] += r.flops; a[3] += r.bytes; a[4] = ms > a[4] ? ms : a[4];
  }
  std::string js = "{";
  bool first = true;
  for (auto& kv : agg) {
    char tmp[256];
    snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"launches\": %.0f, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e, \"max_ms\": %.6f}",
             first ? "" : ", ", kv.first.c_str(), kv.second[0], kv.second[1], kv.second[2], kv.second[3], kv.second[4]);
    js += tmp;
    first = false;
  }
  js += "}";
  if (js.size() + 1 > cap) { fo1::set_error("fo1_profile_collect: buffer too small"); return FO1_ERR_WORKSPACE; }
  memcpy(buf, js.c_str(), js.size() + 1);
  return FO1_OK;
}

extern "C" int fo1_abi_version(void) { return FO1_ABI_VERSION; }
extern "C" const char* fo1_last_error(void) { return fo1::t_err; }
extern "C" uint64_t fo1_launch_count(void) { return fo1::g_launches.load(); }
extern "C" void fo1_launch_count_reset(void) { fo1::g_launches.store(0); }
