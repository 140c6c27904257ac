// engine.cuh -- the model handle behind the C ABI: borrowed weight table, one grow-only device arena,
// cached integer index tables.  Host-side orchestration (layer loops) lives in vit.cu / davit.cu / llm.cu.
#pragma once
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "kernels.cuh"

namespace fo1 {

struct WeightRef {
  const void* ptr = nullptr;
  int dtype = FO1_BF16;
  std::vector<int64_t> shape;
};

// Bump allocator over one device block.  `measure` mode only counts, so every forward can be
// dry-run once to size the block; steady state performs no allocation.
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool measure = false;
  void reset(bool measure_only) { off = 0; peak = 0; measure = measure_only; }
  template <typename T>
  T* alloc(size_t n) {
    off = align_up(off, 256);
    T* p = measure ? reinterpret_cast<T*>(uintptr_t(256)) : reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    if (off > peak) peak = off;
    return p;
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};

struct DeviceInts {  // cached host->device integer table
  int* dev = nullptr;
  size_t n = 0;
};


struct VitBlockW { const bf16 *norm1, *qkv_w, *qkv_b, *proj_w, *proj_b, *norm2, *gateup_w, *gateup_b, *down_w, *down_b; };
struct VitW {
  const bf16* patch_w = nullptr;
  std::vector<VitBlockW> blk;
  const bf16 *ln_q = nullptr, *fc1_w = nullptr, *fc1_b = nullptr, *fc2_w = nullptr, *fc2_b = nullptr;
  bool ok = false;
};
struct DavitHalfW {  // one SpatialBlock or ChannelBlock
  const bf16 *conv1_w9, *conv1_b, *norm1_w, *norm1_b, *qkv_w, *qkv_b, *proj_w, *proj_b;
  const bf16 *conv2_w9, *conv2_b, *norm2_w, *norm2_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
};
struct DavitStageW {
  const bf16 *conv_w, *conv_b, *norm_w, *norm_b;
  std::vector<DavitHalfW> sp, ch;
};
struct DavitW { DavitStageW st[4]; bool ok = false; };
struct FpnLevelW { const bf16 *conv1_w, *ln1_w, *ln1_b, *conv2_w, *ln2_w, *ln2_b; };
struct FpnW {
  const bf16 *l0_dc1_w, *l0_dc1_b, *l0_ln_w, *l0_ln_b, *l0_dc2_w, *l0_dc2_b, *l1_dc_w, *l1_dc_b;
  FpnLevelW lv[4];
  bool ok = false;
};
struct ProjW { std::vector<const bf16*> w, b; std::vector<int> in_dim, out_dim; bool ok = false; };
struct LlmLayerW {
  const bf16 *ln1, *qkv_w, *qkv_b, *o_w, *ln2, *gateup_w, *down_w;
  const bf16 *qkv_dec = nullptr, *gu_dec = nullptr;   // decode copies with the RMSNorm gains folded in (persistent decode kernel)
};
struct LlmW {
  const bf16 *embed = nullptr, *norm = nullptr, *lm_head = nullptr, *head_dec = nullptr;
  std::vector<LlmLayerW> layer;
  bool ok = false;
  bool mega_ok = false;        // every decode copy is present: the greedy loop runs as one persistent kernel
  void* mega_layers = nullptr; // device array of MegaLayer (decode_mega.cuh), owned by llm.cu
};

struct Model {
  fo1_model_config cfg;
  VitW vit; DavitW davit; FpnW fpn; ProjW proj_aux, proj_img; LlmW llm;
  std::unordered_map<std::string, WeightRef> weights;
  bool finalized = false;
  Arena arena;
  std::map<std::string, DeviceInts> int_cache;  // keyed by a shape signature
  int last_decode_path = -1;                    // fo1_last_decode_path(): 1 persistent kernel, 0 per-kernel graph
  // LLM state (llm.cu)
  void* kv_cache = nullptr;
  size_t kv_bytes = 0;
  int kv_batch = 0, kv_cap = 0;
  void* decode_graph = nullptr;  // cudaGraphExec_t
  std::string decode_graph_key;
  void* llm_state = nullptr;     // struct LlmState*, owned by llm.cu
  void* slot_pool = nullptr;     // struct SlotPool* while a slot pool is open (fo1_slots_open), owned by llm.cu

  const WeightRef* find(const std::string& name) const {
    auto it = weights.find(name);
    return it == weights.end() ? nullptr : &it->second;
  }
};

// weight lookup helpers: record the first missing / mis-shaped weight in an error string
struct WeightGetter {
  const Model* m;
  std::string err;
  const bf16* bf(const std::string& name, std::initializer_list<int64_t> shape) {
    const WeightRef* w = m->find(name);
    if (!w) { if (err.empty()) err = "missing weight " + name; return nullptr; }
    if (w->dtype != FO1_BF16) { if (err.empty()) err = "weight " + name + " must be bf16"; return nullptr; }
    if (shape.size() && std::vector<int64_t>(shape) != w->shape) {
      if (err.empty()) {
        err = "weight " + name + " has shape [";
        for (auto d : w->shape) err += std::to_string(d) + ",";
        err += "] expected [";
        for (auto d : shape) err += std::to_string(d) + ",";
        err += "]";
      }
      return nullptr;
    }
    return static_cast<const bf16*>(w->ptr);
  }
};

int arena_ensure(Model* m, size_t bytes);
int int_cache_trim(Model* m, size_t keep_below = 192);   // call at the entry of a forward only
int cached_ints(Model* m, const std::string& key, const std::vector<int>& host, const int** dev, cudaStream_t s);

int vit_finalize(Model* m);
int davit_finalize(Model* m);
int fpn_finalize(Model* m);
int proj_finalize(Model* m);
int llm_finalize(Model* m);

#define FO1_RUN(expr)                \
  do {                               \
    if (!dry) FO1_TRY(expr);         \
  } while (0)

}  // namespace fo1

struct fo1_model : public fo1::Model {};
