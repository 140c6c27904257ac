// vit.cu -- primary tower: Qwen2.5-VL ViT over a packed batch of images.
//
// Follows custom_forward (qwen2_5_vl_encoder.py:86-158): patch-embed GEMM, tokens permuted into window
// order, `depth` blocks of [RMSNorm -> qkv -> 2-D RoPE -> varlen attention (64-token windows, or whole
// image at the full-attention layers) -> proj + residual -> RMSNorm -> gated-SiLU MLP + residual], hidden
// state tapped after every full-attention layer, 2x2 merger MLP, inverse permutation.
// Differences from the reference: all images of the batch run as ONE packed token sequence; the window
// permutation is folded into the fp32->bf16 cast of the pixel rows; the taps are scattered straight
// into un-windowed channels-last maps (what the reference builds later with cat/argsort/permute in
// extract_multi_level_features :37-80); bias / activation / residual live in the GEMM epilogues.
#include "engine.cuh"

namespace fo1 {

// get_window_index (modeling_qwen2_5_vl.py:465-504) for one image (t = 1) + the patch coordinates in
// window order (rot_pos_emb :436-463 composed with the permutation of custom_forward :104-109).
static void vit_window_index_host(const fo1_model_config& c, int gh, int gw, std::vector<int>& window_index,
                                  std::vector<int>& cu_win, std::vector<int>& pos_hw) {
  const int ms = c.vit_merge;
  const int lh = gh / ms, lw = gw / ms;
  const int ws = c.vit_window / ms / c.vit_patch;
  const int pad_h = ws - lh % ws, pad_w = ws - lw % ws;  // a full extra window when already divisible (:477-478)
  const int nwh = (lh + pad_h) / ws, nww = (lw + pad_w) / ws;
  window_index.clear();
  cu_win.assign(1, 0);
  const int unit = ms * ms;
  for (int wy = 0; wy < nwh; ++wy) {
    for (int wx = 0; wx < nww; ++wx) {
      int cnt = 0;
      for (int iy = 0; iy < ws; ++iy)
        for (int ix = 0; ix < ws; ++ix) {
          const int y = wy * ws + iy, x = wx * ws + ix;
          if (y < lh && x < lw) { window_index.push_back(y * lw + x); ++cnt; }
        }
      const int next = cu_win.back() + cnt * unit;
      if (next != cu_win.back()) cu_win.push_back(next);  // unique_consecutive (qwen2_5_vl_encoder.py:109)
    }
  }
  pos_hw.resize((size_t)gh * gw * 2);
  for (size_t j = 0; j < window_index.size(); ++j) {
    const int cell = window_index[j], cy = cell / lw, cx = cell % lw;
    for (int sub = 0; sub < unit; ++sub) {
      const size_t t = j * unit + sub;
      pos_hw[2 * t] = cy * ms + sub / ms;
      pos_hw[2 * t + 1] = cx * ms + sub % ms;
    }
  }
}

static int vit_resolve(Model* m) {
  const fo1_model_config& c = m->cfg;
  WeightGetter g{m, ""};
  VitW& v = m->vit;
  const int64_t H = c.vit_hidden, I2 = 2 * (int64_t)c.vit_inter_pad, Ip = c.vit_inter_pad;
  const int64_t pk = (int64_t)c.vit_in_ch * c.vit_temporal * c.vit_patch * c.vit_patch;
  v.patch_w = g.bf("vit.patch_embed.w", {H, pk});
  v.blk.resize(c.vit_depth);
  for (int i = 0; i < c.vit_depth; ++i) {
    const std::string p = "vit.blk." + std::to_string(i) + ".";
    VitBlockW& b = v.blk[i];
    b.norm1 = g.bf(p + "norm1.w", {H});
    b.qkv_w = g.bf(p + "qkv.w", {3 * H, H});
    b.qkv_b = g.bf(p + "qkv.b", {3 * H});
    b.proj_w = g.bf(p + "proj.w", {H, H});
    b.proj_b = g.bf(p + "proj.b", {H});
    b.norm2 = g.bf(p + "norm2.w", {H});
    b.gateup_w = g.bf(p + "gateup.w", {I2, H});
    b.gateup_b = g.bf(p + "gateup.b", {I2});
    b.down_w = g.bf(p + "down.w", {H, Ip});
    b.down_b = g.bf(p + "down.b", {H});
  }
  const int64_t M4 = H * c.vit_merge * c.vit_merge;
  v.ln_q = g.bf("vit.merger.ln_q.w", {H});
  v.fc1_w = g.bf("vit.merger.fc1.w", {M4, M4});
  v.fc1_b = g.bf("vit.merger.fc1.b", {M4});
  v.fc2_w = g.bf("vit.merger.fc2.w", {(int64_t)c.vit_out_hidden, M4});
  v.fc2_b = g.bf("vit.merger.fc2.b", {(int64_t)c.vit_out_hidden});
  if (!g.err.empty()) { set_error("ViT weights: %s", g.err.c_str()); return FO1_ERR_NOT_FOUND; }
  v.ok = true;
  return FO1_OK;
}

int vit_finalize(Model* m) { return m->cfg.vit_depth > 0 ? vit_resolve(m) : FO1_OK; }

static int vit_forward_impl(Model* m, const float* const* pixel_values, const int32_t* grid_hw, int B, bf16* img_feats,
                            void* const* taps, cudaStream_t s, bool dry) {
  const fo1_model_config& c = m->cfg;
  const VitW& w = m->vit;
  Arena& A = m->arena;
  const int H = c.vit_hidden, heads = c.vit_heads, hd = H / heads;
  const int unit = c.vit_merge * c.vit_merge;
  const int pk = c.vit_in_ch * c.vit_temporal * c.vit_patch * c.vit_patch;

  // ---- integer tables for this list of grids (cached on device) ----
  long long T = 0;
  std::string key = "vit";
  for (int b = 0; b < B; ++b) {
    T += (long long)grid_hw[2 * b] * grid_hw[2 * b + 1];
    key += ":" + std::to_string(grid_hw[2 * b]) + "x" + std::to_string(grid_hw[2 * b + 1]);
  }
  const int Tm = (int)(T / unit);
  const int *d_src_row = nullptr, *d_pos = nullptr, *d_cu_win = nullptr, *d_cu_full = nullptr, *d_pix = nullptr, *d_unperm = nullptr, *d_tiles = nullptr;
  int n_tiles = 0;
  int n_win = 0, max_win = 0, max_full = 0;
  double flops_win = 0.0, flops_full = 0.0;   // 4 * sum len^2 * hidden
  {
    std::vector<int> src_row, pos, cu_win(1, 0), cu_full(1, 0), pix, unperm;
    int tok_off = 0, cell_off = 0;
    for (int b = 0; b < B; ++b) {
      const int gh = grid_hw[2 * b], gw = grid_hw[2 * b + 1];
      std::vector<int> wi, cw, ph;
      vit_window_index_host(c, gh, gw, wi, cw, ph);
      for (size_t j = 0; j < wi.size(); ++j) {
        for (int sub = 0; sub < unit; ++sub) src_row.push_back(wi[j] * unit + sub);  // row inside this image's pixel tensor
        unperm.push_back(cell_off + wi[j]);
      }
      for (size_t t = 0; t < ph.size() / 2; ++t) {
        pos.push_back(ph[2 * t]); pos.push_back(ph[2 * t + 1]);
        pix.push_back(tok_off + ph[2 * t] * gw + ph[2 * t + 1]);
      }
      for (size_t i = 1; i < cw.size(); ++i) {
        cu_win.push_back(tok_off + cw[i]); max_win = std::max(max_win, cw[i] - cw[i - 1]);
        flops_win += 4.0 * (double)(cw[i] - cw[i - 1]) * (cw[i] - cw[i - 1]) * H;
      }
      flops_full += 4.0 * (double)gh * gw * gh * gw * H;
      tok_off += gh * gw;
      cell_off += gh * gw / unit;
      cu_full.push_back(tok_off);
      max_full = std::max(max_full, gh * gw);
    }
    n_win = (int)cu_win.size() - 1;
    std::vector<int> tiles;
    attention_tile_table(cu_full, tiles);   // query tiles restart at every image: an image's bits do not depend on its batch slot
    n_tiles = (int)tiles.size() / 2;
    if (!dry) {
      FO1_TRY(cached_ints(m, key + ":src", src_row, &d_src_row, s));
      FO1_TRY(cached_ints(m, key + ":pos", pos, &d_pos, s));
      FO1_TRY(cached_ints(m, key + ":cuw", cu_win, &d_cu_win, s));
      FO1_TRY(cached_ints(m, key + ":cuf", cu_full, &d_cu_full, s));
      FO1_TRY(cached_ints(m, key + ":pix", pix, &d_pix, s));
      FO1_TRY(cached_ints(m, key + ":unp", unperm, &d_unperm, s));
      FO1_TRY(cached_ints(m, key + ":til", tiles, &d_tiles, s));
    }
  }

  // ---- activations ----
  bf16* px = A.alloc<bf16>((size_t)T * pk);
  bf16* x = A.alloc<bf16>((size_t)T * H);
  bf16* x2 = A.alloc<bf16>((size_t)T * H);
  bf16* xn = A.alloc<bf16>((size_t)T * H);
  bf16* qkv = A.alloc<bf16>((size_t)T * 3 * H);
  bf16* att = A.alloc<bf16>((size_t)T * H);
  bf16* hbuf = A.alloc<bf16>((size_t)T * c.vit_inter_pad);
  float* cs = A.alloc<float>((size_t)T * hd);
  bf16* mg = A.alloc<bf16>((size_t)Tm * H * unit);
  bf16* mo = A.alloc<bf16>((size_t)Tm * c.vit_out_hidden);
  int* rs_win = A.alloc<int>((size_t)T * 2);
  int* rs_full = A.alloc<int>((size_t)T * 2);

  // ---- patch embed: cast + window-order gather, then GEMM (Conv3d with stride == kernel is a GEMM, :88-111) ----
  {
    long long off = 0;
    for (int b = 0; b < B; ++b) {
      const int n = grid_hw[2 * b] * grid_hw[2 * b + 1];
      FO1_RUN(cast_gather_rows_f32_bf16(pixel_values[b], pk, d_src_row + off, px + off * pk, pk, n, pk, s));
      off += n;
    }
  }
  FO1_RUN(linear(px, pk, w.patch_w, pk, x, H, FO1_BF16, (int)T, H, pk, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
  FO1_RUN(vit_rope_table(d_pos, cs, (int)T, hd, 10000.0f, s));
  // key range of every packed row for the two segmentations (windows / whole images): built once, read by every layer
  FO1_RUN(attention_rowseg(d_cu_win, n_win, (int)T, rs_win, s));
  FO1_RUN(attention_rowseg(d_cu_full, B, (int)T, rs_full, s));

  int tap_i = 0;
  for (int L = 0; L < c.vit_depth; ++L) {
    const VitBlockW& b = w.blk[L];
    bool full = false;
    for (int i = 0; i < c.vit_n_fullatt; ++i) full |= (c.vit_fullatt[i] == L);
    FO1_RUN(rmsnorm(x, H, b.norm1, xn, H, (int)T, H, 1e-6f, s));
    FO1_RUN(linear(xn, H, b.qkv_w, H, qkv, 3 * H, FO1_BF16, (int)T, 3 * H, H, b.qkv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
    FO1_RUN(vit_rope_apply(qkv, cs, (int)T, heads, hd, s));
    AttnArgs a;
    a.q = qkv; a.k = qkv + H; a.v = qkv + 2 * H; a.o = att;
    a.ldq = a.ldk = a.ldv = 3 * H; a.ldo = H;
    a.cu_seqlens = full ? d_cu_full : d_cu_win;
    a.n_seqs = full ? B : n_win;
    a.max_seqlen = full ? max_full : max_win;
    a.total_rows = (int)T;
    a.rowseg = full ? rs_full : rs_win;
    a.tiles = d_tiles; a.n_tiles = n_tiles;
    a.flops = full ? flops_full : flops_win;
    a.q_heads = a.kv_heads = heads; a.head_dim = hd;
    a.scale = 1.0f / sqrtf((float)hd);
    a.causal = 0;
    FO1_RUN(attention_varlen(a, s));
    FO1_RUN(linear(att, H, b.proj_w, H, x2, H, FO1_BF16, (int)T, H, H, b.proj_b, FO1_BF16, FO1_EPI_NONE, x, H, 0, s));
    FO1_RUN(rmsnorm(x2, H, b.norm2, xn, H, (int)T, H, 1e-6f, s));
    FO1_RUN(linear(xn, H, b.gateup_w, H, hbuf, c.vit_inter_pad, FO1_BF16, (int)T, 2 * c.vit_inter_pad, H, b.gateup_b, FO1_BF16,
                   FO1_EPI_SILU, nullptr, 0, 1, s));
    FO1_RUN(linear(hbuf, c.vit_inter_pad, b.down_w, c.vit_inter_pad, x, H, FO1_BF16, (int)T, H, c.vit_inter_pad, b.down_b, FO1_BF16,
                   FO1_EPI_NONE, x2, H, 0, s));
    if (full && taps != nullptr && taps[tap_i] != nullptr) {
      // un-window on the way out: token j of the packed sequence lands on pixel pix[j] of its image's map
      FO1_RUN(scatter_rows_bf16(x, H, d_pix, static_cast<bf16*>(taps[tap_i]), H, (int)T, H, s));
    }
    if (full) ++tap_i;
  }
  // ---- merger (:146-159) + inverse window permutation (:155-156) ----
  FO1_RUN(rmsnorm(x, H, w.ln_q, xn, H, (int)T, H, 1e-6f, s));
  const int M4 = H * unit;
  FO1_RUN(linear(xn, M4, w.fc1_w, M4, mg, M4, FO1_BF16, Tm, M4, M4, w.fc1_b, FO1_BF16, FO1_EPI_GELU, nullptr, 0, 0, s));
  FO1_RUN(linear(mg, M4, w.fc2_w, M4, mo, c.vit_out_hidden, FO1_BF16, Tm, c.vit_out_hidden, M4, w.fc2_b, FO1_BF16, FO1_EPI_NONE,
                 nullptr, 0, 0, s));
  FO1_RUN(scatter_rows_bf16(mo, c.vit_out_hidden, d_unperm, img_feats, c.vit_out_hidden, Tm, c.vit_out_hidden, s));
  return FO1_OK;
}

int vit_forward(Model* m, const float* const* pixel_values, const int32_t* grid_hw, int B, void* img_feats, void* const* taps,
                cudaStream_t s) {
  FO1_CHECK_ARG(m->vit.ok, "fo1_vit_forward: model not finalized (ViT weights unresolved)");
  const fo1_model_config& c = m->cfg;
  for (int b = 0; b < B; ++b) {
    const int gh = grid_hw[2 * b], gw = grid_hw[2 * b + 1];
    FO1_CHECK_ARG(gh > 0 && gw > 0 && gh % c.vit_merge == 0 && gw % c.vit_merge == 0, "image %d: grid %dx%d not a multiple of merge %d", b, gh, gw, c.vit_merge);
    FO1_CHECK_ARG(pixel_values[b] != nullptr, "image %d: null pixel_values", b);
  }
  FO1_TRY(int_cache_trim(m));
  m->arena.reset(true);
  FO1_TRY(vit_forward_impl(m, pixel_values, grid_hw, B, nullptr, nullptr, s, true));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  return vit_forward_impl(m, pixel_values, grid_hw, B, static_cast<bf16*>(img_feats), taps, s, false);
}

}  // namespace fo1

using namespace fo1;

extern "C" int fo1_vit_forward(fo1_model* m, const float* const* pixel_values, const int32_t* grid_hw, int32_t n_images,
                               void* img_feats, void* const* taps, void* stream) {
  FO1_CHECK_ARG(m && pixel_values && grid_hw && img_feats, "fo1_vit_forward: null argument");
  if (n_images <= 0) return FO1_OK;
  return vit_forward(m, pixel_values, grid_hw, n_images, img_feats, taps, static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_vit_window_index(const fo1_model_config* cfg, int32_t gh, int32_t gw, int32_t* window_index,
                                    int32_t* cu_window_seqlens, int32_t* n_cu, int32_t* pos_hw) {
  FO1_CHECK_ARG(cfg && window_index && cu_window_seqlens && n_cu && pos_hw, "fo1_vit_window_index: null argument");
  FO1_CHECK_ARG(gh > 0 && gw > 0 && gh % cfg->vit_merge == 0 && gw % cfg->vit_merge == 0, "fo1_vit_window_index: bad grid %dx%d", gh, gw);
  std::vector<int> wi, cw, ph;
  vit_window_index_host(*cfg, gh, gw, wi, cw, ph);
  memcpy(window_index, wi.data(), wi.size() * sizeof(int));
  memcpy(cu_window_seqlens, cw.data(), cw.size() * sizeof(int));
  *n_cu = (int)cw.size();
  memcpy(pos_hw, ph.data(), ph.size() * sizeof(int));
  return FO1_OK;
}
