// davit.cu -- aux perception tower (DaViT, Florence-2 vision backbone), SimpleFPN and the projector MLPs.
//
// DaViT.forward_features (modeling_davit.py:478-506): 4 stages of [ConvEmbed -> depth x (SpatialBlock,
// ChannelBlock)], each stage's token map returned.  Tokens stay channels-last [B*H*W][C] bf16 throughout
// (the reference bounces between NCHW and token layouts at every depth-wise conv, :91-99); dense convs are
// im2col + wgmma GEMM; LayerNorm / depth-wise conv / window (un)partition / channel attention are
// memory-bound SIMT kernels; biases, GELU and residual adds ride in the GEMM epilogues.
#include "engine.cuh"

namespace fo1 {

static int davit_resolve(Model* m) {
  const fo1_model_config& c = m->cfg;
  WeightGetter g{m, ""};
  for (int s = 0; s < 4; ++s) {
    DavitStageW& st = m->davit.st[s];
    const int64_t C = c.davit_dims[s], Cin = s == 0 ? 3 : c.davit_dims[s - 1];
    const int64_t K = s == 0 ? 152 : 9 * Cin;
    const std::string p = "davit.s" + std::to_string(s) + ".";
    st.conv_w = g.bf(p + "conv.w", {C, K});
    st.conv_b = g.bf(p + "conv.b", {C});
    const int64_t nd = s == 0 ? C : Cin;  // patch_prenorm = (False, True, True, True): davit/configs.py:111-116
    st.norm_w = g.bf(p + "norm.w", {nd});
    st.norm_b = g.bf(p + "norm.b", {nd});
    st.sp.resize(c.davit_depths[s]);
    st.ch.resize(c.davit_depths[s]);
    for (int j = 0; j < c.davit_depths[s]; ++j) {
      for (int half = 0; half < 2; ++half) {
        DavitHalfW& h = half ? st.ch[j] : st.sp[j];
        const std::string q = p + "b" + std::to_string(j) + (half ? ".ch." : ".sp.");
        h.conv1_w9 = g.bf(q + "conv1.w9", {9, C}); h.conv1_b = g.bf(q + "conv1.b", {C});
        h.norm1_w = g.bf(q + "norm1.w", {C}); h.norm1_b = g.bf(q + "norm1.b", {C});
        h.qkv_w = g.bf(q + "qkv.w", {3 * C, C}); h.qkv_b = g.bf(q + "qkv.b", {3 * C});
        h.proj_w = g.bf(q + "proj.w", {C, C}); h.proj_b = g.bf(q + "proj.b", {C});
        h.conv2_w9 = g.bf(q + "conv2.w9", {9, C}); h.conv2_b = g.bf(q + "conv2.b", {C});
        h.norm2_w = g.bf(q + "norm2.w", {C}); h.norm2_b = g.bf(q + "norm2.b", {C});
        h.fc1_w = g.bf(q + "fc1.w", {4 * C, C}); h.fc1_b = g.bf(q + "fc1.b", {4 * C});
        h.fc2_w = g.bf(q + "fc2.w", {C, 4 * C}); h.fc2_b = g.bf(q + "fc2.b", {C});
      }
    }
  }
  if (!g.err.empty()) { set_error("DaViT weights: %s", g.err.c_str()); return FO1_ERR_NOT_FOUND; }
  m->davit.ok = true;
  return FO1_OK;
}
int davit_finalize(Model* m) { return m->cfg.davit_dims[0] > 0 ? davit_resolve(m) : FO1_OK; }

static int davit_forward_impl(Model* m, const float* const* images, int H0, int W0, int B, void* const* stage_out, cudaStream_t s,
                              bool dry) {
  const fo1_model_config& c = m->cfg;
  Arena& A = m->arena;
  const int ws = c.davit_window;
  const float eps = 1e-5f;
  // stage geometry
  int Hs[4], Ws[4];
  Hs[0] = (H0 + 6 - 7) / 4 + 1; Ws[0] = (W0 + 6 - 7) / 4 + 1;
  for (int i = 1; i < 4; ++i) { Hs[i] = (Hs[i - 1] + 2 - 3) / 2 + 1; Ws[i] = (Ws[i - 1] + 2 - 3) / 2 + 1; }
  // buffer sizes: maxima over stages
  size_t max_tc = 0, max_wtc = 0, max_col = 0;
  for (int i = 0; i < 4; ++i) {
    const size_t tok = (size_t)B * Hs[i] * Ws[i], C = c.davit_dims[i];
    const size_t wtok = (size_t)B * ceil_div(Hs[i], ws) * ceil_div(Ws[i], ws) * ws * ws;
    max_tc = std::max(max_tc, tok * C);
    max_wtc = std::max(max_wtc, wtok * C);
    max_col = std::max(max_col, tok * (i == 0 ? (size_t)152 : (size_t)9 * c.davit_dims[i - 1]));
  }
  bf16* xa = A.alloc<bf16>(max_tc);
  bf16* xb = A.alloc<bf16>(max_tc);
  bf16* yb = A.alloc<bf16>(max_tc);
  bf16* wb = A.alloc<bf16>(max_wtc);       // partitioned LN output, later the proj output
  bf16* ao = A.alloc<bf16>(max_wtc);       // attention output
  bf16* qkv = A.alloc<bf16>(std::max(max_wtc, max_tc) * 3);
  bf16* hb = A.alloc<bf16>(max_tc * 4);
  bf16* col = A.alloc<bf16>(max_col);
  size_t gram_floats = 0;                  // partial Gram matrices of the channel attention (per token chunk, summed in fixed order)
  for (int i = 0; i < 4; ++i) gram_floats = std::max(gram_floats, channel_attention_ws_floats(B, Hs[i] * Ws[i], c.davit_dims[i]));
  float* gram = A.alloc<float>(gram_floats);

  bf16* x = xa;      // current token map
  bf16* xalt = xb;
  for (int st = 0; st < 4; ++st) {
    const DavitStageW& W = m->davit.st[st];
    const int C = c.davit_dims[st], Hh = Hs[st], Ww = Ws[st];
    const int tok = B * Hh * Ww;
    // ---- ConvEmbed (modeling_davit.py:102-148) ----
    if (st == 0) {
      const int per = Hh * Ww;
      for (int b = 0; b < B; ++b) FO1_RUN(im2col_stem(images[b], col + (size_t)b * per * 152, H0, W0, 152, s));
      FO1_RUN(linear(col, 152, W.conv_w, 152, yb, C, FO1_BF16, tok, C, 152, W.conv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
      FO1_RUN(layernorm(yb, C, W.norm_w, W.norm_b, x, C, tok, C, eps, s));
    } else {
      const int Cin = c.davit_dims[st - 1], Hp = Hs[st - 1], Wp = Ws[st - 1];
      FO1_RUN(layernorm(x, Cin, W.norm_w, W.norm_b, yb, Cin, B * Hp * Wp, Cin, eps, s));
      FO1_RUN(im2col3x3(yb, col, B, Hp, Wp, Cin, 2, s));
      FO1_RUN(linear(col, 9 * Cin, W.conv_w, 9 * Cin, x, C, FO1_BF16, tok, C, 9 * Cin, W.conv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
    }
    const int nwh = ceil_div(Hh, ws), nww = ceil_div(Ww, ws);
    const int n_win = B * nwh * nww, wtok = n_win * ws * ws;
    const int *d_cu = nullptr, *d_tiles = nullptr;
    int n_tiles = 0;
    if (!dry) {
      std::vector<int> cu(n_win + 1), img_cu(B + 1), tiles;
      for (int i = 0; i <= n_win; ++i) cu[i] = i * ws * ws;
      for (int b = 0; b <= B; ++b) img_cu[b] = b * nwh * nww * ws * ws;
      attention_tile_table(img_cu, tiles);    // query tiles restart at every image (its bits do not depend on the batch slot)
      n_tiles = (int)tiles.size() / 2;
      const std::string key = "dv:" + std::to_string(B) + ":" + std::to_string(nwh * nww) + ":" + std::to_string(ws);
      FO1_TRY(cached_ints(m, key + ":cu", cu, &d_cu, s));
      FO1_TRY(cached_ints(m, key + ":til", tiles, &d_tiles, s));
    }
    for (int j = 0; j < c.davit_depths[st]; ++j) {
      for (int half = 0; half < 2; ++half) {
        const DavitHalfW& h = half ? W.ch[j] : W.sp[j];
        // conv1: x <- x + dw3x3(x)
        FO1_RUN(dwconv3x3_residual(x, h.conv1_w9, h.conv1_b, xalt, B, Hh, Ww, C, s));
        std::swap(x, xalt);
        FO1_RUN(layernorm(x, C, h.norm1_w, h.norm1_b, yb, C, tok, C, eps, s));
        if (half == 0) {
          // SpatialBlock: window attention (:225-282)
          FO1_RUN(window_partition(yb, wb, B, Hh, Ww, C, ws, s));
          FO1_RUN(linear(wb, C, h.qkv_w, C, qkv, 3 * C, FO1_BF16, wtok, 3 * C, C, h.qkv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
          AttnArgs a;
          a.q = qkv; a.k = qkv + C; a.v = qkv + 2 * C; a.o = ao;
          a.ldq = a.ldk = a.ldv = 3 * C; a.ldo = C;
          a.cu_seqlens = d_cu; a.n_seqs = n_win; a.max_seqlen = ws * ws; a.total_rows = wtok; a.tiles = d_tiles; a.n_tiles = n_tiles;
          a.flops = 4.0 * wtok * (ws * ws) * C;
          a.q_heads = a.kv_heads = c.davit_heads[st]; a.head_dim = C / c.davit_heads[st];
          a.scale = 1.0f / sqrtf((float)a.head_dim); a.causal = 0;
          FO1_RUN(attention_varlen(a, s));
          FO1_RUN(linear(ao, C, h.proj_w, C, wb, C, FO1_BF16, wtok, C, C, h.proj_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
          FO1_RUN(window_reverse_add(x, wb, xalt, B, Hh, Ww, C, ws, s));
          std::swap(x, xalt);
        } else {
          // ChannelBlock: channel-group attention (:151-172)
          FO1_RUN(linear(yb, C, h.qkv_w, C, qkv, 3 * C, FO1_BF16, tok, 3 * C, C, h.qkv_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
          FO1_RUN(channel_attention(qkv, gram, ao, B, Hh * Ww, C, c.davit_groups[st], s));
          FO1_RUN(linear(ao, C, h.proj_w, C, xalt, C, FO1_BF16, tok, C, C, h.proj_b, FO1_BF16, FO1_EPI_NONE, x, C, 0, s));
          std::swap(x, xalt);
        }
        // conv2 + FFN
        FO1_RUN(dwconv3x3_residual(x, h.conv2_w9, h.conv2_b, xalt, B, Hh, Ww, C, s));
        std::swap(x, xalt);
        FO1_RUN(layernorm(x, C, h.norm2_w, h.norm2_b, yb, C, tok, C, eps, s));
        FO1_RUN(linear(yb, C, h.fc1_w, C, hb, 4 * C, FO1_BF16, tok, 4 * C, C, h.fc1_b, FO1_BF16, FO1_EPI_GELU, nullptr, 0, 0, s));
        FO1_RUN(linear(hb, 4 * C, h.fc2_w, 4 * C, xalt, C, FO1_BF16, tok, C, 4 * C, h.fc2_b, FO1_BF16, FO1_EPI_NONE, x, C, 0, s));
        std::swap(x, xalt);
      }
    }
    if (!dry && stage_out[st] != nullptr)
      FO1_CUDA(cudaMemcpyAsync(stage_out[st], x, (size_t)tok * C * sizeof(bf16), cudaMemcpyDeviceToDevice, s));
  }
  return FO1_OK;
}

int davit_forward(Model* m, const float* const* images, int H, int W, int B, void* const* stage_out, cudaStream_t s) {
  FO1_CHECK_ARG(m->davit.ok, "fo1_davit_forward: model not finalized (DaViT weights unresolved)");
  FO1_CHECK_ARG(H >= 32 && W >= 32, "fo1_davit_forward: image %dx%d too small", H, W);
  for (int i = 0; i < 4; ++i)
    FO1_CHECK_ARG(m->cfg.davit_dims[i] == 32 * m->cfg.davit_heads[i] && m->cfg.davit_dims[i] == 32 * m->cfg.davit_groups[i],
                  "DaViT stage %d: this engine needs 32 channels per head/group", i);
  FO1_TRY(int_cache_trim(m));
  m->arena.reset(true);
  FO1_TRY(davit_forward_impl(m, images, H, W, B, stage_out, s, true));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  return davit_forward_impl(m, images, H, W, B, stage_out, s, false);
}

// ------------------------------------------------------------------------------------------- SimpleFPN
static int fpn_resolve(Model* m) {
  const fo1_model_config& c = m->cfg;
  WeightGetter g{m, ""};
  FpnW& f = m->fpn;
  const int64_t D = c.vit_hidden, O = c.fpn_out;
  f.l0_dc1_w = g.bf("fpn.l0.deconv1.w", {4 * (D / 2), D}); f.l0_dc1_b = g.bf("fpn.l0.deconv1.b", {4 * (D / 2)});
  f.l0_ln_w = g.bf("fpn.l0.ln.w", {D / 2}); f.l0_ln_b = g.bf("fpn.l0.ln.b", {D / 2});
  f.l0_dc2_w = g.bf("fpn.l0.deconv2.w", {4 * (D / 4), D / 2}); f.l0_dc2_b = g.bf("fpn.l0.deconv2.b", {4 * (D / 4)});
  f.l1_dc_w = g.bf("fpn.l1.deconv1.w", {4 * (D / 2), D}); f.l1_dc_b = g.bf("fpn.l1.deconv1.b", {4 * (D / 2)});
  const int64_t cin[4] = {D / 4, D / 2, D, D};
  for (int l = 0; l < 4; ++l) {
    const std::string p = "fpn.l" + std::to_string(l) + ".";
    f.lv[l].conv1_w = g.bf(p + "conv1.w", {O, cin[l]});
    f.lv[l].ln1_w = g.bf(p + "ln1.w", {O}); f.lv[l].ln1_b = g.bf(p + "ln1.b", {O});
    f.lv[l].conv2_w = g.bf(p + "conv2.w", {O, 9 * O});
    f.lv[l].ln2_w = g.bf(p + "ln2.w", {O}); f.lv[l].ln2_b = g.bf(p + "ln2.b", {O});
  }
  if (!g.err.empty()) { set_error("SimpleFPN weights: %s", g.err.c_str()); return FO1_ERR_NOT_FOUND; }
  f.ok = true;
  return FO1_OK;
}
int fpn_finalize(Model* m) { return m->cfg.fpn_out > 0 ? fpn_resolve(m) : FO1_OK; }

static int fpn_forward_impl(Model* m, const bf16* tap, int gh, int gw, int B, void* const* level_out, cudaStream_t s, bool dry) {
  const fo1_model_config& c = m->cfg;
  const FpnW& f = m->fpn;
  Arena& A = m->arena;
  const int D = c.vit_hidden, O = c.fpn_out;
  const float eps = 1e-6f;  // simple_fpn.py:66
  const size_t px = (size_t)B * gh * gw;
  // the 3x3 conv's im2col is chunked over images so the column buffer stays bounded
  const size_t col_budget = (size_t)3 << 30;
  for (int l = 0; l < 4; ++l) {
    const size_t mark = A.mark();
    const int Hl = l == 0 ? gh * 4 : (l == 1 ? gh * 2 : (l == 2 ? gh : gh / 2));
    const int Wl = l == 0 ? gw * 4 : (l == 1 ? gw * 2 : (l == 2 ? gw : gw / 2));
    const size_t pl = (size_t)B * Hl * Wl;
    const bf16* feat = tap;
    int Cin = D;
    if (l == 0) {
      bf16* g1 = A.alloc<bf16>(px * 4 * (D / 2));
      bf16* u1 = A.alloc<bf16>(px * 4 * (D / 2));
      FO1_RUN(linear(tap, D, f.l0_dc1_w, D, g1, 4 * (D / 2), FO1_BF16, (int)px, 4 * (D / 2), D, f.l0_dc1_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
      FO1_RUN(pixel_shuffle2x(g1, u1, B, gh, gw, D / 2, s));
      FO1_RUN(layernorm(u1, D / 2, f.l0_ln_w, f.l0_ln_b, g1, D / 2, (int)(px * 4), D / 2, eps, s));
      FO1_RUN(gelu_bf16(g1, g1, (long long)px * 4 * (D / 2), s));
      bf16* g2 = A.alloc<bf16>(px * 16 * (D / 4));
      bf16* u2 = A.alloc<bf16>(px * 16 * (D / 4));
      FO1_RUN(linear(g1, D / 2, f.l0_dc2_w, D / 2, g2, 4 * (D / 4), FO1_BF16, (int)(px * 4), 4 * (D / 4), D / 2, f.l0_dc2_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
      FO1_RUN(pixel_shuffle2x(g2, u2, B, gh * 2, gw * 2, D / 4, s));
      feat = u2; Cin = D / 4;
    } else if (l == 1) {
      bf16* g1 = A.alloc<bf16>(px * 4 * (D / 2));
      bf16* u1 = A.alloc<bf16>(px * 4 * (D / 2));
      FO1_RUN(linear(tap, D, f.l1_dc_w, D, g1, 4 * (D / 2), FO1_BF16, (int)px, 4 * (D / 2), D, f.l1_dc_b, FO1_BF16, FO1_EPI_NONE, nullptr, 0, 0, s));
      FO1_RUN(pixel_shuffle2x(g1, u1, B, gh, gw, D / 2, s));
      feat = u1; Cin = D / 2;
    } else if (l == 3) {
      bf16* mp = A.alloc<bf16>(pl * D);
      FO1_RUN(maxpool2x2(tap, mp, B, gh, gw, D, s));
      feat = mp;
    }
    bf16* t1 = A.alloc<bf16>(pl * O);
    bf16* t2 = A.alloc<bf16>(pl * O);
    FO1_RUN(linear(feat, Cin, f.lv[l].conv1_w, Cin, t1, O, FO1_BF16, (int)pl, O, Cin, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
    FO1_RUN(layernorm(t1, O, f.lv[l].ln1_w, f.lv[l].ln1_b, t2, O, (int)pl, O, eps, s));
    // 3x3 conv: implicit GEMM (the A tiles are TMA patches of t2, zero padding by the out-of-range fill); shapes that do not
    // tile into 128-pixel patches -- or FO1_FPN_IM2COL, the A/B knob of the parity test -- take im2col + linear
    const bool force_im2col = getenv("FO1_FPN_IM2COL") != nullptr;
    int crc = -1000;
    if (!force_im2col) {
      if (dry) crc = ((O % 64 == 0) && ((size_t)Hl * Wl) % 128 == 0 && ((Wl % 128 == 0) || (128 % Wl == 0 && Hl % (128 / Wl) == 0))) ? FO1_OK : -1000;
      else crc = conv3x3_gemm(t2, B, Hl, Wl, O, f.lv[l].conv2_w, t1, O, O, s);
      if (crc != FO1_OK && crc != -1000) return crc;
    }
    if (crc == -1000) {
      const size_t per_img_col = (size_t)Hl * Wl * 9 * O * sizeof(bf16);
      int chunk = (int)std::max<size_t>(1, col_budget / std::max<size_t>(per_img_col, 1));
      chunk = std::min(chunk, B);
      bf16* colb = A.alloc<bf16>((size_t)chunk * Hl * Wl * 9 * O);
      for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = std::min(chunk, B - b0);
        const size_t o = (size_t)b0 * Hl * Wl;
        FO1_RUN(im2col3x3(t2 + o * O, colb, nb, Hl, Wl, O, 1, s));
        FO1_RUN(linear(colb, 9 * O, f.lv[l].conv2_w, 9 * O, t1 + o * O, O, FO1_BF16, nb * Hl * Wl, O, 9 * O, nullptr, 0, FO1_EPI_NONE, nullptr, 0, 0, s));
      }
    }
    FO1_RUN(layernorm(t1, O, f.lv[l].ln2_w, f.lv[l].ln2_b, static_cast<bf16*>(dry ? nullptr : level_out[l]), O, (int)pl, O, eps, s));
    A.release(mark);
  }
  return FO1_OK;
}

int fpn_forward(Model* m, const void* tap, int gh, int gw, int B, void* const* level_out, cudaStream_t s) {
  FO1_CHECK_ARG(m->fpn.ok, "fo1_fpn_forward: model not finalized (SimpleFPN weights unresolved)");
  FO1_CHECK_ARG(gh % 2 == 0 && gw % 2 == 0, "fo1_fpn_forward: grid %dx%d must be even", gh, gw);
  FO1_TRY(int_cache_trim(m));
  m->arena.reset(true);
  FO1_TRY(fpn_forward_impl(m, static_cast<const bf16*>(tap), gh, gw, B, level_out, s, true));
  FO1_TRY(arena_ensure(m, m->arena.peak));
  m->arena.reset(false);
  return fpn_forward_impl(m, static_cast<const bf16*>(tap), gh, gw, B, level_out, s, false);
}

// ------------------------------------------------------------------------------------------- projectors
static int proj_resolve_one(Model* m, ProjW& P, const char* prefix, int layers, int in_dim, int hidden) {
  WeightGetter g{m, ""};
  P.w.clear(); P.b.clear(); P.in_dim.clear(); P.out_dim.clear();
  for (int k = 0; k < layers; ++k) {
    const int64_t in = k == 0 ? in_dim : hidden;
    const std::string p = std::string(prefix) + "." + std::to_string(k) + ".";
    P.w.push_back(g.bf(p + "w", {(int64_t)hidden, in}));
    P.b.push_back(g.bf(p + "b", {(int64_t)hidden}));
    P.in_dim.push_back((int)in);
    P.out_dim.push_back(hidden);
  }
  if (!g.err.empty()) { set_error("projector weights: %s", g.err.c_str()); return FO1_ERR_NOT_FOUND; }
  P.ok = true;
  return FO1_OK;
}
int proj_finalize(Model* m) {
  const fo1_model_config& c = m->cfg;
  if (c.proj_aux_layers > 0) FO1_TRY(proj_resolve_one(m, m->proj_aux, "proj_aux", c.proj_aux_layers, c.region_dim, c.llm_hidden));
  if (c.proj_img_layers > 0) FO1_TRY(proj_resolve_one(m, m->proj_img, "proj_img", c.proj_img_layers, c.vit_out_hidden, c.llm_hidden));
  return FO1_OK;
}

int project(Model* m, const ProjW& P, const bf16* in, int n, bf16* out, cudaStream_t s) {
  FO1_CHECK_ARG(P.ok, "projector not finalized");
  if (n == 0) return FO1_OK;
  const int L = (int)P.w.size();
  size_t need = 0;
  for (int k = 0; k + 1 < L; ++k) need = std::max(need, (size_t)n * P.out_dim[k] * sizeof(bf16));
  FO1_TRY(arena_ensure(m, 2 * need + 1024));
  m->arena.reset(false);
  bf16* t[2] = {m->arena.alloc<bf16>(need / sizeof(bf16) + 8), m->arena.alloc<bf16>(need / sizeof(bf16) + 8)};
  const bf16* cur = in;
  for (int k = 0; k < L; ++k) {
    bf16* dst = (k == L - 1) ? out : t[k & 1];
    // mlpNx_gelu: Linear [GELU Linear]... (builder.py:100-106): GELU follows every layer but the last
    FO1_TRY(linear(cur, P.in_dim[k], P.w[k], P.in_dim[k], dst, P.out_dim[k], FO1_BF16, n, P.out_dim[k], P.in_dim[k], P.b[k], FO1_BF16,
                   k == L - 1 ? FO1_EPI_NONE : FO1_EPI_GELU, nullptr, 0, 0, s));
    cur = dst;
  }
  return FO1_OK;
}

}  // namespace fo1

using namespace fo1;

extern "C" int fo1_davit_forward(fo1_model* m, const float* const* images, int32_t H, int32_t W, int32_t n_images,
                                 void* const* stage_out, void* stream) {
  FO1_CHECK_ARG(m && images && stage_out, "fo1_davit_forward: null argument");
  if (n_images <= 0) return FO1_OK;
  return davit_forward(m, images, H, W, n_images, stage_out, static_cast<cudaStream_t>(stream));
}
extern "C" int fo1_fpn_forward(fo1_model* m, const void* tap, int32_t gh, int32_t gw, int32_t n_images, void* const* level_out,
                               void* stream) {
  FO1_CHECK_ARG(m && tap && level_out, "fo1_fpn_forward: null argument");
  if (n_images <= 0) return FO1_OK;
  return fpn_forward(m, tap, gh, gw, n_images, level_out, static_cast<cudaStream_t>(stream));
}
extern "C" int fo1_image_project(fo1_model* m, const void* feats, int32_t n, void* out, void* stream) {
  FO1_CHECK_ARG(m && (n == 0 || (feats && out)), "fo1_image_project: null argument");
  FO1_CHECK_ARG(m->cfg.proj_img_layers > 0, "fo1_image_project: mm_projector is the identity for this model (proj_img_layers = 0)");
  return project(m, m->proj_img, static_cast<const bf16*>(feats), n, static_cast<bf16*>(out), static_cast<cudaStream_t>(stream));
}

extern "C" int fo1_region_project(fo1_model* m, const void* feats, int32_t n, void* out, void* stream) {
  FO1_CHECK_ARG(m && (n == 0 || (feats && out)), "fo1_region_project: null argument");
  return project(m, m->proj_aux, static_cast<const bf16*>(feats), n, static_cast<bf16*>(out), static_cast<cudaStream_t>(stream));
}
extern "C" int fo1_model_finalize(fo1_model* m) {
  FO1_CHECK_ARG(m, "fo1_model_finalize: null model");
  FO1_TRY(vit_finalize(m));
  FO1_TRY(davit_finalize(m));
  FO1_TRY(fpn_finalize(m));
  FO1_TRY(proj_finalize(m));
  FO1_TRY(llm_finalize(m));
  m->finalized = true;
  return FO1_OK;
}
