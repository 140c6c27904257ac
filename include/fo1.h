/*
 * fo1.h -- C ABI of libfo1.so, the H100 (sm_90a) engine for the VLM-FO1 inference hot path.
 *
 * Plain C types only: device pointers, sizes, a cudaStream_t passed as void*.  Every entry point
 * returns 0 on success or a negative fo1_status; fo1_last_error() returns a message for the calling
 * thread.  Nothing here allocates on the hot path: callers own inputs/outputs and hand the library a
 * workspace; the model-level handle owns its weights and one arena sized when the model is created.
 * All entry points enqueue on the given stream and return (asynchronous) unless stated otherwise.
 *
 * Each declaration cites the reference interface (om-ai-lab/VLM-FO1 @ e6bef8d) it replaces.
 * The reference has no FFI of its own (pure PyTorch); INTEGRATION.md shows the ctypes binding a
 * maintainer adds under vlm_fo1/model/.
 */
#ifndef FO1_H_
#define FO1_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FO1_ABI_VERSION 4

typedef enum {
  FO1_OK = 0,
  FO1_ERR_INVALID_ARG = -1,
  FO1_ERR_CUDA = -2,
  FO1_ERR_UNSUPPORTED = -3,
  FO1_ERR_WORKSPACE = -4,
  FO1_ERR_NOT_FOUND = -5,
  FO1_ERR_STATE = -6
} fo1_status;

typedef enum { FO1_BF16 = 0, FO1_F32 = 1, FO1_I32 = 2, FO1_I64 = 3, FO1_U8 = 4, FO1_F16 = 5 } fo1_dtype;

int fo1_abi_version(void);
/* Message describing the last failure on this thread ("" if none). */
const char* fo1_last_error(void);
/* Number of kernels this library has launched since load / since the last reset (all threads). */
uint64_t fo1_launch_count(void);
void fo1_launch_count_reset(void);
/* Optional per-launch profiler: CUDA events recorded around the library's GEMM / attention / HFRE launches on
 * the launching stream.  enable(1) clears and starts recording, enable(0) stops; collect() synchronises the
 * device and writes a JSON object {tag: {launches, ms, flops, bytes, max_ms}} (algorithmic flops / bytes). */
void fo1_profile_enable(int on);
int fo1_profile_collect(char* buf, size_t cap);

/* ------------------------------------------------------------------------------------------------
 * HFRE -- Hybrid Fine-grained Region Encoder.
 * Replaces HFREModule.__call__ (vlm_fo1/model/multimodal_visual_prompt_encoder/
 * hybrid_finegrained_region_encoder.py:275-468) as called from encode_regions
 * (vlm_fo1/model/language_model/omchat_qwen2_5_vl.py:101-106): ROIAlign(7x7, adaptive sampling,
 * aligned=False) + mean over bins on every pyramid level of both towers, channel concat, and the
 * sinusoidal box embedding -- WITHOUT materialising the up-sampled/concatenated map (:338-350).
 * ---------------------------------------------------------------------------------------------- */

/* One feature level: bf16, channels-last [H][W][C] in device memory, C % 8 == 0, 16-byte aligned. */
typedef struct {
  const void* data;
  int32_t H, W, C;
  int32_t up_H, up_W;     /* grid the reference bilinearly up-samples this level to before ROIAlign
                             (F.interpolate align_corners=False, :341-346); == H, W when it does not */
  float spatial_scale;    /* ROIAlign spatial_scale on that (up-sampled) grid: 0.25 aux (:357),
                             1/14 taps (:267), 1/3.5 .. 1/28 FPN (:245-253) */
  int32_t box_set;        /* 0: aux boxes, 1: primary-tower ("vt") boxes */
  int32_t out_offset;     /* first output channel written by this level */
} fo1_hfre_level;

#define FO1_HFRE_MAX_LEVELS 8

/* One image's work. */
typedef struct {
  fo1_hfre_level levels[FO1_HFRE_MAX_LEVELS];
  int32_t n_levels;
  int32_t n_boxes;
  const float* boxes_aux;  /* [n_boxes][4] xyxy, aux-tensor pixels (device) */
  const float* boxes_vt;   /* [n_boxes][4] xyxy, primary-tower pixels (device); may equal boxes_aux */
  float* out;              /* [n_boxes][out_dim] fp32 (device) */
  void* out_bf16;          /* optional [n_boxes][out_dim] bf16 copy for the projector GEMM, or NULL */
  float pos_img_w, pos_img_h; /* normaliser of the box embedding (:447-448): grid * 14 */
  int32_t pos_box_set;     /* which boxes feed the embedding (:442-452): 1 = vt */
} fo1_hfre_image;

typedef struct {
  int32_t out_dim;          /* D = mm_region_hidden_size (5888 variant B, 8960 variant A) */
  int32_t roi_size;         /* 7 (omchat_arch.py:18) */
  int32_t apply_pos_embed;  /* mm_apply_position_embedding, bbox_based */
} fo1_hfre_params;

/* Bytes of device workspace fo1_hfre_forward needs for these images (host-side arithmetic only). */
size_t fo1_hfre_workspace_bytes(const fo1_hfre_image* images, int32_t n_images, const fo1_hfre_params* p);
/* Enqueue HFRE for n_images images.  `images` is a HOST array (device pointers inside). */
int fo1_hfre_forward(const fo1_hfre_image* images, int32_t n_images, const fo1_hfre_params* p,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense contraction: D[M,N] = epilogue(A[M,K] . W[N,K]^T) -- bf16 operands, fp32 accumulate in registers
 * (wgmma, operands staged by TMA).  Replaces every nn.Linear / 1x1 conv / patch-embed on the
 * path (modeling_qwen2_5_vl.py:88-111, 176-177, 151-155, 731-734, 633-635; modeling_davit.py:62-66,
 * 157-158, 235-236; simple_fpn.py:143-175; multimodal_projector/builder.py:100-106).
 * ---------------------------------------------------------------------------------------------- */
typedef enum {
  FO1_EPI_NONE = 0,
  FO1_EPI_GELU = 1,          /* exact erf GELU (nn.GELU default) */
  FO1_EPI_SILU = 2
} fo1_epilogue_act;

typedef struct {
  int32_t M, N, K;
  const void* A; int64_t lda;      /* bf16 [M][K], row stride lda elements (lda*2 % 16 == 0) */
  const void* W; int64_t ldw;      /* bf16 [N][K] (nn.Linear weight layout) */
  void* D; int64_t ldd;            /* output [M][N], bf16 or fp32 */
  int32_t d_dtype;                 /* FO1_BF16 or FO1_F32 */
  const void* bias;                /* optional [N], bias_dtype */
  int32_t bias_dtype;              /* FO1_BF16 or FO1_F32 */
  int32_t act;                     /* fo1_epilogue_act, applied after bias */
  const void* residual; int64_t ldr; /* optional bf16 [M][N] added after act */
  int32_t gated;                   /* 1: W rows interleave [32 gate | 32 up] blocks -> D[M][N/2] =
                                      act(gate)*up  (Qwen2MLP, modeling_qwen2_5_vl.py:84-85,638-640) */
  int32_t tile_n;                  /* 0 = library heuristic; 32 / 64 / 128 / 256 pins the tile width (tuning, tests) */
  int32_t split_k;                 /* with tile_n != 0: number of K splits reduced in-kernel (>= 1); 0 = 1 */
} fo1_gemm_desc;

int fo1_gemm_bf16(const fo1_gemm_desc* d, void* stream);



/* ------------------------------------------------------------------------------------------------
 * Variable-length softmax attention over packed token rows (replaces flash_attn_varlen_func at
 * modeling_qwen2_5_vl.py:205 and _flash_attention_forward at :895, and DaViT's window attention
 * modeling_davit.py:261-268) on wgmma with TMA-fed K/V rings.  q/k/v/o: bf16 rows with the given
 * pitches (elements, multiples of 8; 16-byte aligned bases); head h of a row starts at h*head_dim.
 * cu_seqlens: device int32 [n_seqs+1]; total_rows = cu_seqlens[n_seqs] (the host passes it: it sizes the grid).
 * head_dim in {32, 64, 80, 128}.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const void* q; const void* k; const void* v; void* o;
  int64_t ldq, ldk, ldv, ldo;
  const int32_t* cu_seqlens;
  int32_t n_seqs, max_seqlen;
  int32_t q_heads, kv_heads, head_dim;
  float scale;
  int32_t causal;
  int32_t total_rows;
} fo1_attn_desc;
int fo1_attention_varlen(const fo1_attn_desc* d, void* stream);

/* DaViT channel-group attention (ChannelAttention.forward, modeling_davit.py:151-172) for n_images maps of n_tokens tokens:
 * qkv bf16 [n_images][n_tokens][3*channels] (q | k | v as the fused Linear emits them), groups * 32 == channels;
 * out bf16 [n_images][n_tokens][channels] = (softmax_c2((q N^-0.5)^T k) v^T)^T per group of 32 channels.  Both contractions
 * run on wgmma (the Gram over the token axis with MN-major operands straight from the TMA tiles); partial Grams of the
 * token chunks live in `workspace` and are summed in a fixed order (bit-reproducible, no atomics). */
size_t fo1_channel_attention_workspace_bytes(int32_t n_images, int32_t n_tokens, int32_t channels);
int fo1_channel_attention(const void* qkv, int32_t n_images, int32_t n_tokens, int32_t channels, int32_t groups, void* out,
                          void* workspace, size_t workspace_bytes, void* stream);

/* DaViT conditional position encoding (PreNorm(None, DepthWiseConv2d), modeling_davit.py:29-48, 72-99): y = x + dwconv3x3(x) + bias over
 * NHWC bf16 maps [n_images][height][width][channels]; w9 bf16 [9][channels] (tap-major repack of [channels][1][3][3]), bias bf16
 * [channels].  channels % 8 == 0; x and y must not alias.  Exposed for the parity test of the kernel; fo1_davit_forward runs the same code. */
int fo1_dwconv3x3_residual(const void* x, const void* w9, const void* bias, void* y, int32_t n_images, int32_t height, int32_t width,
                           int32_t channels, void* stream);

/* Row normalisation of bf16 rows x [rows][cols] (pitch ldx) into y (pitch ldy): rms = 1 is Qwen2RMSNorm (modeling_qwen2_5_vl.py:126-140,
 * the normalised value rounded to bf16 before the gain; beta must be NULL), rms = 0 is nn.LayerNorm (fp32 two-pass statistics).
 * gamma / beta bf16 [cols] or NULL (1 / 0).  cols and pitches multiples of 8, cols <= 8192; 16-byte aligned pointers.
 * kernel 0: one warp per row (what the towers and the prefill layers run); kernel 1: one block per row, cols <= 4096 (what the decode
 * steps and the prefill's last rows run).  Exposed for the parity test of the two kernels; the engine names one per call site. */
int fo1_row_norm(const void* x, int64_t ldx, const void* gamma, const void* beta, void* y, int64_t ldy, int32_t rows, int32_t cols,
                 float eps, int32_t rms, int32_t kernel, void* stream);

/* Single-query GQA attention of one decode step over the K/V cache (the per-step attention of the HF generate loop,
 * modeling_qwen2_5_vl.py:731-780 with past_key_values; mm_utils.py:640-654 drives it).  The step's own K/V must already
 * sit in the cache at index cache_len[b].  head_dim 128, q_heads / kv_heads <= 8.  Exposed so the parity tests can
 * check the kernel directly; fo1_llm_generate runs the same code. */
typedef struct {
  const void* q; int64_t ldq;        /* bf16 [n_seqs][q_heads*128] (rotated), row stride ldq elements */
  const void* k_cache;               /* bf16 [n_seqs][cap][kv_heads*128] */
  const void* v_cache;
  const int32_t* cache_len;          /* device [n_seqs]: keys 0 .. cache_len[b] (inclusive) are attended */
  int32_t n_seqs, cap, q_heads, kv_heads, head_dim;
  float scale;
  void* out; int64_t ldo;            /* bf16 [n_seqs][q_heads*128] */
  void* workspace;                   /* fp32 partials, fo1_decode_attention_workspace_bytes(n_seqs, q_heads) */
  size_t workspace_bytes;
} fo1_decode_attn_desc;
size_t fo1_decode_attention_workspace_bytes(int32_t n_seqs, int32_t q_heads);
int fo1_decode_attention(const fo1_decode_attn_desc* d, void* stream);

/* Causal attention of a sequence's own rows against its K/V cache, the attention of fo1_llm_generate with d.prefix: own row i of
 * sequence b (query row own_off_b + i of q, own rows of the sequences packed in order) attends the cache keys 0 .. P_b + i of b.
 * Its own K/V must already sit in the cache at row P_b + i.  Key tiles start at key 0 of the sequence, as in the full-sequence
 * prefill, so each row's output is bit-identical to what fo1_attention_varlen (causal) gives that row over the whole sequence.
 * The cache rows P_b + own_b .. up to the next multiple of 64 are read with weight zero and must hold finite values.
 * head_dim 128.  Exposed so the kernel can be checked on its own. */
typedef struct {
  const void* q; int64_t ldq;        /* bf16 [sum own_b][ldq], rotated */
  const void* k_cache;               /* bf16 [n_seqs][cap][kv_heads*head_dim] */
  const void* v_cache;
  int32_t n_seqs, cap;               /* cap: a multiple of 64 */
  const int32_t* prefix_lens;        /* HOST [n_seqs]: P_b >= 0 */
  const int32_t* own_lens;           /* HOST [n_seqs]: own_b >= 0, P_b + own_b <= cap */
  int32_t q_heads, kv_heads, head_dim;
  float scale;
  void* out; int64_t ldo;            /* bf16 [sum own_b][ldo] */
} fo1_prefix_attn_desc;
int fo1_prefix_attention(const fo1_prefix_attn_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Model-level engine.  One handle per GPU / rank; calls on one handle are not re-entrant.
 * Weights are BORROWED device pointers (the caller keeps them alive): the Python loader prepares
 * them once (layout changes listed in DESIGN.md section "weights") from the checkpoint tensors that
 * vlm_fo1/model/builder.py:90-131 loads.
 * ---------------------------------------------------------------------------------------------- */
typedef struct fo1_model fo1_model;

typedef struct {
  /* primary tower: Qwen2.5-VL ViT (configuration_qwen2_5_vl.py:30-66) */
  int32_t vit_depth, vit_hidden, vit_heads, vit_inter, vit_inter_pad, vit_out_hidden;
  int32_t vit_patch, vit_merge, vit_temporal, vit_in_ch, vit_window;
  int32_t vit_n_fullatt; int32_t vit_fullatt[8];   /* fullatt_block_indexes, also the tap layers */
  /* aux tower: DaViT (davit/configs.py:70-136) */
  int32_t davit_dims[4], davit_depths[4], davit_heads[4], davit_groups[4], davit_window;
  /* SimpleFPN on the last tap (simple_fpn.py:100-216) */
  int32_t fpn_out;                 /* 512; 0 = FPN absent (variant A) */
  /* region projector / image projector (multimodal_projector/builder.py:39-115) */
  int32_t region_dim;              /* mm_region_hidden_size */
  int32_t proj_aux_layers;         /* mlpNx_gelu depth; 1 = linear */
  int32_t proj_img_layers;         /* 0 = identity */
  /* LLM: Qwen2.5 decoder (configuration_qwen2_5_vl.py:193-253) */
  int32_t llm_layers, llm_hidden, llm_heads, llm_kv_heads, llm_head_dim, llm_inter, llm_vocab;
  int32_t mrope_section[3];
  float rope_theta, rms_eps;
  int32_t tie_embeddings;
} fo1_model_config;

int fo1_model_create(const fo1_model_config* cfg, fo1_model** out);
/* Entries of the handle's cache of device-side integer tables (window indices, cu_seqlens ...).  The cache is trimmed
 * only at the entry of a forward, never while one is using its tables; exposed for the test of that rule. */
int fo1_int_cache_entries(fo1_model* m);
/* Which decode path the handle's last fo1_generate took: 1 = the persistent kernel (decode_mega.cu, the whole greedy loop as one
 * cooperative launch), 0 = the per-kernel CUDA graph, -1 = no generate yet.  Reported by bench.py next to the decode roofline. */
int fo1_last_decode_path(fo1_model* m);
void fo1_model_destroy(fo1_model* m);
/* Register one prepared weight (device pointer, borrowed).  Names: see DESIGN.md / vlm-fo1_b200/weights.py. */
int fo1_model_set_weight(fo1_model* m, const char* name, const void* dev_ptr, int32_t dtype, int32_t ndim,
                         const int64_t* shape);
/* Check that every weight the configured towers need is present with the right shape. */
int fo1_model_finalize(fo1_model* m);

/* Primary tower forward over a batch of images (replaces Qwen2_5_VlVisionTower.forward ->
 * custom_forward + extract_multi_level_features, qwen2_5_vl_encoder.py:86-158, 37-80, 228-257).
 * pixel_values[b]: device fp32 [gh*gw][in_ch*temporal*patch*patch] as Qwen2VLImageProcessor emits it;
 * grid_hw: host int32 [B][2].  Outputs (device, caller-owned, bf16):
 *   img_feats : [sum_b gh*gw/merge^2][out_hidden]   merged tokens, images back to back, raster order
 *   taps[t]   : [sum_b gh*gw][hidden] for each full-attention layer t -- image b's slice is its
 *               channels-last map [gh][gw][hidden] (un-windowed; what HFRE / SimpleFPN read). */
int fo1_vit_forward(fo1_model* m, const float* const* pixel_values, const int32_t* grid_hw, int32_t n_images,
                    void* img_feats, void* const* taps, void* stream);
/* Integer bookkeeping of the tower, exposed for bit-exact parity tests against
 * get_window_index / rot_pos_emb (modeling_qwen2_5_vl.py:436-504).  Host outputs, sized by the caller:
 * window_index [gh*gw/merge^2], cu_window_seqlens [<= n_windows+1] (count returned), pos_hw [gh*gw][2]
 * in window order. */
int fo1_vit_window_index(const fo1_model_config* cfg, int32_t gh, int32_t gw, int32_t* window_index,
                         int32_t* cu_window_seqlens, int32_t* n_cu, int32_t* pos_hw);

/* Aux tower forward (replaces DavitVisionTower.forward -> DaViT.forward_features,
 * davit_aux_encoder.py:54-73, modeling_davit.py:478-506) for n_images images of the SAME size H x W.
 * images[b]: device fp32 [3][H][W] (CLIP-normalised).  stage_out[s]: bf16 [B][H_s][W_s][C_s], s = 0..3. */
int fo1_davit_forward(fo1_model* m, const float* const* images, int32_t H, int32_t W, int32_t n_images,
                      void* const* stage_out, void* stream);

/* SimpleFPN (replaces SimpleFP.forward, simple_fpn.py:197-216) on n_images last-tap maps of the SAME grid.
 * tap: bf16 [B][gh][gw][hidden] ; level_out[l]: bf16 [B][gh*f][gw*f][fpn_out], f = 4, 2, 1, 1/2. */
int fo1_fpn_forward(fo1_model* m, const void* tap, int32_t gh, int32_t gw, int32_t n_images, void* const* level_out,
                    void* stream);

/* Region projector mm_projector_aux (omchat_qwen2_5_vl.py:107): bf16 [n][region_dim] -> bf16 [n][llm_hidden]. */
int fo1_region_project(fo1_model* m, const void* feats, int32_t n, void* out, void* stream);
/* Image projector mm_projector (encode_images, omchat_qwen2_5_vl.py:58-66; multimodal_projector/builder.py:39-76) for the
 * `linear` / `mlpNx_gelu` types: bf16 [n][vit_out_hidden] -> bf16 [n][llm_hidden].  The released checkpoint uses
 * `identity` (proj_img_layers = 0): the call is then an error and the caller passes the tower output through. */
int fo1_image_project(fo1_model* m, const void* feats, int32_t n, void* out, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Device-side image pre-processing (SURVEY.md section 8f rank 1): uint8 RGB [H][W][3] in device memory -> the tensors the two
 * host processors produce, bit-identical (integer resize; float32 normalisation in the processors' operation order).
 * ---------------------------------------------------------------------------------------------- */
/* PIL's bicubic resize of an 8-bit image (what Qwen2VLImageProcessor / CLIPImageProcessor call: mm_utils.py:615, :596 ->
 * PIL Image.resize(BICUBIC)): horizontal pass then vertical pass with the uint8 intermediate.  bounds: host-computed, DEVICE
 * int32 [out][2] = (first input index, count); coef: DEVICE int32 [out][ksize], 22 fractional bits (PIL's normalised
 * coefficients; vlm-fo1_b200/preprocess.py computes them).  tmp: [H][out_w][3] bytes when both axes change.  A pass whose
 * size does not change is skipped (its tables may be NULL). */
int fo1_resize_bicubic_u8(const void* img, int32_t H, int32_t W, int32_t out_h, int32_t out_w, const int32_t* h_bounds,
                          const int32_t* h_coef, int32_t h_ksize, const int32_t* v_bounds, const int32_t* v_coef, int32_t v_ksize,
                          void* tmp, void* out, void* stream);
/* Qwen2VLImageProcessor's rescale + normalise + patchify (2x2-merge order, frame repeated over the temporal patch) of an image
 * whose sides are already multiples of patch*merge: -> fp32 [H/patch * W/patch][3*temporal*patch*patch].  mean / std: HOST [3]. */
int fo1_preprocess_primary_u8(const void* img, int32_t H, int32_t W, int32_t patch, int32_t merge, int32_t temporal, const float* mean,
                              const float* std, float* pixel_values, void* stream);
/* CLIPImageProcessor's rescale + normalise + channels-first (davit/image_processing_clip.py:344-358): -> fp32 [3][H][W]. */
int fo1_preprocess_aux_u8(const void* img, int32_t H, int32_t W, const float* mean, const float* std, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LLM half: embedding splice, M-RoPE bookkeeping, prefill and greedy decode.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t image_token_id;        /* config.image_token_id (151655) */
  int32_t video_token_id;        /* config.video_token_id (151656) */
  int32_t vision_start_token_id; /* config.vision_start_token_id (151652) */
  int32_t merge;                 /* vision_config.spatial_merge_size */
  int32_t image_placeholder;     /* IMAGE_TOKEN_INDEX  (-200, vlm_fo1/constants.py) */
  int32_t region_placeholder;    /* DEFAULT_REGION_INDEX (-300) */
} fo1_splice_cfg;

/* Integer work of prepare_inputs_labels_for_qwen2_5_vl_multimodal (omchat_qwen2_5_vl.py:291-373, 434-458)
 * + get_rope_index (modeling_qwen2_5_vl.py:1546-1721) for ONE sample (host only, bit-exact):
 * every image placeholder expands to that image's gh*gw/merge^2 feature rows (ids <- image_token_id), every
 * region placeholder keeps one slot (id stays region_placeholder); then the 3-axis position ids.
 * Outputs (host, capacity elements each; position_ids 3*capacity laid out [3][capacity]):
 *   new_ids, src_kind (0 text / 1 image row / 2 region row), src_index (token id / row in the image- /
 *   region-feature matrix of this sample), position_ids, *rope_delta, *out_len.
 * Returns FO1_ERR_WORKSPACE if capacity is too small (out_len then holds the needed length). */
int fo1_splice_plan(const int64_t* input_ids, int32_t n_ids, const int32_t* image_grid_hw, int32_t n_images,
                    int32_t n_regions, const fo1_splice_cfg* cfg, int64_t* new_ids, int32_t* src_kind,
                    int32_t* src_index, int32_t* position_ids, int32_t* rope_delta, int32_t* out_len,
                    int32_t capacity);

/* The same integer work for a whole BATCH of prompts in one launch, on the device (SURVEY.md section 8f rank 2): all pointers
 * are DEVICE int32 arrays.  ids / id_off: the prompts' ids concatenated + offsets [n_samples+1]; grids / img_off: (gh, gw) of
 * every image + offsets [n_samples+1]; n_regions [n_samples]; out_off [n_samples+1]: row offsets of the spliced sequences
 * (L_b = n_ids_b - n_img_b + sum gh*gw/merge^2, host arithmetic); img_row_off / reg_row_off [n_samples]: first row of the
 * sample in the batch's image- / region-feature matrices (added to src_index).  Outputs over total_rows = out_off[n_samples]:
 * new_ids, src_kind, src_index [total_rows], position_ids [3][total_rows], rope_delta / status [n_samples] (status 0 or a
 * fo1_status per sample).  Bit-identical to fo1_splice_plan sample by sample. */
int fo1_splice_plan_batch(const int32_t* ids, const int32_t* id_off, const int32_t* grids, const int32_t* img_off,
                          const int32_t* n_regions, const int32_t* out_off, const int32_t* img_row_off,
                          const int32_t* reg_row_off, int32_t n_samples, int64_t total_rows, const fo1_splice_cfg* cfg,
                          int32_t* new_ids, int32_t* src_kind, int32_t* src_index, int32_t* position_ids, int32_t* rope_delta,
                          int32_t* status, void* stream);

/* extract_predictions_to_indexes (vlm_fo1/mm_utils.py:346-369) over the decoded TOKEN IDS of a batch, on the device, for
 * tokenizers that hold "<ground>", "</ground>", "<objects>", "</objects>" and every "<regionN>" as single tokens: tokens DEVICE
 * int32 [n_samples][ld], lens [n_samples]; region_ids DEVICE [n_region_ids] (id of <region0>, <region1>, ...); newline_bitmap
 * DEVICE, bit t set iff the text of token t contains a newline ("." of the reference's regex does not cross one), or NULL.
 * records DEVICE [n_samples][max_records][3] = (first label token, label end token (exclusive), N or -1 for a label without
 * regions), n_records DEVICE [n_samples]. */
int fo1_parse_predictions(const int32_t* tokens, int64_t ld, const int32_t* lens, int32_t n_samples, int32_t ground_start_id,
                          int32_t ground_end_id, int32_t objects_start_id, int32_t objects_end_id, const int32_t* region_ids,
                          int32_t n_region_ids, const uint32_t* newline_bitmap, int32_t vocab, int32_t* records, int32_t max_records,
                          int32_t* n_records, void* stream);

/* inputs_embeds[r] = embed_tokens[src_index[r]] | img_feats[src_index[r]] | region_feats[src_index[r]]
 * (omchat_qwen2_5_vl.py:333-368).  src_kind / src_index: device int32 [n_rows]; feature matrices bf16
 * [*, llm_hidden] with indices already offset per sample by the caller. */
int fo1_llm_build_embeds(fo1_model* m, const int32_t* src_kind, const int32_t* src_index, int32_t n_rows,
                         const void* img_feats, const void* region_feats, void* inputs_embeds, void* stream);

typedef struct fo1_sampling_desc fo1_sampling_desc;
typedef struct fo1_score_desc fo1_score_desc;
typedef struct fo1_stream_desc fo1_stream_desc;
typedef struct fo1_prefix_desc fo1_prefix_desc;
typedef struct fo1_processor_desc fo1_processor_desc;
typedef struct fo1_lookup_desc fo1_lookup_desc;
typedef struct fo1_beam_desc fo1_beam_desc;

typedef struct {
  int32_t n_seqs;
  const int32_t* seq_lens;        /* host [n_seqs]: L_b, prompt length after the splice */
  const void* inputs_embeds;      /* device bf16 [sum L_b][llm_hidden], sequences packed back to back */
  const int32_t* position_ids;    /* device int32 [3][sum L_b] */
  const int32_t* rope_deltas;     /* host [n_seqs] */
  int32_t max_new_tokens;
  const int32_t* stop_ids;        /* host [n_stop_ids]: generation stops after emitting one of these */
  int32_t n_stop_ids;
  int32_t pad_id;
  int32_t* out_tokens;            /* device int32 [n_seqs][max_new_tokens], pad_id after the stop token */
  int32_t* out_lens;              /* device int32 [n_seqs], counts the stop token */
  float* prefill_logits;          /* optional device fp32 [n_seqs][vocab]: logits at the last prompt position */
  float* all_logits;              /* optional device fp32 [sum L_b][vocab]: logits at every prompt position */
  int32_t early_exit_interval;    /* host polls "all sequences stopped" every k decode steps (0 = never) */
  int32_t steps_run;              /* out: decode iterations actually executed */
  const int32_t* rope_deltas_device; /* optional DEVICE [n_seqs] (what fo1_splice_plan_batch wrote); overrides rope_deltas when set */
  /* decoding options, each described in its section below; NULL: the option is off */
  const fo1_sampling_desc* sampling;     /* per-sequence sampling (NULL: greedy) */
  const fo1_score_desc* scores;          /* per-token scores */
  const fo1_stream_desc* stream;         /* live token streaming */
  const fo1_prefix_desc* prefix;         /* shared-prefix prefill */
  const fo1_processor_desc* processors;  /* logits processors */
  const fo1_lookup_desc* lookup;         /* prompt-lookup decoding */
  const fo1_beam_desc* beam;             /* beam search */
} fo1_generate_desc;

/* Prefill + decode (replaces OmChatQwen25VLForCausalLM.forward / HF generate's decoding loop /
 * DynamicCache for this path: omchat_qwen2_5_vl.py:466-532, modeling_qwen2_5_vl.py:1126-1242, 1848-1876).
 * The K/V cache and the decode loop state live on the device; the host only launches.  With every option NULL (a
 * zero-initialised descriptor plus the inputs and outputs) the call is greedy.
 *
 * An option that asks for nothing is the call without it: a `scores` whose three outputs are NULL, a `prefix` with
 * n_groups == 0, and `processors` in which no sequence has a set (seq_set[b] == -1 for every b).
 *
 * Which options combine (any pair not listed combines):
 *   beam        takes none of sampling, scores, stream, prefix, processors, lookup; refuses all_logits, allows prefill_logits
 *   lookup      takes sampling, scores and prefix; refuses stream, processors and beam
 *   prefix      refuses all_logits
 *   processors  takes sampling, scores, stream and prefix
 * A refused pair returns FO1_ERR_UNSUPPORTED, with a message that names both options, before any option's own checks and before
 * the model is touched.  Every argument is checked on the host before anything is enqueued; a failed check of an option returns
 * FO1_ERR_INVALID_ARG with the message "fo1_llm_generate: <option>: <rule>". */
int fo1_llm_generate(fo1_model* m, fo1_generate_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sampled decoding (replaces HF generate's sampling branch as the reference drives it, mm_utils.py:630-654 ->
 * GenerationMixin._sample with the warpers TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper and
 * torch.multinomial, transformers/generation/logits_process.py).  Per row: x = logits / T (fp32); keep the tokens whose
 * x >= the k-th largest (ties kept); keep the tokens whose softmax mass ranked above them is < p; draw with
 * u = (x0 >> 8) * 2^-24 of Philox4x32-10(key = seed, counter = (step, 0, 0, 0)), ranking by x descending, then index
 * ascending.  top_k == 1 is greedy (lowest index among equal maxima).  A row's token depends only on its logits, its
 * parameters and its step.  The parameter arrays are validated on the host before any CUDA call.
 * ---------------------------------------------------------------------------------------------- */
struct fo1_sampling_desc {
  const float* temperature;  /* HOST [n]: > 0 and finite; 1.0 = no scaling */
  const float* top_p;        /* HOST [n]: (0, 1]; 1.0 = off */
  const int32_t* top_k;      /* HOST [n]: >= 0; 0 or >= vocab = off */
  const uint64_t* seed;      /* HOST [n]: Philox key of each row / sequence */
};
size_t fo1_sample_tokens_workspace_bytes(int32_t n_rows);
/* One token per row of fp32 logits [n_rows][ld] (device); step: DEVICE int32 [n_rows], the Philox counter of each row. */
int fo1_sample_tokens(const float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_sampling_desc* sp,
                      const int32_t* step /* DEVICE [n_rows] */, int32_t* out_tokens /* DEVICE [n_rows] */,
                      void* workspace, size_t workspace_bytes, void* stream);
/* fo1_llm_generate with d.sampling samples each sequence with its parameters (the step of a sequence's token is its output column). */

/* ------------------------------------------------------------------------------------------------
 * Per-token scores (HF generate's return_dict_in_generate with output_logits / output_scores, and the log-probability of each
 * emitted token that model.compute_transition_scores(..., normalize_logits=True) derives from them).  For sequence b at output
 * column t (0 <= t < out_lens[b]):
 *   logits[t][b]  the fp32 row the token was chosen from, as the LM head produced it (persistent kernel: the fp32 head epilogue;
 *                 per-kernel path: the LM-head GEMM output).  Column 0 is the prefill's last-position row, bit-identical to
 *                 prefill_logits.  Unlike the reference's outputs.logits.float(), these are not rounded to bf16.
 *   scores[t][b]  the processed row, as HF's _sample forms next_token_scores: a greedy (raw) row is its logits unchanged; a sampled
 *                 row is x = logits / T (IEEE fp32 division) where the token is kept and -inf elsewhere.  The kept set is the
 *                 sampler's: top-k keeps x >= the k-th largest (ties included), top-p the canonical order and fixed-point weights;
 *                 for top_k == 1 it is every token equal to the maximum (HF's TopK rule; the token drawn is still the
 *                 lowest-index maximum).
 *   logprobs[b][t] ln of the emitted token's probability under scores[t][b]: (x_tok - x_max) - ln(Z_kept * 2^-40), Z_kept the
 *                 sampler's fixed-point sum of exp(x - x_max) over the kept set (a raw row: the whole vocabulary, T = 1).  0 at
 *                 or past out_lens[b].  Depends only on the row, its parameters and the token (not on the slot, batch or path).
 * Rows of scores / logits past a sequence's stop column, or of steps an early exit skipped, are unspecified.  Asking for any
 * of these never changes a token: the tokens are bit-identical to the same call without scoring.
 * ---------------------------------------------------------------------------------------------- */
struct fo1_score_desc {
  float* logprobs;          /* optional DEVICE fp32 [n_seqs][max_new_tokens] */
  float* scores;            /* optional DEVICE fp32 [max_new_tokens][n_seqs][vocab] (HF output_scores) */
  float* logits;            /* optional DEVICE fp32 [max_new_tokens][n_seqs][vocab] (HF output_logits) */
  const int32_t* raw_rows;  /* optional HOST [n_seqs]: 1 = greedy sequence (top_k 1, temperature 1), scored on its raw logits.
                               Ignored without d.sampling: every sequence is then greedy and raw. */
};
/* fo1_llm_generate with d.scores: a greedy call with scoring samples with top_k 1, which is bit-identical to greedy.
 * fo1_score_rows is that scoring for arbitrary tokens: rows [n_rows] of fp32 logits (DEVICE, pitch ld) -> logprobs[r]
 * of tokens[r] (-inf for a token outside the kept set) and, optionally, the processed rows scores[r] (pitch ld_scores).
 * sp == NULL or raw_rows[r] == 1: the row is scored raw (T = 1, nothing cut). */
int fo1_score_rows(const float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_sampling_desc* sp /* NULL: raw */,
                   const int32_t* raw_rows /* HOST, optional */, const int32_t* tokens /* DEVICE [n_rows] */,
                   float* logprobs /* DEVICE [n_rows] */, float* scores /* DEVICE, optional */, int64_t ld_scores, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Streamed decoding (what HF generate's `streamer` needs: each token as it is produced, and a way to stop early).  The decode
 * loop stays on the device with no per-token host sync; the device publishes every output column into host memory the caller
 * owns, and the host reads it whenever it chooses.
 *   Layout: tokens [n_seqs][max_new_tokens] and lens [n_seqs] mirror out_tokens / out_lens; progress is one int32 holding
 *           columns_published | FO1_STREAM_DONE; cancel is one int32 the host may set.  All are HOST pointers to pinned memory
 *           mapped for the device (cudaHostAlloc, or cudaHostRegister with cudaHostRegisterMapped); pageable memory is rejected.
 *   Publication: the code that records column t (the persistent kernel's CTA 0, or the per-kernel path's update kernel, which
 *           also records column 0 after the prefill on both paths) writes column t of tokens, and lens, with exactly the values
 *           out_tokens / out_lens get (pad included), fences at system scope, then release-stores progress = (t + 1) | done.
 *           So after an acquire load of progress == c, columns < c of tokens are final, and lens[b] is final for every
 *           sequence that stopped before column c (a running sequence may already show the next column's length).
 *   done:   set at the last column: no sequence is active after this column's stop test, t + 1 == max_new_tokens, or the column
 *           was cancelled.  Nothing is published after it, so the final progress is done | max(out_lens).  The call stores
 *           progress = 0 before it enqueues anything, and done | 0 at once when max_new_tokens == 0.
 *   cancel: read once per column, with a system-scope load, before the column is recorded.  When it is set, column t is still
 *           recorded normally; then every running sequence ends there (out_lens = t + 1) and the loop stops.  For each sequence
 *           the tokens before that cut are bit-identical to the same call without a cancel; the tail is pad.  The call never
 *           clears cancel: the caller zeroes it before the call.
 * Streaming changes no token, score or logit: the outputs are bit-identical to the same call without it.
 * ---------------------------------------------------------------------------------------------- */
#define FO1_STREAM_DONE (1 << 30)
struct fo1_stream_desc {
  int32_t* tokens;          /* HOST mapped [n_seqs][max_new_tokens] */
  int32_t* lens;            /* HOST mapped [n_seqs] */
  int32_t* progress;        /* HOST mapped [1] */
  const int32_t* cancel;    /* HOST mapped [1], optional (NULL: the loop cannot be cancelled) */
};
/* fo1_llm_generate with d.stream: the buffers are validated (non-NULL, pinned and mapped) before anything is launched; the device
 * uses their cudaHostGetDevicePointer aliases. */
/* Acquire load of *progress and release store of 1 to *cancel: plain host code (no device, no model), for hosts whose language
 * cannot express the ordering (and for CPUs with a weaker memory model than x86). */
int32_t fo1_stream_progress(const int32_t* progress);
void fo1_stream_cancel(int32_t* cancel);

/* ------------------------------------------------------------------------------------------------
 * Shared-prefix prefill (many questions about one image).  Sequences of a group start with the same P_g rows (same embeddings,
 * same M-RoPE positions).  Those rows are prefilled once: one causal segment per group, packed before the sequences' own rows
 * through every layer, and their rotated K/V rows are written into the cache slot of every member at rows 0 .. P_g - 1.  The
 * remaining "own" rows of each sequence attend its cache (fo1_prefix_attention).  Decode is unchanged: each sequence owns a full
 * copy of its prefix K/V.  Every output (tokens, lengths, prefill logits, scores, logits, streamed columns) is bit-identical to
 * fo1_llm_generate without d.prefix on the full sequences.
 * ---------------------------------------------------------------------------------------------- */
struct fo1_prefix_desc {
  int32_t n_groups;
  const int32_t* prefix_lens;          /* HOST [n_groups]: P_g >= 1 */
  const void* prefix_embeds;           /* DEVICE bf16 [sum P_g][llm_hidden], groups back to back */
  const int32_t* prefix_position_ids;  /* DEVICE int32 [3][sum P_g] */
  const int32_t* seq_group;            /* HOST [n_seqs]: the sequence's group, or -1 (no shared prefix) */
};
/* fo1_llm_generate with d.prefix: seq_lens stays the full length L_b; inputs_embeds / position_ids hold only each sequence's own
 * rows (L_b - P_g, or L_b without a group), packed in sequence order.  Checked on the host before any CUDA call: group indices in
 * range, at least two members per group, P_g < L_b for every member, non-NULL pointers, and no all_logits. */

/* ------------------------------------------------------------------------------------------------
 * Teacher-forced scoring (the reference's forward(labels=...): omchat_qwen2_5_vl.py:466-532 with HF's ForCausalLMLoss).  The prefill
 * of fo1_llm_generate (same layers, same launches, optionally a shared prefix), then, instead of decoding, the log-likelihood of each
 * scored row's target under the LM head: only the scored rows are gathered, normed (the kernel the all_logits output uses) and run
 * through the LM-head GEMM with a log-likelihood epilogue; nothing vocabulary-sized is written unless all_logits is asked for.
 *
 * Rows are the packed rows of the FULL sequences (sum L_b, sequence b's rows back to back), with or without a prefix, as all_logits
 * lays them out.  targets[r] is the id row r predicts (the labels already shifted by one), or -100: not scored.  Per scored row:
 *   target_logit  the fp32 logit of the target, bit-identical to all_logits[r][target]
 *   lse           log sum_v exp(logit_v), from per-128-column partials (max, sum of exp(x - max)) merged in column order
 *   greedy        1 when the target is the lowest-index maximum of the row
 *   logprobs[r]   target_logit - lse (0 where the row is not scored)
 * and per sequence seq_logprob = the fp64 sum of its rows' logprobs in row order, seq_count = its scored rows.  Every reduction runs
 * in an order that depends on the row alone: a sequence's outputs are bit-identical whatever else is in the call and with or
 * without its prefix shared.
 *
 * Checked on the host before anything is enqueued, with the message "fo1_llm_loglik: <rule>": non-NULL inputs and outputs, targets
 * in [0, vocab) or -100, no scored last row of a sequence (it has nothing to predict), no scored row inside a shared prefix (the
 * row predicting the first own token is itself an own row), no all_logits with a prefix (as fo1_llm_generate), no open slot pool
 * (the call writes the K/V cache, as fo1_llm_generate does).
 *
 * ABI: fo1_llm_loglik and fo1_loglik_desc are additions; no existing declaration changed, so FO1_ABI_VERSION stays 4.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t n_seqs;
  const int32_t* seq_lens;         /* HOST [n_seqs]: L_b after the splice */
  const void* inputs_embeds;       /* DEVICE bf16 [rows][llm_hidden]: every row, or with `prefix` only each sequence's own rows */
  const int32_t* position_ids;     /* DEVICE int32 [3][rows], rows as inputs_embeds */
  const fo1_prefix_desc* prefix;   /* optional shared prefix (fo1_prefix_desc, checked as fo1_llm_generate checks it) */
  const int32_t* targets;          /* HOST int32 [sum L_b]: HOST because the host checks them and sizes the head from them */
  float* logprobs;                 /* DEVICE fp32 [sum L_b] */
  int32_t* greedy;                 /* optional DEVICE int32 [sum L_b] (0 where not scored) */
  double* seq_logprob;             /* DEVICE fp64 [n_seqs] */
  int32_t* seq_count;              /* DEVICE int32 [n_seqs] */
  float* all_logits;               /* optional DEVICE fp32 [sum L_b][vocab], as fo1_llm_generate's (refused with prefix) */
  float* lse;                      /* optional DEVICE fp32 [n_scored]: lse of the scored rows, in row order */
  float* target_logits;            /* optional DEVICE fp32 [n_scored]: their target logits, in row order */
} fo1_loglik_desc;
int fo1_llm_loglik(fo1_model* m, const fo1_loglik_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Beam search (HF generate with num_beams > 1 and do_sample=False: transformers' GenerationMixin._beam_search and its helpers).
 * Each of the n_seqs prompts runs as if it were alone in the call, with num_beams = N decode rows and cache slots.  Per step,
 * over log_softmax(logits) of the running beams: accumulated = log-prob + running score (initially [0, -1e9, ...]); the best
 * n_keep = K of the N * V continuations (score descending, then beam * V + token ascending); a continuation hits the stop test
 * if its token is a stop id or it reaches max_new_tokens; the running set is the best N of (score + hit * -1e9); hits among the
 * best N enter the finished set with score / (float)pow(len, length_penalty) unless the prompt is full (early_stopping True) or
 * cannot improve (the early-stop heuristic); the finished set keeps the best N (old entries before new on equal scores).  The
 * prompt stops when HF's _beam_search_has_unfinished_sequences would for it alone.  Every fp32 operation is HF's, in its order,
 * so the selection is bit-identical to HF's fed the same log-prob rows.  The prompt is prefilled once; its K/V is written into
 * its N slots, and after each step the generated rows of each new beam are copied from its parent's slot.
 * In d: out_tokens [n_seqs * num_return][max_new_tokens] (pad_id past each length) and out_lens [n_seqs * num_return] receive the
 * best num_return hypotheses of each prompt, best first; all_logits is refused, prefill_logits is allowed; steps_run is the number
 * of decode iterations the loop ran.  Always the per-kernel decode path (fo1_last_decode_path() == 0).
 * ---------------------------------------------------------------------------------------------- */
struct fo1_beam_desc {
  int32_t num_beams;         /* N: 2 .. 16 */
  int32_t n_keep;            /* K: HF's max(2, 1 + number of eos ids) * N; 2N <= K <= 128 and K <= vocab */
  double length_penalty;     /* finite; double, as HF's Python float: the divisors are (float)pow(len, length_penalty) */
  int32_t early_stopping;    /* 0 = False, 1 = True, 2 = "never" */
  int32_t num_return;        /* 1 .. N hypotheses per prompt */
  float* sequence_scores;    /* DEVICE fp32 [n_seqs * num_return]: the hypotheses' length-penalised scores */
  int32_t* beam_indices;     /* DEVICE int32 [n_seqs * num_return][max_new_tokens]: prompt * N + parent beam per token, -1 past the length */
  int32_t* steps_run;        /* DEVICE int32 [n_seqs]: steps the prompt ran (rows of scores / logits it wrote) */
  float* scores;             /* optional DEVICE fp32 [max_new_tokens][n_seqs * N][vocab]: log_softmax of each beam row (HF output_scores) */
  float* logits;             /* optional DEVICE fp32 [max_new_tokens][n_seqs * N][vocab]: the raw rows (HF output_logits) */
  float* logprobs;           /* optional DEVICE fp32 [n_seqs * num_return][max_new_tokens]: each returned token's log-probability
                                under its parent beam's row (HF's compute_transition_scores with beam_indices); 0 past the length */
};
/* fo1_llm_generate with d.beam: checked on the host before any CUDA call: 2 <= N <= 16, 1 <= num_return <= N,
 * 2N <= n_keep <= min(128, vocab), a finite length_penalty, early_stopping in {0, 1, 2}, max_new_tokens >= 1, the outputs non-NULL
 * and no all_logits. */

/* ------------------------------------------------------------------------------------------------
 * Prompt-lookup decoding (HF generate's prompt_lookup_num_tokens / max_matching_ngram_size).  Each sequence's corpus is its
 * prompt ids as the caller passes them (placeholders included), followed by every token it has emitted.  Per step, the drafts are
 * HF's PromptLookupCandidateGenerator.get_candidates: for n = min(max_ngram, len - 1) down to 1, the leftmost occurrence of the
 * last n ids with a non-empty continuation gives up to K following ids, cut at the first stop id.  The engine also cuts them at
 * the first negative id, caps them at max_new_tokens - emitted - 1 and K at 16.  One verify step runs B * (K + 1) rows, each
 * bit-identical to the plain per-kernel step's row for that position; the longest draft prefix equal to the rows' tokens is
 * accepted and n_matches + 1 tokens are emitted (stopping at a stop id or max_new_tokens).  So tokens, lengths and the score
 * outputs (rows up to each length) equal those of the plain per-kernel call (FO1_NO_MEGA=1), greedy, sampled or scored.  Always
 * the per-kernel decode path; the K/V cache slot grows by K rows.  steps_run is the number of verify steps the loop ran: with
 * early_exit_interval > 0 the loop polls after every verify step, one step behind (at most one step runs after the last sequence
 * ends); with 0 it never polls and runs max_new_tokens - 1 steps.
 * ---------------------------------------------------------------------------------------------- */
struct fo1_lookup_desc {
  int32_t num_tokens;               /* K >= 1 (drafts per step; more than 16 proposes 16) */
  int32_t max_ngram;                /* >= 1 */
  const int32_t* corpus;            /* HOST int32, the n_seqs corpora packed */
  const int32_t* corpus_offsets;    /* HOST int32 [n_seqs + 1]: corpus b is corpus[offsets[b] .. offsets[b + 1]) */
  int32_t* steps;                   /* optional DEVICE int32 [n_seqs]: verify steps the sequence took part in */
  int32_t* accepted;                /* optional DEVICE int32 [n_seqs]: drafts accepted */
};
/* fo1_llm_generate with d.lookup: checked on the host before any CUDA call: num_tokens >= 1, max_ngram >= 1, corpus offsets present,
 * starting at 0 and non-decreasing, corpus present when non-empty.  d.sampling, d.scores and d.prefix work as without lookup (the
 * prefill is unchanged). */
/* The draft rule alone: corpora DEVICE int32 [n_seqs][ld] with lengths lens [n_seqs] -> drafts DEVICE int32 [n_seqs][num_tokens]
 * and n_draft [n_seqs].  stop_ids DEVICE [n_stop]; emitted (DEVICE [n_seqs], optional) with max_new_tokens caps the drafts at
 * max_new_tokens - emitted - 1.  1 <= num_tokens <= 16, max_ngram >= 1. */
int fo1_lookup_drafts(const int32_t* corpus, int64_t ld, const int32_t* lens, int32_t n_seqs, int32_t num_tokens, int32_t max_ngram,
                      const int32_t* stop_ids, int32_t n_stop, const int32_t* emitted, int32_t max_new_tokens, int32_t* drafts,
                      int32_t* n_draft, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Logits processors (HF generate's sequence_bias, no_repeat_ngram_size, bad_words_ids, min_length, min_new_tokens, suppress_tokens
 * and begin_suppress_tokens: transformers' GenerationMixin._get_logits_processor).  Before a column's token is chosen, the row of a
 * sequence with a processor set is edited in place, in HF's order
 *   SequenceBias -> NoRepeatNGram -> NoBadWords -> MinLength -> MinNewTokensLength -> SuppressTokens -> SuppressTokensAtBegin,
 * over HF's input_ids: the sequence's prompt ids as the caller passes them (placeholders included), then the tokens it has emitted.
 *   sequence_bias: a sequence of length 1 always adds its bias to its token; a longer one adds it to its last token when the history
 *                  ends with the others.  A token's biases are summed in fp32 from 0, the length-1 bias first, then the longer
 *                  sequences in their given order, and the sum is added once.
 *   bad words:     the same match; the last token becomes -inf.
 *   no_repeat_ngram_size n: with L history ids and L + 1 >= n, every earlier n-gram whose first n - 1 ids equal the last n - 1
 *                  history ids bans its last id (-inf; a negative prompt id bans vocab + id, as torch indexing wraps it).
 *   min_length:    the eos ids are -inf while L < min_length (the prompt counts).  min_new_tokens: while the column < min_new_tokens.
 *   suppress:      always -inf.  begin_suppress: -inf at column 0.
 * Column 0, drawn from the prefill's last row, is processed too.  A row without a set is never edited: its outputs are bit-identical
 * to the same call without processors.  Scores: `logits` stays the raw row, `scores` is the processed one (then the sampler's cut),
 * and the log-probabilities are those of the processed row.  A row that ends up all -inf (every token banned) draws token 0, the
 * arg-max rule, on every path, greedy or sampled; nothing is kept, so its log-probability is -inf.
 * ---------------------------------------------------------------------------------------------- */
struct fo1_processor_desc {
  int32_t n_sets;                          /* >= 1 processor sets, each used by any number of sequences */
  const int32_t* seq_set;                  /* HOST [n_seqs]: the sequence's set, or -1 (no processors) */
  const int32_t* prompt;                   /* HOST: the sequences' prompt ids packed, each in [-vocab, vocab) */
  const int32_t* prompt_offsets;           /* HOST [n_seqs + 1]: prompt b is prompt[offsets[b] .. offsets[b + 1]), offsets[0] == 0 */
  const int32_t* no_repeat_ngram_size;     /* HOST [n_sets]: >= 0 (0: off) */
  const int32_t* min_length;               /* HOST [n_sets]: >= 0 (0: off) */
  const int32_t* min_new_tokens;           /* HOST [n_sets]: >= 0 (0: off) */
  /* id lists of set s: ids[offsets[s] .. offsets[s + 1]), each offsets array HOST [n_sets + 1], non-decreasing, <= n_ids */
  const int32_t* eos_offsets;              /* the eos ids MinLength / MinNewTokens mask (HF's eos_token_id, not the stop list) */
  const int32_t* suppress_offsets;
  const int32_t* begin_suppress_offsets;
  /* token sequences of set s: sequences [offsets[s] .. offsets[s + 1]), each offsets array HOST [n_sets + 1], non-decreasing,
   * <= n_sequences; sequence k is ids[seq_offsets[k] .. seq_offsets[k + 1]) (non-empty) */
  const int32_t* bias_offsets;             /* sequence_bias, in its given order */
  const int32_t* bad_offsets;              /* bad_words_ids */
  int32_t n_sequences;
  const int32_t* seq_offsets;              /* HOST [n_sequences + 1], non-decreasing, <= n_ids */
  const float* bias;                       /* HOST [n_sequences]: the bias of each sequence_bias sequence, finite (bad words: unread) */
  int32_t n_ids;
  const int32_t* ids;                      /* HOST [n_ids]: token ids in [0, vocab) */
};
/* fo1_llm_generate with d.processors: checked on the host before any launch: the ranges above.  A greedy call with processors chooses
 * through the sampler with top_k 1 (bit-identical to the arg-max), on the persistent kernel too. */
/* The row routine alone: rows [n_rows] of fp32 logits (DEVICE, pitch ld) edited in place; row r is sequence r of pr at output column
 * cols[r] (HOST), its emitted tokens outputs[r][0 .. cols[r]) (DEVICE, pitch ld_out; may be NULL when every column is 0). */
int fo1_logits_process(float* logits, int64_t ld, int32_t n_rows, int32_t vocab, const fo1_processor_desc* pr, const int32_t* outputs,
                       int64_t ld_out, const int32_t* cols, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Slot pool: in-flight batching of many requests (replaces the reference callers' one-image-at-a-time generate loop,
 * eval_coco.py:36-88 / eval_countbench.py:30-60, for a whole request list).  n_slots K/V cache slots and decode-state rows live
 * across calls; the host repeats: admit waiting requests into free slots (fo1_slots_admit), decode every slot until at most exit_at
 * sequences still run (fo1_slots_decode), take out the finished ones.  A slot's output column is its own: its index in the slot's
 * output row, the Philox step of its sampler, and what is tested against its own max_new_tokens; a slot that reaches its limit or a
 * stop id finishes and stays idle (its cache stops growing) until it is admitted again.  Every step runs all n_slots rows, so the
 * decode attention's key split and the decode path follow n_slots for the life of the pool: each request's tokens and length equal
 * its tokens and length in a static fo1_llm_generate call of n_slots sequences (with d.sampling) on the same decode path, whatever its
 * companions and whenever it was admitted.  Greedy and sampled decoding; no scores, streaming, beams, lookup or shared prefixes.
 * While a pool is open it owns the model's K/V cache: every fo1_llm_generate call is refused.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t n_slots;              /* 1 .. 65535 */
  int32_t cap;                  /* K/V rows per slot: a request needs prompt length + max_new_tokens <= cap */
  int32_t max_new_tokens;       /* the widest per-request limit: the pitch of out_tokens (1 .. cap - 1) */
  const int32_t* stop_ids;      /* HOST [n_stop_ids] */
  int32_t n_stop_ids;
  int32_t pad_id;
  int32_t sampled;              /* 1: some request may sample (a greedy one then draws with top_k 1, bit-identical to greedy) */
  int32_t early_exit_interval;  /* >= 1: the per-kernel path polls the running count every k steps */
  int32_t* out_tokens;          /* DEVICE [n_slots][max_new_tokens]: slot b's current or last request, pad_id past its length */
  int32_t* out_lens;            /* DEVICE [n_slots] */
  int32_t* finished;            /* DEVICE [n_slots]: 1 once the slot's request has stopped (and for a slot never admitted) */
} fo1_slots_desc;
/* Opens the pool (all slots idle).  Refused while one is open. */
int fo1_slots_open(fo1_model* m, const fo1_slots_desc* o, void* stream);

typedef struct {
  int32_t n;                             /* requests admitted, 1 .. n_slots */
  const int32_t* slots;                  /* HOST [n]: distinct free slots */
  const int32_t* seq_lens;               /* HOST [n]: prompt lengths after the splice */
  const void* inputs_embeds;             /* DEVICE bf16 [sum seq_lens][llm_hidden], packed */
  const int32_t* position_ids;           /* DEVICE int32 [3][sum seq_lens] */
  const int32_t* rope_deltas_device;     /* DEVICE int32 [n] (what fo1_splice_plan_batch wrote) */
  const int32_t* max_new_tokens;         /* HOST [n]: each request's own limit, 1 .. the pool's max_new_tokens */
  const fo1_sampling_desc* sampling;     /* NULL: greedy; else per request (a pool opened with sampled = 1) */
  const fo1_processor_desc* processors;  /* NULL: none; else per request, checked as fo1_llm_generate checks d.processors.  The
                                            pool keeps each admitted request's set and prompt ids until its slot is admitted again. */
} fo1_slots_admit_desc;
/* Prefills the n requests into their slots (the prefill of fo1_llm_generate with the slots as the cache-write members) and records
 * column 0.  Checked on the host before any launch: slot in range, slot free (never admitted, or seen finished by the last
 * fo1_slots_decode), no slot twice, 1 <= max_new_tokens <= the pool's, prompt + max_new_tokens <= cap, sampling parameters. */
int fo1_slots_admit(fo1_model* m, const fo1_slots_admit_desc* a, void* stream);
/* Decodes every slot until at most exit_at requests still run (0: all stopped): one launch of the persistent kernel (n_slots <= 32
 * and a supported model shape), else the per-kernel loop polling every early_exit_interval steps.  *steps_run = the decode steps
 * run (0 when no more than exit_at run already).  Synchronises the stream; on return out_tokens / out_lens / finished are final for
 * every finished slot, until it is admitted again. */
int fo1_slots_decode(fo1_model* m, int32_t exit_at, int32_t* steps_run, void* stream);
/* Closes the pool (synchronises the device). */
int fo1_slots_close(fo1_model* m);

#ifdef __cplusplus
}
#endif
#endif /* FO1_H_ */
