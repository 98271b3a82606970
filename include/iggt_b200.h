/*
 * iggt_b200.h -- C ABI of the Hopper-native (sm_90a) IGGT inference kernels (libiggt_b200.so).
 *
 * The reference (lifuguan/IGGT_official) has no FFI on this path: everything below
 * `IGGT.forward` (iggt/models/vggt.py:149-230) is torch.nn modules.  This header is therefore the
 * boundary SURVEY.md 8(b) asks the builder to define: one `extern "C"` launcher per fused operator,
 * raw device pointers + sizes + a CUDA stream, `int` return (0 = ok, <0 = argument/setup error,
 * >0 = cudaError_t).  Each entry cites the reference call site it replaces.  All pointers are device
 * pointers unless stated otherwise; all launches are asynchronous on `stream`.
 *
 * dtype: 0 = fp16, 1 = bf16 (16-bit activations / weights; accumulation is always fp32).
 */
#ifndef IGGT_B200_H_
#define IGGT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* iggt_stream_t; /* cudaStream_t */

/* Library / device probe. Returns 0 and fills sm (e.g. 100) and num_sms, or >0 cudaError_t. */
int iggt_device_info(int* sm, int* num_sms);
const char* iggt_version(void);

/* ---- GEMM family (wgmma / TMA).  A:[M,K] lda, W:[N,K] ldw (torch Linear layout), 16-bit. */

/* out16[M,N] = act(A W^T + bias) (+ addend[(row % add_rows), :]).  act: 0 none, 1 exact-erf GELU,
 * 2 ReLU, 3 LeakyReLU(0.01).  Replaces mlp.fc1 (iggt/layers/mlp.py:35-36), DPT `projects` 1x1 conv +
 * pos-embed (iggt/heads/dpt_head.py:238-240), generic Linear layers. */
int iggt_gemm_store16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out, int64_t ldo,
                      int M, int N, int K, int dtype, const float* bias, int act,
                      const void* addend, int add_rows, int64_t add_ld, iggt_stream_t stream);

/* x32[M,N] += gamma * r(A W^T + bias)   (fp32 residual stream, TMA reduce-add); r() rounds to the 16-bit
 * dtype when round_out16 != 0 (what an autocast nn.Linear returns before LayerScale), identity otherwise.
 * Replaces attn.proj / mlp.fc2 + LayerScale + residual (iggt/layers/attention.py:74-75, mlp.py:38,
 * layer_scale.py:27, block.py:105-106). */
int iggt_gemm_resid32(const void* A, int64_t lda, const void* W, int64_t ldw, float* x, int64_t ldx,
                      int M, int N, int K, int dtype, const float* bias, const float* gamma,
                      int round_out16, iggt_stream_t stream);

/* out32[M,N] = act(A W^T + bias) (fp32 output). */
int iggt_gemm_store32(const void* A, int64_t lda, const void* W, int64_t ldw, float* out, int64_t ldo,
                      int M, int N, int K, int dtype, const float* bias, int act, iggt_stream_t stream);

/* qkv16[M,3C] = A Wqkv^T + bias, then (if qk_norm) per 64-wide head of the q and k column ranges:
 * LayerNorm(64, eps 1e-5, affine) followed by 2-D RoPE (first 32 dims by y, last 32 by x, rotate-half
 * of 16, table [npos][16]).  Row r is token r % T of its view; pos_yx[T][2] holds (y,x).
 * Replaces iggt/layers/attention.py:52-58 + iggt/layers/rope.py:154-188.
 * gather_maps / n_gather / gather_rows (may be NULL / 0 / 0): see iggt_kv_gather_maps - the K | V chunks are also stored to every
 * rank's gathered buffer (the all-gather of view sharding fused into this GEMM). */
int iggt_gemm_qkv(const void* A, int64_t lda, const void* W, int64_t ldw, void* qkv, int64_t ldo,
                  int M, int C, int K, int dtype, const float* bias, int qk_norm,
                  const float* qn_w, const float* qn_b, const float* kn_w, const float* kn_b,
                  const float* rope_cos, const float* rope_sin, const int* pos_yx, int T,
                  const void* gather_maps, int n_gather, int gather_rows, iggt_stream_t stream);

/* View sharding (new design, SURVEY 8e): n tensor maps (written to the device array dev_maps, 128 B each) through
 * which iggt_gemm_qkv (gather_maps / n_gather / gather_rows = rows) stores the K | V chunks of every tile into each
 * rank's gathered K|V buffer as well - dst[i] = this rank's first row inside rank i's buffer ([scenes][world*rows][cols],
 * row pitch ld, scene pitch scene_ld elements), a peer-mapped pointer (torch symmetric memory over NVLink).  The
 * collective it replaces: one all-gather of K|V per global block (reference shape: iggt/models/aggregator.py:308-336,
 * attention over all S*T keys of a scene).  dev_maps receives n * 136 + 16 bytes: the n maps, the n raw pointers and
 * (ld, scene_ld) - rows of a tile that belong to a later scene than its first row are stored through the pointers. */
int iggt_kv_gather_maps(void* const* dst, int n, int64_t rows, int64_t cols, int64_t ld, int64_t scenes, int64_t scene_ld,
                        int dtype, void* dev_maps);

/* 3x3 (pad 1, stride 1) or 1x1 convolution as implicit GEMM over an NHWC 16-bit tensor:
 * out[NB,H,W,Cout] = act_post(act(conv(x[NB,H,W,Cin], Wp[Cout, taps*Cin]) + bias) + resid + resid2)
 * (resid / resid2: optional [NB,H,W,Cout] 16-bit tensors; act codes as above).
 * Wp is packed tap-major: k = (ky*3+kx)*Cin + ci.  Cin % 64 == 0.
 * Replaces the Conv2d layers of iggt/heads/dpt_head.py:298-316,369-411. */
int iggt_conv_nhwc(const void* x, const void* Wp, void* out, int NB, int H, int W, int Cin, int Cout,
                   int taps, int dtype, const float* bias, int act, const void* resid,
                   const void* resid2, int act_post, iggt_stream_t stream);


/* ---- Flash attention forward (wgmma QK^T / PV, register accumulators, online softmax), head_dim 64.
 * q/k/v/o: token-major [rows, ld] 16-bit, head h in columns [64h, 64h+64).  Sequence s owns q/o rows
 * [s*Lq,(s+1)*Lq) and k/v rows [s*Lk,(s+1)*Lk).  Non-causal, no mask.
 * Replaces F.scaled_dot_product_attention at iggt/layers/attention.py:61-66. */
int iggt_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                       int64_t ldv, void* o, int64_t ldo, int num_seq, int Lq, int Lk, int H,
                       int head_dim, float scale, int dtype, iggt_stream_t stream);

/* Split-KV form of iggt_attention_fwd for launches with fewer work items than SMs (view-sharded ranks: local queries
 * against the gathered keys).  iggt_attention_plan picks the number of kv ranges for the shape (1 = do not split;
 * sms <= 0: the current device's SM count) and the fp32 workspace it needs; iggt_attention_fwd_ws runs the flash kernel
 * per (item, kv range) into the workspace (un-normalised O, running max, row sum) and merges the ranges.
 * Same reference call site: F.scaled_dot_product_attention, iggt/layers/attention.py:61-66. */
int iggt_attention_plan(int num_seq, int Lq, int Lk, int H, int sms, int* splits, int64_t* ws_bytes);
int iggt_attention_fwd_ws(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                          int64_t ldo, int num_seq, int Lq, int Lk, int H, int head_dim, float scale, int dtype,
                          int splits, void* ws, int64_t ws_bytes, iggt_stream_t stream);
/* Host-side view of the split launch's static schedule (no GPU needed): see iggt_attention_schedule. */
int iggt_attention_schedule_splits(int num_seq, int Lq, int Lk, int H, int splits, int grid, int cta, int* items,
                                   int max_items, int* tiles_per_split);

/* ---- HBM-bound trunk kernels. */

/* LayerNorm over C (1024 or 2048) fp32 features, one warp per row.  Output row g*out_rows_per_group +
 * out_off + i  <-  input row g*rows_in + in_off + i, for g < groups, i < rows_out.  w/b may be NULL.
 * out_kind: 0 fp16, 1 bf16, 2 fp32.  Replaces nn.LayerNorm at iggt/layers/block.py:50,66,
 * iggt/layers/vision_transformer.py:274, iggt/heads/dpt_head.py:234. */
int iggt_layernorm(const float* x, int64_t ldx, void* y, int64_t ldy, int C, const float* w,
                   const float* b, float eps, int64_t groups, int rows_out, int rows_in, int in_off,
                   int out_rows_per_group, int out_off, int out_kind, iggt_stream_t stream);

/* images [NI,3,H,W] fp32 in [0,1] -> A[NI*(H/14)*(W/14), KP] 16-bit im2col rows of the 14x14/s14 patch
 * conv (k = c*196 + ky*14 + kx, zero padded to KP >= 588), fused with the ImageNet (x-mean)/std.
 * Replaces iggt/models/aggregator.py:206 + iggt/layers/patch_embed.py:75-77 (the GEMM follows). */
int iggt_patchify(const float* images, void* A, int NI, int H, int W, int KP, int dtype,
                  iggt_stream_t stream);

/* DINOv2 token assembly: x[n,0]=cls+pos[0]; x[n,1..R]=reg; x[n,1+R+p]=pe16[n,p]+pos[1+p]  (fp32 out).
 * Replaces iggt/layers/vision_transformer.py:217-236. */
int iggt_dino_assemble(const void* pe16, const float* cls, const float* reg, const float* pos, float* x,
                       int NI, int P, int R, int C, int dtype, iggt_stream_t stream);

/* Aggregator camera/register tokens into rows [n*T, n*T+1+R) of x (variant 0 for view 0 of a scene).
 * Replaces iggt/models/aggregator.py:230-234,338-361. */
int iggt_special_tokens(const float* cam, const float* reg, float* x, int NI, int T, int R, int C,
                        int S_loc, int view_offset, iggt_stream_t stream);

/* ---- Dense-head / camera-head kernels (NHWC 16-bit activations). */

/* F.interpolate(bilinear, align_corners=True) [NB,h,w,C] -> [NB,H,W,C], optionally + the UV sinusoid
 * pos-embed split as tabx[W][C/2] (first half of the channels) and taby[H][C/2] (second half), both fp32.
 * Replaces iggt/heads/dpt_head.py:251-259,478 (+ :274-284). */
int iggt_upsample_bilinear_nhwc(const void* x, void* out, int NB, int h, int w, int H, int W, int C,
                                const float* tabx, const float* taby, int dtype, iggt_stream_t stream);

/* ConvTranspose2d with kernel == stride k: y[(n,yy,xx), (dy*k+dx)*C+co] -> out[n, k*yy+dy, k*xx+dx, co].
 * Replaces the scatter half of iggt/heads/dpt_head.py:85-92 (the GEMM half is iggt_gemm_store16). */
int iggt_deconv_shuffle(const void* y, void* out, int NB, int h, int w, int C, int k, iggt_stream_t stream);

/* im2col of a 3x3 / stride 2 / pad 1 conv: [NB,h,w,C] -> [NB*ho*wo, 9*C], k = tap*C + c.
 * Replaces the gather half of iggt/heads/dpt_head.py:94-97. */
int iggt_im2col3x3_s2(const void* x, void* A, int NB, int h, int w, int C, iggt_stream_t stream);

/* Per-pixel 1x1 conv 32 -> OC (fp32 weights w[OC][32], b[OC]) + head activation on x[NB,H,W,32].
 * mode 0 (depth): main[NB,H,W,OC-1] = exp, conf[NB,H,W] = 1+exp;  mode 1 (points): sign*expm1|.|;
 * mode 2 (part_feat): raw, channels-first main[NB,OC,H,W].
 * Replaces iggt/heads/dpt_head.py:264-265 + iggt/heads/head_act.py:61-125, part_head.py:240-243. */
int iggt_dpt_tail(const void* x, const float* w, const float* b, float* out_main, float* out_conf, int NB,
                  int H, int W, int OC, int mode, int dtype, iggt_stream_t stream);

/* The dense heads' last stage in one launch: 3x3 conv 128 -> 32 (pad 1, weights Wp[32][9*128] tap-major 16-bit,
 * bias[32]) + ReLU + 1x1 conv 32 -> OC in fp32 (w2[OC][32], b2[OC]) + the head activation of iggt_dpt_tail
 * (mode 0 / 1 / 2), x = [NB,H,W,128] 16-bit NHWC.  The 32-channel map never leaves registers.  With w2 == NULL the
 * ReLU map is stored instead (out16 [NB,H,W,32] 16-bit) - the unfused form, kept for A/B checks.
 * Replaces iggt/heads/dpt_head.py:120-126 (`output_conv2`) + :264-265 + iggt/heads/head_act.py:61-125, and
 * iggt/heads/part_head.py:240-243. */
int iggt_dpt_tail_fused(const void* x, const void* Wp, const float* bias, const float* w2, const float* b2,
                        float* out_main, float* out_conf, void* out16, int NB, int H, int W, int OC, int mode,
                        int dtype, iggt_stream_t stream);

/* out[M,N] = resid + gamma * act(x[M,K] W[N,K]^T + bias), M <= 32, fp32 activations, 16-bit weights
 * (weight-bandwidth bound; act: 0 none, 1 GELU, 2 ReLU, 4 SiLU).  Camera-head Linear layers,
 * iggt/heads/camera_head.py:83-154. */
int iggt_skinny_gemm(const float* x, int64_t ldx, const void* W, int64_t ldw, const float* bias,
                     const float* gamma, const float* resid, int64_t ldr, float* out, int64_t ldo, int M,
                     int N, int K, int act, int dtype, iggt_stream_t stream);

/* fp32 softmax attention for tiny sequences: qkv[B*N, 3*H*d] -> out[B*N, H*d] (camera tokens). */
int iggt_small_attention(const float* qkv, float* out, int B, int N, int H, int d, float scale,
                         iggt_stream_t stream);

/* The whole camera head in ONE persistent launch (B*S <= 16 camera tokens; larger batches use iggt_skinny_gemm /
 * iggt_small_attention per layer).  Replaces iggt/heads/camera_head.py:83-154 (`CameraHead.forward` + `trunk_fn`:
 * token_norm, 4 x [embed_pose -> SiLU + Linear -> AdaLN modulate -> 4 Blocks(2048, 16 heads) -> trunk_norm ->
 * Mlp(2048 -> 1024 -> 9) -> accumulate]) and `activate_pose` (iggt/heads/head_act.py:12-35: ReLU on the FoV dims).
 * All weight matrices are 16-bit row-major [N, K] (torch Linear layout); vectors fp32.  tokens: fp32 camera-token rows,
 * row (b*S + s) at tokens + (b*S + s) * ld_tokens (ld_tokens = T*2048 reads layer 23's tokens[:, :, 0] in place).
 * out: fp32 [iters][B*S][9].  workspace: iggt_camera_head_workspace(B*S) bytes, 16-byte aligned.
 * Returns -7 when B*S > 16 (use the per-layer launchers). */
typedef struct {
  const float *n1w, *n1b; const void* qkv_w; const float* qkv_b; const void* proj_w; const float* proj_b; const float* ls1;
  const float *n2w, *n2b; const void* fc1_w; const float* fc1_b; const void* fc2_w; const float* fc2_b; const float* ls2;
} iggt_camera_block;
typedef struct {
  const void* emb_w; const float* emb_b;     /* embed_pose: [2048, 16] (K = 9 zero-padded to 16), [2048] */
  const void* mod_w; const float* mod_b;     /* poseLN_modulation[1]: [6144, 2048] */
  iggt_camera_block blk[4];
  const float *tok_w, *tok_b, *trk_w, *trk_b;  /* token_norm, trunk_norm */
  const void* pb1_w; const float* pb1_b;     /* pose_branch.fc1 [1024, 2048] */
  const void* pb2_w; const float* pb2_b;     /* pose_branch.fc2 [9, 1024] */
  const float* empty;                        /* empty_pose_tokens, 16 floats (9 valid, rest 0) */
} iggt_camera_weights;
int64_t iggt_camera_head_workspace(int M);
int iggt_camera_head(const iggt_camera_weights* w, const float* tokens, int64_t ld_tokens, float* out, void* workspace,
                     int64_t ws_bytes, int B, int S, int iters, int dtype, iggt_stream_t stream);

/* ---- Part (instance-feature) path kernels. */

/* LayerNorm (affine) over C in {64,128,256} channels of 16-bit rows -> 16-bit.
 * Replaces nn.LayerNorm in iggt/heads/window_sa.py (patch_embed.norm, norm1, norm2, norm). */
int iggt_layernorm16(const void* x, void* y, int64_t rows, int C, const float* w, const float* b, float eps,
                     int dtype, iggt_stream_t stream);

/* ConvTranspose2d(k4,s2,p1) gather: Y[(n,iy,ix), (ky*4+kx)*C+co] (GEMM output) -> out[NB,2h,2w,C] + bias.
 * Replaces the scatter half of iggt/heads/adaptor.py:152-157. */
int iggt_col2im_k4s2p1(const void* Y, const float* bias, void* out, int NB, int h, int w, int C, int dtype,
                       iggt_stream_t stream);

/* OCAB window cross-attention on projected q,k,v [NB,h,w,256] (4 heads x 64; 8x8 query windows gathered with
 * the reference's scrambled partition, 12x12 zero-padded key windows, bias table[361][4] indexed by
 * rpi[64][144] (already wrapped to [0,361)).  Replaces iggt/heads/window_sa.py:280-314. */
int iggt_ocab_attention(const void* q, const void* k, const void* v, const float* table, const int* rpi,
                        void* out, int NB, int h, int w, int dtype, iggt_stream_t stream);

/* HAB 8x8 window self-attention on qkv [NB,h,w,384] (4 heads x 32) -> [NB,h,w,128].
 * Replaces iggt/heads/window_sa.py:214-219 + iggt/heads/block.py:113-130. */
int iggt_window_attention(const void* qkv, void* out, int NB, int h, int w, int dtype, iggt_stream_t stream);

/* Per-image channel means of x[NB,hw,C] -> mean[NB,C] fp32 (AdaptiveAvgPool2d(1), window_sa.py:29). */
int iggt_channel_mean(const void* x, float* mean, int NB, int64_t hw, int C, int dtype, iggt_stream_t stream);

/* y = y0 + alpha * cx * sigmoid(W2 relu(W1 mean + b1) + b2)   (ChannelAttention + HAB combine,
 * iggt/heads/window_sa.py:26-38,225); w1 [R,C], w2 [C,R]. */
int iggt_se_scale_add(const void* y0, const void* cx, const float* mean, const float* w1, const float* b1,
                      const float* w2, const float* b2, void* y, int NB, int64_t hw, int C, int R, float alpha,
                      int dtype, iggt_stream_t stream);

/* ---- Post-processing on the device (what demo.py does on the host after a full D2H copy). */

/* pose_enc [n,9] (T, quaternion xyzw, fov_h, fov_w) -> extrinsics [n,3,4] = [R|T], intrinsics [n,3,3] (may be NULL).
 * Replaces iggt/utils/pose_enc.py:65-130 + iggt/utils/rotation.py:14-44. */
int iggt_pose_to_cameras(const float* pose_enc, float* extrinsics, float* intrinsics, int n, int H, int W,
                         iggt_stream_t stream);

/* depth [n,H,W] + cameras -> world points [n,H,W,3] (X_world = R^T (X_cam - t)) and validity mask [n,H,W] u8
 * (eps < d < z_far; mask may be NULL).  Replaces iggt/utils/geometry.py:151-300 (per-frame numpy loop). */
int iggt_unproject_depth(const float* depth, const float* extrinsics, const float* intrinsics, float* world,
                         uint8_t* mask, int n, int H, int W, float eps, float z_far, iggt_stream_t stream);

/* ---- Track head (iggt/heads/track_head.py, track_modules/*): the non-GEMM, non-attention pieces. */

/* One pyramid level: x [NB,H,W,C] 16-bit -> y [NB,H/2,W/2,C] (2x2 mean).  Replaces F.avg_pool2d at blocks.py:173. */
int iggt_avgpool2_nhwc(const void* x, void* y, int NB, int H, int W, int C, int dtype, iggt_stream_t stream);

/* out[n,r,:] fp32 = bilinear sample of x[n] (NHWC 16-bit) at coords[n,r] = (x,y) pixels, align_corners, border
 * padding.  Replaces sample_features4d (track_modules/utils.py:199-226). */
int iggt_sample_bilinear_nhwc(const void* x, const float* coords, float* out, int NB, int R, int H, int W, int C,
                              int dtype, iggt_stream_t stream);

/* Correlation lookup: for every row (b,n,s) and each of the 7 pyramid levels (NHWC [B*S,H_l,W_l,128] 16-bit), the
 * 9x9 window of <target, fmap>/sqrt(128) around coords / 2^level, bilinear, zero padding -> out 16-bit [rows, ldo]
 * (7*81 values then zeros).  Replaces CorrBlock.corr_sample (track_modules/blocks.py:187-246). */
int iggt_corr_sample(const void* const* levels, const int* Hs, const int* Ws, const float* targets, const float* coords,
                     void* out, int B, int N, int S, int ldo, int dtype, iggt_stream_t stream);

/* Transformer input of one refinement iteration, rows (b,n,s): flow embedding | flows/518 | corr feature | track
 * feature, + pos[(b,n)] + ref_tok[s>0], LayerNorm(388) -> out 16-bit [rows, ldo]; raw (optional) = fp32 [rows,388]
 * before the LayerNorm.  Replaces base_track_predictor.py:139-165 + blocks.py:103. */
int iggt_track_input(const float* coords, const float* fcorr, const float* tfeat, const float* pos,
                     const float* ref_tok, const float* ln_w, const float* ln_b, void* out, float* raw, int rows, int S,
                     int ldo, float eps, int dtype, iggt_stream_t stream);

/* LayerNorm over C <= 2048 of fp32 rows (pitch ldx) -> y32 [rows,C] and / or y16 [rows,ld16] zero padded (either may
 * be NULL).  Used for the 384-wide blocks of the update transformer (track_modules/modules.py:136-218). */
int iggt_layernorm_rows(const float* x, int64_t ldx, int C, const float* w, const float* b, float eps, int64_t rows,
                        float* y32, void* y16, int ld16, int dtype, iggt_stream_t stream);

/* ---- Host-side schedules (no GPU work, callable without a GPU): what the launchers above decide before launching.
 * They exist so that tile selection, CTA pairing, stream-K and the attention work distribution are unit-tested. */

/* Schedule of a GEMM launch. epi: 0 store16, 1 resid32, 2 qkv (N = 3C), 3 store32.
 * out[7] = {bn, pair (always 0: no CTA pairs on sm_90), stream_k, m_tiles, n_tiles, k_blocks, grid}. */
int iggt_gemm_plan(int epi, int M, int N, int K, int* out);

/* Work items of CTA `cta` of a `grid`-CTA iggt_attention_fwd launch, in processing order, as quadruples
 * (query-tile pair, head, sequence, tile B has rows); returns their number (first max_items are written). */
int iggt_attention_schedule(int num_seq, int Lq, int Lk, int H, int grid, int cta, int* items, int max_items);

/* ---- Pre-processing on the device (what iggt/utils/load_fn.py:82-98 does on the host with Pillow + torchvision).
 * Bit-exact restatement of Pillow's 8-bit ImagingResample: kk = fixed-point (22 fractional bits) filter taps
 * [out_size, ksize] and bounds = (first tap, tap count) pairs [out_size, 2], both built on the host in double. */

/* Horizontal pass: src u8 [rows, *, 3] (row stride in bytes) -> dst u8 [rows, w_out, 3].
 * Replaces `img.resize(..., BICUBIC)`'s horizontal pass (iggt/utils/load_fn.py:82). */
int iggt_resample_h_u8(const uint8_t* src, int64_t src_row_stride, int rows, int w_out, const int32_t* kk,
                       const int32_t* bounds, int ksize, uint8_t* dst, iggt_stream_t stream);

/* Vertical pass + ToTensor: tmp u8 [*, w_out, 3] (row 0 of tmp is source row y_shift) -> planar fp32 x/255 for output
 * rows [oy0, oy0 + out_rows), written at dst[c * plane_stride + r * row_stride + x].
 * Replaces the vertical pass of `img.resize` + `to_tensor(img)` + the crop / pad of iggt/utils/load_fn.py:82-98. */
int iggt_resample_v_u8_f32(const uint8_t* tmp, int w_out, const int32_t* kk, const int32_t* bounds, int ksize,
                           int y_shift, int oy0, int out_rows, float* dst, int64_t plane_stride, int64_t row_stride,
                           iggt_stream_t stream);

/* ---- k-NN feature smoothing on the device (iggt/utils/misc.py:24-78: torch_geometric knn_graph + scatter_mean).
 * Exact search: Morton-ordered tiles of 256 points + bounding boxes, block-pruned brute force (csrc/knn.cu). */

/* 63-bit Morton code of every point [n,3] on a cubic lattice over the bounding box lo[3]..hi[3] (device pointers). */
int iggt_knn_morton(const float* points, int64_t n, const float* lo, const float* hi, int64_t* codes,
                    iggt_stream_t stream);

/* order[n] (a permutation, e.g. argsort of the codes) -> sorted4 [n,4] = (x, y, z, original index as int bits) and
 * aabb [ceil(n/256), 6] = (min xyz, max xyz) of every tile of 256 consecutive sorted points. */
int iggt_knn_reorder(const float* points, const int64_t* order, int64_t n, float* sorted4, float* aabb,
                     iggt_stream_t stream);

/* For every point: its k (<= 32) nearest other points (knn_graph(loop=False)); out[n,F] = mean of their rows of
 * feats[n,F] (scatter_mean), indexed by ORIGINAL point index.  Optional out_idx [n,k] int32 (-1 = none) and
 * out_d2 [n,k] squared distances.  feats/out may both be NULL when only the graph is wanted.  stats (may be NULL):
 * 3 device counters that are incremented by (tiles staged, warp-tiles searched, queue drains) for profiling. */
int iggt_knn_mean_features(const float* sorted4, const float* aabb, int64_t n, int k, const float* feats, int F,
                           float* out, int32_t* out_idx, float* out_d2, uint64_t* stats, iggt_stream_t stream);

/* ---- HDBSCAN of the instance features (iggt/utils/misc.py:81-170: cluster_features_to_masks_mv, contrib `hdbscan`
 * semantics).  8-d fp32 points; Morton-ordered tiles of 256 points with 8-d boxes, exact block-pruned searches
 * (csrc/cluster.cu).  Distances are squared throughout. */

/* 56-bit Morton key of every point feats8 [n,8] on a 128^8 lattice over the per-axis extent lo[8]..hi[8]. */
int iggt_cluster_morton(const float* feats8, int64_t n, const float* lo, const float* hi, int64_t* codes,
                        iggt_stream_t stream);

/* order[n] (a permutation) -> sorted8 [n,8], orig [n] (original index of each sorted point) and
 * box [ceil(n/256), 16] = (min 8, max 8) of every tile of 256 consecutive sorted points. */
int iggt_cluster_reorder(const float* feats8, const int64_t* order, int64_t n, float* sorted8, int32_t* orig,
                         float* box, iggt_stream_t stream);

/* core2 [n] (sorted order): squared distance of every point to its k-th nearest OTHER point, 1 <= k <= 512, k < n. */
int iggt_cluster_core(const float* sorted8, const float* box, int64_t n, int k, float* core2, iggt_stream_t stream);

/* Host query: *bytes = device workspace size of iggt_cluster_mst for n points. */
int iggt_cluster_mst_workspace(int64_t n, int64_t* bytes);

/* Minimum spanning tree of the mutual-reachability graph max(core_i, core_j, d_ij) by Boruvka (ties: lower weight,
 * then smaller, then larger original index).  Writes n-1 unsorted edges edge_a/edge_b (original indices, edge_a is
 * the endpoint in the component that picked the edge) and edge_w2 (squared weights); *rounds (host pointer, may be
 * NULL) = Boruvka rounds.  Synchronises the stream once per pointer-jumping pass.  -2 / -3: no spanning tree was found. */
int iggt_cluster_mst(const float* sorted8, const float* box, const int32_t* orig, const float* core2, int64_t n,
                     void* workspace, int32_t* edge_a, int32_t* edge_b, float* edge_w2, int32_t* rounds,
                     iggt_stream_t stream);

/* Noise fill: label [n] (sorted order, -1 = noise; at least one labelled point) -> out_label [n] int64 at the original
 * index, a noise point taking the label of its nearest labelled point (ties: lowest original index).  With out_rgb
 * [n,3] (may be NULL), also palette[label] (uint8 [labels,3]).  tile_count: workspace of ceil(n/256) ints. */
int iggt_cluster_fill(const float* sorted8, const float* box, const int32_t* orig, const int32_t* label, int64_t n,
                      int32_t* tile_count, const uint8_t* palette, int64_t* out_label, uint8_t* out_rgb,
                      iggt_stream_t stream);

/* HOST function (no GPU): orients every edge of mst [n-1,3] (a, b, weight) in place from parent to child of the tree
 * rooted at point `root`.  scikit-learn builds its MST with Prim's algorithm from point 0, which records every edge
 * from the tree side, and the single-linkage tree puts the first endpoint's side on the left: with root 0, the cluster
 * numbering of iggt_hdbscan_labels then follows scikit-learn's for the same tree.  -2: not a spanning tree. */
int iggt_mst_orient(double* mst, int64_t n, int64_t root);

/* HOST function (no GPU): labels [n] (-1 = noise) from an MST given as mst [n-1,3] = (a, b, weight) rows in float64,
 * sorted by weight, exactly as scikit-learn 1.9's tree_to_labels(make_single_linkage(mst), min_cluster_size, "eom",
 * allow_single_cluster=False, cluster_selection_epsilon=eps).  -2: the edges do not form a spanning tree. */
int iggt_hdbscan_labels(const double* mst, int64_t n, int64_t min_cluster_size, double eps, int64_t* labels);

/* ---- PCA feature colours (iggt/utils/misc.py:272-332: apply_pca_colormap, torch.pca_lowrank + torch.quantile) and
 * exact quantiles (csrc/pca.cu).  x [n, C] fp32, 3 <= C <= 8. */

/* Host query: *bytes = device workspace size of iggt_pca_basis for C channels. */
int iggt_pca_basis_workspace(int C, int64_t* bytes);

/* One pass over x: moments [C + C(C+1)/2] fp64 = sums of d = x - x[0] and of d d^T (upper triangle, row-major) and
 * *nonfinite = number of non-finite values, reduced in a fixed order (bit-identical on repeated calls on one device);
 * then one CTA forms cov [C, C] = the sample covariance (all 0 if nonfinite > 0), decomposes it as iggt_sym_eig does
 * (evals [C], evecs [C, C]) and writes V [C, 3] fp32 = the first three eigenvectors. */
int iggt_pca_basis(const float* x, int64_t n, int C, void* workspace, double* moments, double* cov, double* evals,
                   double* evecs, float* V, int64_t* nonfinite, iggt_stream_t stream);

/* y [3, n] (row pitch ldy) = (x V)^T: y[j, i] = sum_c x[i, c] V[c, j], fp32 fmas in channel order. */
int iggt_pca_project(const float* x, int64_t n, int C, const float* V, float* y, int64_t ldy, iggt_stream_t stream);

/* Host query: *bytes = device workspace size of iggt_quantile for `rows` rows (<= 65535). */
int iggt_quantile_workspace(int64_t rows, int64_t* bytes);

/* out [rows, nq] fp32 = torch.quantile(y[r, :n], q[i]) (linear interpolation), bit for bit, for every row r of
 * y [rows, n] (row pitch ld) and every q[i] in [0, 1] (q is a HOST array).  The rank is float32(q) * float32(n - 1)
 * (clamped to n - 1); the floor and ceil order statistics come from a radix selection, no sort, any n < 2^32.
 * A row holding a NaN gives NaN. */
int iggt_quantile(const float* y, int64_t rows, int64_t n, int64_t ld, const float* q, int nq, void* workspace,
                  float* out, iggt_stream_t stream);

/* out [n, 3] = clamp((y[j, i] - lo_j) / (hi_j - lo_j), 0, 1), or 0.5 where hi_j <= lo_j, for y [3, n] (row pitch ldy)
 * and qv [3, 2] = (lo_j, hi_j) (device pointer, e.g. iggt_quantile's output for q = 0.02, 0.98). */
int iggt_pca_stretch(const float* y, int64_t n, int64_t ldy, const float* qv, float* out, iggt_stream_t stream);

/* HOST function (no GPU): symmetric eigendecomposition of a [C, C] (row-major fp64, upper triangle read, 1 <= C <= 8)
 * by cyclic Jacobi, the same code iggt_pca_basis runs on the device.  evals [C] descending (ties: lower index first);
 * evecs [C, C] row-major with eigenvector j in column j, its largest-magnitude component positive (the first one
 * when several tie).  -1: a non-finite entry. */
int iggt_sym_eig(const double* a, int C, double* evals, double* evecs);

#ifdef __cplusplus
}
#endif
#endif /* IGGT_B200_H_ */
