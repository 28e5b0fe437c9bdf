/*
 * hi3d_b200.h -- C ABI of libhi3d_b200.so: the H100 (sm_90a) kernels behind the Hi3D denoising hot path.
 *
 * Boundary (SURVEY.md 8b): the reference is pure Python/PyTorch; its "FFI" for this path is the set of
 * ATen / cuDNN / cuBLAS / xformers calls its nn.Modules make.  Each entry point below replaces one such
 * call site (cited as reference file:line, relative to the Hi3D-Official tree) and is what a maintainer
 * of the reference would bind with ctypes/cffi (stub shown in INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers + sizes; no torch types.  All pointers are DEVICE pointers unless noted.
 *   - activations are fp16, channels-last: a feature map is [N, H, W, C] == a token matrix [N*H*W, C];
 *     frames of a clip are consecutive samples, n = b*T + t (reference "(b t)" order, video_model.py:71).
 *   - every call only enqueues work on `stream` (a cudaStream_t passed as void*): no allocation, no
 *     host synchronisation, safe to capture in a CUDA graph.  Workspaces are caller-owned.
 *   - return 0 on success, negative on error; hi3d_last_error() returns a thread-local message.
 */
#ifndef HI3D_B200_H_
#define HI3D_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HI3D_MAX_SEGS 24
#define HI3D_MAX_PEERS 16   /* ranks of one frame-sharded video (16 frames) */

/* library ------------------------------------------------------------------------------------ */
int hi3d_abi_version(void);
const char* hi3d_last_error(void);
/* Number of kernels this library has launched since load (for bench.py's `gpu_launches`). */
int64_t hi3d_launch_count(void);
/* sm count etc. of the current device (cached).  Returns 0 or negative error. */
int hi3d_device_info(int* sm_count, int* cc_major, int* cc_minor, int* max_smem_optin);

/* ---------------------------------------------------------------------------------------------
 * Implicit-GEMM engine.  out[M, N] = epilogue( A[M, K] * W[N, K]^T )
 *
 * A is never materialised: its K axis is a list of segments, each a (tap, channel-range) view of an
 * NHWC fp16 tensor.  This one entry point replaces, in the reference:
 *   nn.Linear                      attention.py:272-278 (to_q/k/v/out), :90 (GEGLU proj), :109 (ff out),
 *                                  video_attention.py:221-223 (time_pos_embed), openaimodel.py:286 (emb)
 *   nn.Conv2d 3x3 s1/s2, 1x1       openaimodel.py:135,192,260,297,314; model.py:63,82,110,117,127
 *   nearest-x2 + Conv2d            openaimodel.py:154-156; model.py:67-70     (ups = 1)
 *   F.pad(0,1,0,1) + Conv2d s2 p0  model.py:84-88                              (taps dy,dx in {0,1,2})
 *   nn.Conv3d (3,1,1)              openaimodel.py:260,297 with dims=3 via video_model.py:42-55 (mode 2)
 *   th.cat([h, hs.pop()], 1)       video_model.py:491  (two segments per tap = virtual concat)
 *   skip_connection 1x1 / nin_shortcut   openaimodel.py:314,354; model.py:127,149 (extra K segments)
 * and in the epilogue: + bias, + emb[:, :, None, None] (openaimodel.py:352), residual adds
 * (attention.py:551-572), GEGLU x*gelu(gate) (attention.py:92-94), AlphaBlender (util.py:358-369).
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  const void* src;   /* fp16 NHWC source tensor                                            */
  int32_t ld;        /* elements between consecutive pixels/rows of src (its channel count) */
  int32_t c_off;     /* first channel of the segment                                        */
  int32_t C;         /* channels in the segment; multiple of 64                             */
  int32_t dy, dx;    /* spatial tap offset in (upsampled) input coordinates                 */
  int32_t dt;        /* temporal tap offset in frames (mode 2)                              */
} hi3d_seg;

enum { HI3D_ROWS_PLAIN = 0, HI3D_ROWS_CONV2D = 1, HI3D_ROWS_TEMPORAL = 2 };
/* GELU: exact erf GELU (nn.GELU, open_clip ViT-H MLP); QUICKGELU: x*sigmoid(1.702x) (OpenAI CLIP clip/model.py MLP); RELU:
 * max(x, 0) (the MiDaS DPT head and residual conv units, annotator/midas/blocks.py, dpt_depth.py:89-96).  All three are
 * applied in fp32 to the fp16-rounded value (+ bias) in the epilogue's store pass, before the residual add. */
enum { HI3D_ACT_NONE = 0, HI3D_ACT_SILU = 1, HI3D_ACT_GEGLU = 2, HI3D_ACT_GELU = 3, HI3D_ACT_QUICKGELU = 4, HI3D_ACT_RELU = 5 };

typedef struct {
  int32_t M, N, K;          /* K == sum of seg[i].C; N multiple of 8                                   */
  int32_t mode;             /* HI3D_ROWS_*                                                             */
  int32_t Ho, Wo;           /* CONV2D: output H, W (M == Nimg*Ho*Wo).  TEMPORAL: Ho*Wo = rows per frame */
  int32_t Hs, Ws;           /* CONV2D: source H, W (before the optional x2 nearest upsample)           */
  int32_t stride;           /* CONV2D: 1 or 2                                                          */
  int32_t ups;              /* CONV2D: 1 -> taps address the x2 nearest-upsampled source               */
  int32_t T;                /* TEMPORAL: frames per clip                                               */
  int32_t out_up;           /* CONV2D: 1 -> rows index an (n, y, x) grid of Ho x Wo but are WRITTEN to the x2 grid at
                               (2y + out_py, 2x + out_px): one parity class of nearest-x2 + conv3x3, which is a 2x2
                               conv on the source grid with pre-summed taps (4 launches, 4/9 of the FLOPs)       */
  int32_t out_py, out_px;
  int32_t Tin, t_off;       /* TEMPORAL: frames per clip in the SOURCE tensors and frame offset of output frame 0 in it
                               (0, 0 -> Tin = T).  Frame-sharded runs read a haloed [B, T_local + 2, HW, C] buffer:
                               Tin = T + 2, t_off = 1; taps that fall outside [0, Tin) read zeros.            */
  int32_t nseg;
  hi3d_seg seg[HI3D_MAX_SEGS];
  const void* W;            /* fp16 [N, K], K contiguous, K ordered as the segments                    */
  const float* bias;        /* [N] or NULL                                                             */
  const void* rowbias;      /* fp16 [R, rb_ld] or NULL; row r = (m / rb_div) % rb_mod                  */
  int32_t rb_div, rb_mod, rb_ld;
  int32_t act;              /* HI3D_ACT_*; GEGLU: W rows interleaved (value, gate), output width N/2   */
  const void* residual;     /* fp16 [M, res_ld] or NULL, added after the activation                    */
  int32_t res_ld;
  const void* blend_x;      /* fp16 [M, blend_ld] or NULL: out = alpha*blend_x + (1-alpha)*value       */
  int32_t blend_ld;
  float alpha;
  void* out;                /* fp16 [M, out_ld]                                                        */
  int32_t out_ld;
} hi3d_gemm_params;

int hi3d_gemm(const hi3d_gemm_params* p, void* stream);
/* Same contract on the Hopper-native engine (TMA operand staging through an mbarrier ring, wgmma with register
 * accumulators, warp-specialised producer / MMA warpgroups): the production path.  Geometries it does not cover (N < 32,
 * upsample-fused convs, > 4 distinct A sources, ...) are forwarded to hi3d_gemm, with identical results. */
int hi3d_gemm_tc5(const hi3d_gemm_params* p, void* stream);
/* Test / tuning hooks of hi3d_gemm_tc5, process-wide: whether a CTA owns one 128-row tile (8 MMA / epilogue warps) or a pair of
 * consecutive row tiles sharing each B tile (16 warps, tile widths <= 128).  set_pair_mode: -1 = automatic (default, or
 * HI3D_TC5_PAIR at first use), 0 = single tiles, 1 = pairs.  set_epilogue_warps: -1 = automatic (default, or HI3D_TC5_EW),
 * 8 = single tiles, 16 = pairs; a forced pair mode takes precedence. */
int hi3d_gemm_tc5_set_pair_mode(int mode);
int hi3d_gemm_tc5_set_epilogue_warps(int warps);
/* The same engine with e4m3 (float8_e4m3fn) operands: every segment source and W are e4m3, K-major like the fp16 ones (src
 * [rows, ld] with ld a multiple of 16, W [N, K]); wgmma k32, each chain of 128 K elements added into fp32 accumulators (the
 * tensor cores' own FP8 accumulation has reduced precision), in the same order at every tile.  The epilogue first scales the
 * accumulator of column n by w_scale[n] (fp32 [N], W's dequantisation scale, see pack.pack_e4m3), then applies exactly the fp16
 * sequence: bias, rowbias, activation, residual, blend (rowbias, residual and blend_x stay fp16).  out_fp8 = 0: out is fp16; 1: out is
 * e4m3, each value the fp16 result converted with cvt.rn.satfinite (nearest even, saturating to +-448).  Tile width, tile pairs
 * and the hooks above follow the fp16 rules.  There is no other e4m3 engine: a geometry this one does not cover (see
 * hi3d_gemm_tc5) returns an error. */
int hi3d_gemm_tc5_fp8(const hi3d_gemm_params* p, const float* w_scale, int out_fp8, void* stream);
/* Whether hi3d_gemm_tc5_fp8 covers the GEMM described by p: 1 yes, 0 no, negative for malformed parameters.  Only the
 * geometry is read (M, N, mode, Ho, Wo, Hs, Ws, stride, ups, out_up, T, the segments' sources and lds, rowbias alignment), so a
 * launch plan can ask before its buffers exist: leave the pointers NULL and list one segment per distinct source. */
int hi3d_gemm_tc5_fp8_covers(const hi3d_gemm_params* p);
/* The schedule and tile width hi3d_gemm_tc5 runs the GEMM described by p with, under the current hooks: schedule * 1000 + tile
 * width, with schedule 1 = one 128-row tile per CTA, 2 = tile pairs, 3 = ping-pong (a persistent grid, two consumer warpgroups
 * that take turns on the tensor cores, each epilogue overlapping the other's main loop); 0 = the mma.sync engine (geometry not
 * covered); negative for malformed parameters.  Host-only: launches nothing. */
int hi3d_gemm_tc5_schedule(const hi3d_gemm_params* p);

/* Tiny channel counts (UNet input 8|17 ch, VAE image 3 ch / latent 4 ch) are zero-padded to 64 channels by
 * hi3d_sampler_pre / hi3d_nchw_to_nhwc so that the same engine serves input_blocks.0.0 (video_model.py:186-191),
 * encoder.conv_in (model.py:517) and decoder.conv_in (model.py:654); tiny C_out (4 | 8 | 3) is padded to 8. */

/* ---------------------------------------------------------------------------------------------
 * Normalisation
 * --------------------------------------------------------------------------------------------- */
/* GroupNorm(32 groups) [+ SiLU] over `rows_per_sample` consecutive rows x (C/32) channels, on the virtual channel-concat of
 * up to two NHWC fp16 sources (x1: C1 channels, x2: C2 channels or NULL).  Replaces GroupNorm32 (util.py:274-276; eps 1e-5;
 * temporal ResBlock: the reduction over (C/32, T, H, W) of video_model.py:71-76), Normalize (attention.py:125-128,
 * model.py:52-55; eps 1e-6) and the following nn.SiLU / x*sigmoid(x).  Output y: fp16 [rows, C1+C2].
 *
 * Statistics travel as unit tables: fp32 [n_images, C/unit, 2] = (sum, sum of squares) per image and per `unit` consecutive
 * channels, accumulated (zero the table first).  A producer's table is made by calling hi3d_groupnorm_unit_stats on its
 * output after it (after the last of an up-conv's four parity-class launches, once the tensor is complete).  Units, not the
 * 32 groups, because a consumer may normalise the channel concat of two tensors (video_model.py:491) whose groups straddle
 * the boundary.  unit must divide C1, C2 and C/32, with at most 256 units per tensor.
 *
 * Reproducibility: hi3d_groupnorm_unit_stats and hi3d_groupnorm_group_sums use no float atomics and sum in a fixed order.
 *  - The same input gives the same table bits on every call.
 *  - An image's entries depend only on that image's rows, rows_per_image, C and unit, never on the other images of the
 *    launch: an image alone and the same image inside any batch get the same bits.
 *  - Each table entry has exactly one writer per launch, which adds this launch's sum to the value already there; launches
 *    into the same table are ordered by the stream. */
int hi3d_groupnorm_unit_stats(const void* x, int C, int n_images, int64_t rows_per_image, int unit, float* stats, void* stream);

/* GroupNorm(32)[+SiLU] in ONE launch, its statistics read from the unit tables of x1 (stats1) and x2 (stats2, or NULL).
 * Sample n spans images [n*imgs_per_sample, (n+1)*imgs_per_sample): 1 for the spatial GroupNorm32, T for the temporal
 * ResBlock.  count_rows = rows per sample the statistics cover (rows_per_sample).  Output layout and halo arguments as
 * hi3d_groupnorm_apply_halo (y_sample_rows = 0 and frame_rows = 0: dense output like x). */
int hi3d_groupnorm_apply_stats(const void* x1, int C1, const float* stats1, const void* x2, int C2, const float* stats2,
                               int unit, int n_samples, int64_t rows_per_sample, int imgs_per_sample, int64_t count_rows,
                               const float* gamma, const float* beta, float eps, int apply_silu, void* y, int64_t y_sample_rows,
                               int64_t y_row_off, void* y_prev_rank, void* y_next_rank, int64_t frame_rows, void* stream);

/* hi3d_groupnorm_apply_stats with a dense e4m3 output y [rows, C1+C2] (no halo): each value is the fp16 value
 * hi3d_groupnorm_apply_stats stores, converted with cvt.rn.satfinite.e4m3x2.f16x2 (nearest even, saturating to +-448).  The
 * producer of an e4m3 GEMM operand (hi3d_gemm_tc5_fp8). */
int hi3d_groupnorm_apply_stats_fp8(const void* x1, int C1, const float* stats1, const void* x2, int C2, const float* stats2,
                                   int unit, int n_samples, int64_t rows_per_sample, int imgs_per_sample, int64_t count_rows,
                                   const float* gamma, const float* beta, float eps, int apply_silu, void* y, void* stream);

/* Frame-sharded runs, where the temporal ResBlock's GroupNorm reduces over (C/32, T, H, W) with T split over GPUs
 * (SURVEY F9): hi3d_groupnorm_group_sums folds unit tables into `sums` fp32 [n_samples, 32, 2] of the local rows; the host
 * all-reduces them over ranks and hi3d_groupnorm_apply_halo normalises with count_rows = the GLOBAL rows per sample.
 * y may be a haloed buffer: sample n starts at row n * y_sample_rows + y_row_off (0, 0 = dense).  With the one-frame halo
 * exchange of the temporal (3,1,1) conv fused into the stores: y = [n, T_local + 2, frame_rows, C] (y_sample_rows =
 * (T_local + 2) * frame_rows, y_row_off = frame_rows); the first local frame is also stored into the trailing halo slot of
 * `y_prev_rank` (the same buffer of the rank holding the previous frames, mapped through hi3d_symm_open) and the last local
 * frame into the leading slot of `y_next_rank`; NULL at the clip boundaries: the local halo slot is then zero-filled (the
 * Conv3d zero padding, openaimodel.py:252-261).  A hi3d_peer_exchange must separate this launch from the conv that reads
 * the halo slots. */
int hi3d_groupnorm_group_sums(const float* stats1, int C1, const float* stats2, int C2, int unit, int n_samples,
                              int imgs_per_sample, float* sums, void* stream);
int hi3d_groupnorm_apply_halo(const void* x1, int C1, const void* x2, int C2, int n_samples, int64_t rows_per_sample,
                              const float* sums, int64_t count_rows, const float* gamma, const float* beta, float eps,
                              int apply_silu, void* y, int64_t y_sample_rows, int64_t y_row_off, void* y_prev_rank,
                              void* y_next_rank, int64_t frame_rows, void* stream);

/* LayerNorm over the last dim C (<= 2560, multiple of 8) of [M, C] fp16 (+ optional broadcast add before the norm:
 * x + addvec[((m / add_div) % add_mod), :], the `x_mix = x + emb` of video_attention.py:286-287).
 * Replaces nn.LayerNorm at attention.py:520-522, video_attention.py:51,79,93-94.  y fp16 [M, C]. */
int hi3d_layernorm(const void* x, const void* addvec, int add_div, int add_mod, int64_t M, int C, const float* gamma,
                   const float* beta, float eps, void* y, void* stream);
/* hi3d_layernorm with an e4m3 output y [M, C]: each value is the fp16 value hi3d_layernorm stores, converted with
 * cvt.rn.satfinite.e4m3x2.f16x2 (nearest even, saturating to +-448). */
int hi3d_layernorm_fp8(const void* x, const void* addvec, int add_div, int add_mod, int64_t M, int C, const float* gamma,
                       const float* beta, float eps, void* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Attention
 * --------------------------------------------------------------------------------------------- */
/* Spatial self-attention core, head dim 64: softmax(Q K^T * scale) V per (image, head).
 * qkv: fp16 [n_img*L, 3*C] with q | k | v column blocks, heads contiguous (C = heads*64); out fp16 [n_img*L, C].
 * Replaces F.scaled_dot_product_attention / xformers.memory_efficient_attention at attention.py:334,427-439. */
int hi3d_attention_d64(const void* qkv, int n_img, int L, int heads, float scale, void* out, void* stream);
/* same contract on TMA + wgmma (S and O accumulators in registers, P fed back to the tensor cores from registers); any L. */
int hi3d_attention_d64_tc5(const void* qkv, int n_img, int L, int heads, float scale, void* out, void* stream);
/* Tuning / test hooks of hi3d_attention_d64_tc5, process-wide.  set_variant: 0 .. 6 select the key tile and the depth of the
 * K/V ring -- (64 keys, 2 stages), (64, 4), (64, 3), (128, 2), (128, 3), (128, 4), (64, 5) = default; default from
 * HI3D_FMHA_VARIANT.  set_exp_emulation: `quarters` / 4 of the softmax exponentials (0 .. 4; 5 / 6 / 7 = 3/8, 1/8, 5/8) are
 * evaluated on the FMA pipe (range reduction + cubic, relative error 1.6e-4 before the fp16 rounding of P) instead of MUFU;
 * default 0, or HI3D_FMHA_EMU. */
int hi3d_attention_tc5_set_variant(int variant);
int hi3d_attention_tc5_set_exp_emulation(int quarters);

/* The same attention with e4m3 (float8_e4m3fn) operands, in two launches.
 *
 * hi3d_attention_vt_e4m3 writes V in the layout FP8 wgmma needs for P V (B K-major, i.e. keys contiguous):
 *   qkv8: e4m3 [n_img*L, 3*C] (q | k | v column blocks, C = heads*64), as the q|k|v GEMM writes it, unscaled;
 *   vt:   e4m3 [n_img, heads, 64, Lp], Lp = L rounded up to a multiple of 128.  Row (i, h, d) holds V column h*64 + d of
 *         image i, one byte per key, with the keys permuted inside every aligned block of 32 columns: column 32*b + k holds
 *         key 32*b + pi(k), pi(k) = (k & 16) + 8*((k >> 1) & 1) + 2*((k >> 2) & 3) + (k & 1).  Columns whose key is >= L are
 *         written as zero on every call.
 *   pi makes the f32 S accumulator fragment of a thread (keys 8i + 2*t4 + {0, 1}) coincide with its e4m3 A fragment of
 *   the k32 P V product (K columns 4*t4 + 0..3 and 16 + 4*t4 + 0..3).  The caller owns vt; its size in bytes is
 *   hi3d_attention_vt_e4m3_bytes (negative for bad arguments).
 *
 * hi3d_attention_d64_tc5_fp8 computes out fp16 [n_img*L, C] = softmax(Q K^T * scale) V per (image, head) from qkv8's Q and K
 * and vt's V.  Any L >= 1 and any number of images; rows of out past n_img*L are not touched.  S is accumulated by the FP8
 * tensor cores (reduced-precision accumulation), the softmax runs in fp32 with scale applied there, P is scaled by 2^8 and
 * rounded to e4m3 for P V, each 128-key tile's P V is added into fp32 O registers, and the fp32 row sum comes from the
 * unrounded P.  Not the result of hi3d_attention_d64_tc5 on dequantised inputs: P's e4m3 rounding is a relative 2^-4. */
int hi3d_attention_vt_e4m3(const void* qkv8, int n_img, int L, int heads, void* vt, void* stream);
int64_t hi3d_attention_vt_e4m3_bytes(int n_img, int L, int heads);
int hi3d_attention_d64_tc5_fp8(const void* qkv8, const void* vt, int n_img, int L, int heads, float scale, void* out,
                               void* stream);

/* Same contract for head dim 80 (C = heads*80): the OpenCLIP ViT-H/14 image tower's attention (open_clip transformer.py
 * nn.MultiheadAttention, 16 heads of 80; the conditioner's FrozenOpenCLIPImageEmbedder, modules.py:570-728).  Any L >= 1;
 * keys of the next image are masked.  TMA + wgmma, with each 80-column head row staged as a 64-column SWIZZLE_128B box plus a
 * 16-column SWIZZLE_32B box (no padding of the head dimension). */
int hi3d_attention_d80_tc5(const void* qkv, int n_img, int L, int heads, float scale, void* out, void* stream);

/* Temporal self-attention core over the frame axis (T <= 16), head dim 64, for every (clip, pixel, head):
 * token row of (b, t, s) is (b*T + t)*S + s -- the "(b t) s c -> (b s) t c" rearrange of
 * video_attention.py:114,137-139 is done by addressing, never materialised.
 * qkv fp16 [B*T*S, 3*C]; out fp16 [B*T*S, C].  Replaces attn1 core at video_attention.py:125. */
int hi3d_temporal_attention_d64(const void* qkv, int B, int T, int S, int heads, float scale, void* out,
                                void* stream);

/* Frame-sharded form (SURVEY 8e; the reference has no multi-GPU inference, README.md:56-64): rank r owns frames
 * [r*T_local, (r+1)*T_local) of every clip in its own qkv / out buffers (layout as above with T = T_local) and computes
 * pixel strip r of all T_local*world frames: q|k|v rows of the other ranks' frames are READ from `qkv_of_rank[owner]` and the
 * output rows of their frames are STORED into `out_of_rank[owner]` (device pointers of the peers' buffers mapped with
 * hi3d_symm_open; entry [rank] = the local buffers).  One hi3d_peer_exchange before (all q|k|v written) and one after (all
 * outputs stored) order it against the producing / consuming GEMMs. */
int hi3d_temporal_attention_d64_sharded(void* const* qkv_of_rank, void* const* out_of_rank, int rank, int world, int B,
                                        int T_local, int S, int heads, float scale, void* stream);

/* VAE mid-block attention (AttnBlock, model.py:180-201; xformers path model.py:204-265): ONE head of dimension 512,
 * softmax(q k^T * scale) v per image with scale = 512^-0.5, as a flash-attention kernel (TMA + wgmma): fp32
 * scores and softmax, no L x L matrix in memory.  qkv: fp16 [n_img*L, 1536] = q | k | v column blocks (the three 1x1 convs as
 * one GEMM); out fp16 [n_img*L, 512].  L must be a multiple of 128 ((H/8)*(W/8) at every Hi3D size). */
int hi3d_attention_d512_tc5(const void* qkv, int n_img, int L, float scale, void* out, void* stream);

/* Row softmax in place on fp16 [rows, L] (scores * scale), and 2-D transpose [R, Cc] -> [Cc, R] (fp16):
 * building blocks of the VAE single-head d=512 attention (model.py:180-195) on top of hi3d_gemm. */
int hi3d_softmax_rows(void* s, int64_t rows, int L, float scale, void* stream);
int hi3d_transpose(const void* in, int R, int Cc, int in_ld, void* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sampler-side fused elementwise kernels (EulerEDMSampler / Denoiser / LinearPredictionGuider)
 * --------------------------------------------------------------------------------------------- */
/* timestep_embedding (util.py:207-231): t fp32 [n] -> fp16 [n, dim] = [cos | sin]. */
int hi3d_timestep_embedding(const float* t, int n, int dim, float max_period, void* out, void* stream);

/* Build the UNet input for one CFG-batched step: prepare_inputs (guiders.py:88-99) + Denoiser c_in scaling
 * (denoiser.py:33-37) + OpenAIWrapper concat (wrappers.py:27) + NCHW->NHWC fp16.
 * x fp32 NCHW [F, Cx, H, W]; sigma fp32 [F]; concat_uc / concat_c fp16-or-fp32 NCHW [F, Cc, H, W] (concat_uc may be
 * NULL == zeros); out fp16 NHWC [2F, H, W, Cpad] (channels [x*c_in | concat | 0-pad]); first F samples = uc half.
 * c_noise_out (optional) fp32 [2F] receives c_noise = 0.25*ln(sigma) (denoiser_scaling.py:58), the UNet `timesteps`. */
int hi3d_sampler_pre(const float* x, const float* sigma, const void* concat_uc, const void* concat_c,
                     int concat_is_fp32, int F, int Cx, int Cc, int H, int W, int Cpad, void* out, float* c_noise_out,
                     void* stream);

/* Finish the step: denoised = net*c_out + x*c_skip per half (denoiser.py:36-39), CFG combine with the per-frame
 * scale (guiders.py:78-86), d = (x - denoised)/sigma and Euler update x += d*(sigma_next - sigma)
 * (sampling.py:99-103, sampling_utils.py:34).  net fp16 NHWC [2F, H, W, net_ld] (first Cx channels used);
 * x fp32 NCHW [F, Cx, H, W] updated in place (x_out may alias x); scale fp32 [T] (frame t = f % T);
 * denoised_out optional fp32 NCHW [F, Cx, H, W] (the guided D(x, sigma), for teacher-forced parity checks). */
int hi3d_sampler_post(const void* net, int net_ld, const float* x, const float* sigma, const float* sigma_next,
                      const float* scale, int T, int F, int Cx, int H, int W, float* x_out, float* denoised_out,
                      void* stream);

/* Solver algebra of the multi-evaluation samplers on the fp32 sampler state (SURVEY 8f N4): out = sum_k c_k[f] * x_k, up to four
 * terms (x1..x3 may be NULL), fp32 NCHW tensors of F samples x per_sample values, coefficients fp32 [F] on the device.
 * HeunEDMSampler (sampling.py:236-254): x + dt/2 (d + d') with d = (x - D)/sigma, d' = (x_e - D')/sigma'
 *   = (1 + dt/(2 sigma)) x - dt/(2 sigma) D + dt/(2 sigma') x_e - dt/(2 sigma') D'.
 * DPMPP2MSampler (sampling.py:305-379): (sigma'/sigma) x - expm1(-h) ((1 + 1/(2r)) D - 1/(2r) D_old). */
int hi3d_sampler_lincomb4(float* out, const float* x0, const float* x1, const float* x2, const float* x3, const float* c0,
                          const float* c1, const float* c2, const float* c3, int F, int64_t per_sample, void* stream);

/* hi3d_sampler_pre for every guider and for churned EDM steps.  guided = 1: out holds 2F rows, uc half first, as
 * hi3d_sampler_pre; guided = 0 (IdentityGuider, guiders.py:24-29): F rows of x and concat_c only.  sigma fp32 [F] is the noise
 * level the network sees.  eps (optional) fp32 NCHW [F, Cx, H, W]: the network sees the churned
 * x_hat = x + (eps * s_noise) * sqrt(sigma^2 - sigma_from^2) (EDMSampler, sampling.py:94-97; sigma = sigma_hat), which is also
 * written to x_hat_out (required with eps) for the post step. */
int hi3d_sampler_pre_ex(const float* x, const float* sigma, const float* sigma_from, const float* eps, float s_noise,
                        const void* concat_uc, const void* concat_c, int concat_is_fp32, int guided, int F, int Cx, int Cc,
                        int H, int W, int Cpad, void* out, float* c_noise_out, float* x_hat_out, void* stream);

/* The post step of every guider with an ancestral update (AncestralSampler, sampling.py:158-170; get_ancestral_step gives
 * sigma_to = sigma_down and sigma_up).  scale fp32 [T] (frame t = f % T): net holds 2F rows, CFG-combined as in
 * hi3d_sampler_post; scale NULL: net holds F rows (IdentityGuider).  x_out = x + (x - D)/sigma * (sigma_to - sigma), then
 * + (eps * s_noise) * sigma_up where sigma_next > 0 when eps (fp32 NCHW [F, Cx, H, W]) is given.  denoised_out optional: the
 * guided D(x, sigma) (DPM-Solver++(2S) extrapolates from it). */
int hi3d_sampler_post_ancestral(const void* net, int net_ld, const float* x, const float* sigma, const float* sigma_to,
                                const float* scale, int T, const float* eps, float s_noise, const float* sigma_up,
                                const float* sigma_next, int F, int Cx, int H, int W, float* x_out, float* denoised_out,
                                void* stream);

/* out = sum_k c_k[f] * x_k over nterms = 1..8 terms; xs / cs are HOST arrays of nterms device pointers (fp32 tensors of F
 * samples x per_sample values, coefficients fp32 [F]).  LinearMultistepSampler (sampling.py:190-225) of order 4 is one launch
 * over (x, D) of the last four steps; DPMPP2SAncestralSampler (sampling.py:279-301) selects its update and adds the ancestral
 * noise in one launch. */
int hi3d_sampler_lincomb(float* out, const float* const* xs, const float* const* cs, int nterms, int F, int64_t per_sample,
                         void* stream);

/* Stage-2 re-noise blend (pipeline_i2v_eval_v02.py:131-132): lat = lat*(1-a) + (init*sigma + z)*a, fp32. */
int hi3d_renoise_blend(float* lat, const float* init, const float* z, float alpha, float sigma, int64_t n,
                       void* stream);

/* Layout / dtype helpers: NCHW (fp32 or fp16) -> NHWC fp16 with channel padding, and NHWC fp16 -> NCHW fp32/fp16
 * (first C channels), used at the VAE / latent boundaries (autoencoder.py:468-505, diffusion.py:117-150). */
int hi3d_nchw_to_nhwc(const void* in, int in_is_fp32, int N, int C, int H, int W, int Cpad, float scale, void* out,
                      void* stream);
int hi3d_nhwc_to_nchw(const void* in, int in_ld, int N, int C, int H, int W, float scale, void* out, int out_is_fp32,
                      void* stream);

/* Patch rows of a CLIP vision tower (open_clip / OpenAI CLIP VisionTransformer.conv1, a stride = kernel = `patch` conv without
 * bias, as one plain hi3d_gemm_tc5 against conv1.weight.reshape(width, 3*patch*patch) zero-padded to Kpad columns).
 * img: NCHW [n, 3, H, W] fp32 or fp16, H and W multiples of `patch`; normalize = 1 applies the CLIP mean / std
 * ((x - mean) / std, (0.48145466, 0.4578275, 0.40821073) / (0.26862954, 0.26130258, 0.27577711)) on the way.
 * out: fp16 [n * (1 + P), Kpad], P = (H/patch)*(W/patch): per image an all-zero row (the class-token slot) then the P patches
 * in raster order, K ordered (c, ky, kx), columns >= 3*patch*patch zero.  Kpad: multiple of 8. */
int hi3d_clip_patchify(const void* img, int img_is_fp32, int n, int H, int W, int patch, int normalize, int Kpad, void* out,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * MiDaS DPT-Hybrid depth tower (annotator/midas/{dpt_depth,vit,blocks}.py, timm vit_base_resnet50_384; hi3d_official_b200/midas.py).
 * Its convs and linears are hi3d_gemm_tc5 calls; these kernels do what the GEMM epilogues cannot.
 * --------------------------------------------------------------------------------------------- */
/* Patch rows of BiT's 7x7 stride-2 stem conv with TF "same" zero padding (timm StdConv2dSame: before the first row
 * ((ceil(H/2) - 1) * 2 + 7 - H) / 2, i.e. 2 for even H; columns alike), for one plain GEMM against the standardised
 * weight.reshape(Co, 147) zero-padded to Kpad columns.  img: NCHW [n, 3, H, W] fp32 or fp16; out: fp16
 * [n * ceil(H/2) * ceil(W/2), Kpad], K ordered (c, ky, kx), columns >= 147 zero.  Kpad: multiple of 8, >= 147. */
int hi3d_dpt_stem_rows(const void* img, int img_is_fp32, int n, int H, int W, int Kpad, void* out, void* stream);
/* 3x3 stride-2 max-pool with TF "same" padding by -inf (timm MaxPool2dSame after the stem): x fp16 NHWC [n, H, W, C] ->
 * y [n, ceil(H/2), ceil(W/2), C]; for even sizes the pad is one row / column after the image.  C multiple of 8. */
int hi3d_maxpool3x3s2_same(const void* x, int n, int H, int W, int C, void* y, void* stream);
/* y = [ReLU](GroupNorm32(x) + addend) in one pass, for the bottlenecks of BiT (timm ResNetV2 Bottleneck, preact=False:
 * act3(norm3(conv3) + shortcut)) and its stem's GroupNorm + ReLU.  x fp16 [n_images * rows_per_image, C]; its group statistics
 * come from `stats`, the hi3d_groupnorm_unit_stats table of x (fp32 [n_images, C / unit, 2]); gamma /
 * beta fp32 [C].  The addend is NULL, a raw fp16 tensor of x's shape (add_stats NULL), or a second GroupNorm-affine tensor
 * GroupNorm32(add) with its own table and parameters (the projection shortcut of a stage's first block).  Statistics are
 * combined in fp64; the arithmetic is fp32 and y is rounded once.  y may be haloed: image i starts at row
 * i * y_sample_rows + y_row_off (0, 0 = dense).  C multiple of 32 and 8, <= 2048; unit divides C / 32. */
int hi3d_groupnorm_apply_add(const void* x, const float* stats, const float* gamma, const float* beta, const void* add,
                             const float* add_stats, const float* add_gamma, const float* add_beta, int C, int unit, int n_images,
                             int64_t rows_per_image, float eps, int apply_relu, void* y, int64_t y_sample_rows,
                             int64_t y_row_off, void* stream);
/* F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) of the fusion blocks and the head (blocks.py
 * FeatureFusionBlock_custom, Interpolate) on fp16 NHWC [n, H, W, C] -> y [n, 2H, 2W, C], plus an optional addend of y's shape
 * (the next fusion block's xs[0] + resConfUnit1(xs[1])), in fp32 with one rounding.  C multiple of 8. */
int hi3d_upsample2x_bilinear_ac(const void* x, int n, int H, int W, int C, const void* add, void* y, void* stream);
/* y = max(x, 0) over n fp16 values (n multiple of 8): the ReLU that opens a residual conv unit (blocks.py
 * ResidualConvUnit_custom), whose input x is still needed for the unit's residual. */
int hi3d_relu_copy(const void* x, int64_t n, void* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * U^2-Net background removal (U-2-Net model/u2net.py, the default network of rembg's `remove`; hi3d_official_b200/u2net.py).
 * Its convs (3x3, dilations 1 / 2 / 4 / 8, BatchNorm folded, ReLU epilogue, the RSU's `+ hxin` as the residual epilogue) are
 * hi3d_gemm_tc5 calls; these kernels do the rest.  x_ld / y_ld are the channel strides of source and destination, so either
 * may be a channel slice of a wider (concat) buffer: pass the slice's first element.  C, x_ld, y_ld multiples of 8.
 * --------------------------------------------------------------------------------------------- */
/* nn.MaxPool2d(2, 2, ceil_mode=True) (RSU pool1..pool5, U2NET pool12..pool56): fp16 NHWC [n, H, W, C] -> [n, ceil(H/2),
 * ceil(W/2), C]; a window over the bottom / right edge takes the max of its valid elements. */
int hi3d_maxpool2x2_ceil(const void* x, int x_ld, int n, int H, int W, int C, void* y, int y_ld, void* stream);
/* F.interpolate(size=(Ht, Wt), mode='bilinear', align_corners=False) (u2net.py _upsample_like): fp16 NHWC [n, Hs, Ws, C] ->
 * [n, Ht, Wt, C], any sizes.  Source coordinate max(0, (dst + 0.5) * Hs / Ht - 0.5) with Hs / Ht and the fused multiply-add in
 * fp32; the blend in fp32 with one rounding. */
int hi3d_resize_bilinear(const void* x, int x_ld, int n, int Hs, int Ws, int C, void* y, int y_ld, int Ht, int Wt, void* stream);
/* Output 0 of U2NET.forward, sigmoid(outconv(cat(d1..d6))) with every d_k upsampled to H x W, when outconv's weights are folded
 * into the side heads: out = sigmoid(b0 + sum_k resize(side_k)), fp32 [n, H, W].  sides[k]: fp16 NHWC [n, side_h[k],
 * side_w[k], side_ld[k]], channel 0 read; the arrays are host memory of n_sides (<= 8) entries. */
int hi3d_u2net_fuse_sides(const void* const* sides, const int* side_ld, const int* side_h, const int* side_w, int n_sides, float b0,
                          int n, int H, int W, float* out, void* stream);

/* DiagonalGaussianDistribution.sample / mode (distributions.py:24-41,71) * scale_factor (diffusion.py:149):
 * moments fp16 NHWC [N, H, W, ld] (mean = ch 0..C-1, logvar = ch C..2C-1), noise fp32 NCHW or NULL (mode),
 * out fp32 NCHW [N, C, H, W]. */
int hi3d_gaussian_sample(const void* moments, int ld, const float* noise, int N, int C, int H, int W, float scale,
                         float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Peer memory for the frame-sharded step (one process per GPU; SURVEY 8e).  No reference counterpart.
 * --------------------------------------------------------------------------------------------- */
/* Symmetric buffers: hi3d_symm_alloc = cudaMalloc + zero fill + cudaIpcGetMemHandle (handle64: 64 bytes the host ships to
 * the other ranks, e.g. with torch.distributed.all_gather_object); hi3d_symm_open maps a peer's buffer into this process
 * (cudaIpcOpenMemHandle, enabling peer access); hi3d_symm_close / hi3d_symm_free undo them. */
int hi3d_symm_alloc(int64_t bytes, void** ptr, void* handle64);
int hi3d_symm_open(const void* handle64, void** ptr);
int hi3d_symm_close(void* ptr);
int hi3d_symm_free(void* ptr);
/* Size of one rank's exchange area (flags + payload slots + epoch word) for hi3d_peer_exchange. */
int64_t hi3d_peer_xchg_bytes(int world);
/* One exchange point of the sharded step, a single-CTA kernel on `stream`: every rank announces a new epoch in its slot of
 * every peer's flag array and waits until all peers have announced it -- everything the ranks stored into each other's
 * buffers before this point is visible after it.  With n > 0 (<= 1024) it is also an all-reduce: out[j] = sum over ranks of
 * payload[j] in rank order (the [B, 32, 2] partial sums of the temporal GroupNorm, video_model.py:71-76).  xchg[r] = rank
 * r's exchange area (zero-initialised symmetric memory); every rank must issue the same sequence of exchanges. */
int hi3d_peer_exchange(void* const* xchg, int rank, int world, const float* payload, int n, float* out, void* stream);

/* One-time weight packing (device -> device), the C twin of hi3d_official_b200/pack.py for hosts without torch:
 * reference layouts as stored in the checkpoints -- nn.Linear [Co, Ci] (taps = 1; attention.py:269-278, 87-113),
 * Conv2d OIHW (taps = kh*kw; openaimodel.py:107-207, 263-304, model.py:67-151), Conv3d (Co, Ci, 3, 1, 1) (taps = 3;
 * video_model.py:45-60) -- into the fp16 [cout_pad, taps * cin_pad] K-major matrix of hi3d_gemm (K ordered (tap, ci),
 * zero padded).  geglu_interleave: rows of the GEGLU projection [value ; gate] are interleaved (value_j, gate_j).
 * hi3d_pack_bias: fp32 [n_pad] (b may be NULL -> zeros).  Caller owns all buffers. */
int hi3d_pack_weight(const void* w, int w_is_fp32, int Co, int Ci, int taps, int cin_pad, int cout_pad,
                     int geglu_interleave, void* out, void* stream);
int hi3d_pack_bias(const void* b, int b_is_fp32, int n, int n_pad, int geglu_interleave, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HI3D_B200_H_ */
