/* gcd_b200 — C ABI of the H100-native (sm_90a) GCD denoising hot path.
 *
 * The reference (basilevh/gcd, gcd-model/sgm) is pure Python/PyTorch and has NO FFI of its own
 * (SURVEY.md §8(b)); the drop-in boundary upstream is the `instantiate_from_config` plugin surface
 * (gcd-model/sgm/util.py:168-185). This header is the C boundary *underneath* the plugin classes in
 * gcd_b200/ (VideoUNet, Denoiser, EulerEDMSampler, VideoDecoder): each entry point states which reference
 * torch call(s) it replaces. Conventions (all entry points):
 *   - raw DEVICE pointers, caller-owned, never freed or retained by the library;
 *   - plain ints / POD structs, no torch types;  `stream` is a cudaStream_t passed as void*;
 *   - returns 0 on success, negative on error; message via gcd_last_error() (thread-local);
 *   - kernels are asynchronous on `stream`.
 * 16-bit tensors ("act") are IEEE fp16 unless the library was built with -DGCD_ACT_BF16
 * (query with gcd_act_dtype()). Activations are channels-last: [frames, H, W, C] == [rows, C].
 */
#ifndef GCD_B200_H
#define GCD_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* gcd_last_error(void);
int gcd_version(void);
/* 0 = fp16 operands, 1 = bf16 operands */
int gcd_act_dtype(void);
/* number of kernels launched by this library since load (bench.py `gpu_launches`) */
int64_t gcd_launch_count(void);

/* Fused epilogue applied to every tensor-core op (rows r of the output, columns n):
 *   x      = acc[r,n] + bias[n] + rowvec[(r / rows_per_vec) * ld_rowvec + n]
 *   x      = act(x)                      (act: 0 none, 1 SiLU, 2 exact GELU 0.5 x (1 + erf(x / sqrt 2)) = nn.GELU(),
 *                                          3 ReLU = nn.ReLU (LPIPS's VGG16 convolutions))
 *   geglu: columns come in interleaved blocks of 16 value / 16 gate;  x = value * gelu_erf(gate)
 *          and the output has N/2 columns          (attention.py:87-94 GEGLU)
 *   out    = a_acc * x + a_res1 * res1[r,n] + a_res2 * res2[r,n]
 * which covers: conv bias, `h + emb_out[..., None, None]` (openaimodel.py:349-355), residual adds
 * (openaimodel.py:357, attention.py:551-572), AlphaBlender (util.py:341-369), len-1 cross-attention bias.
 */
typedef struct gcd_epilogue {
    const float* bias;     /* [N] or NULL */
    const float* rowvec;   /* [n_groups, ld_rowvec] or NULL */
    int32_t rows_per_vec;
    int32_t ld_rowvec;
    const void* res1;      /* [rows, ld_res1] or NULL */
    int32_t ld_res1;
    int32_t res1_f32;      /* 1: float32, 0: act */
    const void* res2;
    int32_t ld_res2;
    int32_t res2_f32;
    float a_acc, a_res1, a_res2;
    void* out;             /* [rows, ld_out] */
    int32_t ld_out;
    int32_t out_f32;
    int32_t geglu;
    int32_t act;
    /* Optional fused GroupNorm statistics of the tensor being written (the NEXT GroupNorm's input):
     * gn_stats[(row / gn_rows_per_img) * gn_groups + col / gn_cpg][0..1] += (sum, sum of squares) of the stored values.
     * Zero the buffer first. Only produced when every output tile (64 rows for ops with a residual or an fp32 output, else 128) lies inside one statistics image and all
     * tiles are full; otherwise gcd_tc_run returns 1 (success, statistics NOT produced: run gcd_groupnorm_stats). */
    double* gn_stats;
    int32_t gn_cpg;
    int32_t gn_groups;
    int64_t gn_rows_per_img;
} gcd_epilogue;

/* Generic wgmma implicit-GEMM:  acc[r, n] = sum_{tap, c} A[(x,y,z)(r) * in_mul + tap_off(tap), c] * W[n, tap*Cin + c]
 * A is a 4-D channels-last act tensor (C innermost, then X, Y, Z) with element strides; out-of-range
 * coordinates read as zero (= conv zero padding). Output rows are (z*Yo + y)*Xo + x.
 * Replaces nn.Linear / nn.Conv2d(3x3, 1x1, stride 1|2) / nn.Conv3d((3,1,1)) / torch.bmm on the hot path. */
typedef struct gcd_tc_op {
    const void* A;
    int32_t C;                 /* channels per tap (multiple of 8) */
    int32_t Xi, Yi, Zi;        /* input extents */
    int64_t sx, sy, sz;        /* input strides in elements (channel stride is 1) */
    int32_t Xo, Yo, Zo;        /* output extents */
    int32_t in_mul;            /* 1, or 2 for stride-2 conv */
    int32_t ntaps;             /* 1..9 */
    int8_t tap_dx[9], tap_dy[9], tap_dz[9];
    int32_t gemm_tile;         /* 1: plain GEMM tiling (one tile = consecutive x), 0: search conv tile */
    const void* W;             /* [N, ldw] act, K-contiguous, ldw >= ntaps*C ; batched over y if w_batch_stride != 0 */
    int64_t ldw;
    int64_t w_batch_stride;    /* elements between per-y weight matrices (batched GEMM), else 0 */
    int32_t N;                 /* accumulator columns */
    gcd_epilogue ep;
} gcd_tc_op;
/* returns 0 on success, 1 on success without the requested fused GroupNorm statistics, < 0 on error */
int gcd_tc_run(const gcd_tc_op* op, void* stream);

/* ---- normalisation (HBM-bound kernels) ------------------------------------------------------------------ */
/* GroupNorm statistics over `rows_per_group_img` rows x (C/groups) channels: util.py:274-276 GroupNorm32,
 * attention.py:125-128 Normalize. in: [n_img*rows, C] float32 (in_f32=1) or act. stats: double[n_img*groups*2]
 * (sum, sumsq), must be zeroed by the caller (gcd_memset_async) before the call. The sums are accumulated in fp64 from
 * each element on, so the variance gcd_groupnorm_apply derives from them (sumsq/n - mean^2) holds for groups whose mean
 * is large against their spread. */
int gcd_groupnorm_stats(const void* in, int in_f32, int64_t n_img, int64_t rows, int C, int groups, double* stats,
                        void* stream);
/* y = (x-mean)*rstd*gamma+beta, optional SiLU, written as act. */
int gcd_groupnorm_apply(const void* in, int in_f32, int64_t n_img, int64_t rows, int C, int groups,
                        const double* stats, const float* gamma, const float* beta, float eps, int silu, void* out,
                        void* stream);
/* LayerNorm over C per row (attention.py BasicTransformerBlock norm1-3, video_attention.py norm_in/1/2/3).
 * in: float32 [rows, C]. Optional `add` [n_add, C] float32 is added first with index (row / add_rows_per) % add_mod
 * (video_attention.py:266-287 time_pos_embed). When sum_out is non-NULL, the tensor that is normalised (in + add, or in
 * alone without `add`) is written to it as float32, for every C. */
int gcd_layernorm(const float* in, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                  const float* add, int64_t add_rows_per, int64_t add_mod, float* sum_out, void* out, void* stream);
/* The same LayerNorm (with the same optional `add`) written as float32 [rows, C]: open_clip VisionTransformer's ln_pre, whose
 * output is the residual stream of the tower. `out` must not alias `in`. */
int gcd_layernorm_f32(const float* in, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                      const float* add, int64_t add_rows_per, int64_t add_mod, float* out, void* stream);

/* ---- attention ------------------------------------------------------------------------------------------- */
/* Spatial self-attention softmax(QK^T/sqrt(64))V, head_dim 64 (attention.py:255-344 CrossAttention with
 * context=None). qkv: act [frames, tokens, 3*heads*64] = (q | k | v), head index outer within each third.
 * out: act [frames, tokens, heads*64]. */
int gcd_attention_spatial(const void* qkv, int frames, int tokens, int heads, void* out, void* stream);
/* Temporal self-attention over T frames per (clip, spatial position) (video_attention.py:109-140 attn1 after the
 * "(b t) s c -> (b s) t c" rearrange, done here by indexing). qkv/out laid out as above with frames = clips*T. */
int gcd_attention_temporal(const void* qkv, int clips, int T, int tokens, int heads, void* out, void* stream);
/* ViT self-attention with head_dim 80 (open_clip ViT-H/14 resblocks: nn.MultiheadAttention, 16 heads, 257 tokens):
 * softmax(q k^T / sqrt(80)) v per (image, head) with fp32 softmax; scores are never written to memory.
 * qkv: act [n, L, 3*heads*80] = in_proj output (q | k | v, head index outer within each third); out: act [n, L, heads*80].
 * L in 1..1024. */
int gcd_attention_d80(const void* qkv, int n, int L, int heads, void* out, void* stream);
/* Row softmax of float32 scores [rows, cols] * scale -> act probs (model.py:161-201 AttnBlock, d=512 single head). */
int gcd_softmax_rows(const float* in, int64_t rows, int cols, float scale, void* out, void* stream);

/* ---- element-wise / layout ------------------------------------------------------------------------------- */
int gcd_memset_async(void* p, int value, int64_t bytes, void* stream);
/* float32 [rows, C] -> act [rows, C] */
int gcd_cast_f32_to_act(const float* in, int64_t n, void* out, void* stream);
/* nearest x2 upsample of channels-last float32 [n,H,W,C] -> act [n,2H,2W,C] (openaimodel.py:110-160, model.py:58-71) */
int gcd_upsample2x_to_act(const float* in, int n, int H, int W, int C, void* out, void* stream);
/* channel concat of two float32 channels-last tensors: out[r, :Ca]=a, out[r, Ca:]=b  (video_model.py:525 th.cat) */
int gcd_concat_channels(const float* a, int Ca, const float* b, int Cb, int64_t rows, float* out, void* stream);
/* the same concat of [n_img*rows, Ca] and [n_img*rows, Cb] fused with the GroupNorm statistics of the result (the skip concat
 * of the UNet's output blocks feeds a ResBlock whose first op is GroupNorm32, openaimodel.py / video_model.py:536-540):
 * stats[n_img, groups, 2] float64 (sum, sum of squares), zeroed by the caller, accumulated in a fixed order per block. */
int gcd_concat_channels_stats(const float* a, int Ca, const float* b, int Cb, int64_t n_img, int64_t rows, int groups,
                              float* out, double* stats, void* stream);
/* Same, the concatenated tensor written in the 16-bit activation type only (statistics of the fp32 inputs): for consumers that read
 * 16-bit operands anyway — the UNet's output ResBlocks (cin != cout: 1x1 skip conv + first GroupNorm), openaimodel.py `th.cat`. */
int gcd_concat_channels_stats_act(const float* a, int Ca, const float* b, int Cb, int64_t n_img, int64_t rows, int groups,
                                  void* out, double* stats, void* stream);
/* act(x) on act tensor: SiLU (emb_layers SiLU, openaimodel.py:262-268) */
int gcd_silu_act(const void* in, int64_t n, void* out, void* stream);
/* SiLU on a float32 tensor, written as act (emb_layers' nn.SiLU on `emb`, openaimodel.py:262-268) */
int gcd_silu_f32_to_act(const float* in, int64_t n, void* out, void* stream);
/* NCHW float32 [N,C,HW] -> channels-last act [N,HW,Cpad] (zero-padded channels): entry glue of VideoUNet.forward /
 * VideoDecoder.forward when called through the plugin surface with torch NCHW tensors. */
int gcd_nchw_to_act_nhwc(const float* in, int N, int C, int HW, int Cpad, void* out, void* stream);
/* channels-last float32 [N,HW,ld] (first C columns) -> NCHW float32 [N,C,HW]: exit glue. */
int gcd_nhwc_to_nchw_f32(const float* in, int ld, int N, int C, int HW, float* out, void* stream);
/* AE3DConv.time_mix_conv (temporal_ae.py:86-107): Conv3d(3->3,(3,1,1)) over frames of the VAE's 3-channel output.
 * in: channels-last float32 [B*T, HW, ld] (first 3 columns); w: [3,3,3] (co,ci,kt); out: NCHW float32 [B*T,3,HW]. */
int gcd_vae_time_mix(const float* in, int ld, int B, int T, int HW, const float* w, const float* b, float* out,
                     void* stream);
/* timestep_embedding (util.py:207-231): t[n] float32 -> act [n, dim] = cat(cos, sin)(t * exp(-ln(max_period) k / half)) */
int gcd_timestep_embedding(const float* t, int n, int dim, float max_period, void* out_act, float* out_f32,
                           void* stream);

/* SphericalEmbedder.forward (encoders/modules.py:247-287; SURVEY.md 8(f) rank 1): x[n,3] = (azimuth, elevation, radius) float32
 * -> out[n,dim] float32 = [cos/sin of 1x,2x,4x azimuth | same for elevation | radius] * w[dim,13]^T + b[dim]. */
int gcd_spherical_embed(const float* x, int n, const float* w, const float* b, int dim, float* out, void* stream);

/* FrozenOpenCLIPImageEmbedder.preprocess (encoders/modules.py:703-715) + the ViT's conv1 patch unfold, fp32 arithmetic:
 * kornia 0.7.0 resize(x, (224, 224), bicubic, align_corners=True, antialias) -> (x + 1) / 2 -> (x - mean[c]) / std[c].
 * in: float32 NCHW [n, 3, H, W]. Antialias (when ks_x > 0): separable Gaussian blur, taps_x (ks_x, odd) along W first, then
 * taps_y along H, 'reflect' border; taps are device float32 arrays computed by the host. Then PyTorch bicubic
 * (A = -0.75, align_corners=True, clamped taps); a 224x224 input is used unchanged (no blur, no resize).
 * scratch: float32 [2*n*3*H*W] when blurring, else unused. mean_std: device float32 {mean[3], std[3]}.
 * out: [n*257, 640], act (out_f32 = 0) or float32 (1); row 0 of every image is zero (class-token slot), row
 * 1 + py*16 + px holds the 14x14x3 patch at (py, px) ordered (ky, kx, c) in columns 0..587, columns 588..639 zero. */
int gcd_clip_preprocess(const float* in, int n, int H, int W, const float* taps_x, int ks_x, const float* taps_y, int ks_y,
                        float* scratch, const float* mean_std, void* out, int out_f32, void* stream);

/* ---- sampler step (sampling.py:101-121, denoiser.py:23-49, guiders.py:79-100, wrappers.py:23-34) ------------ */
/* The scalar coefficients c_in/c_out/c_skip (denoiser_scaling.py:53-61) and dt = sigma_next - sigma_hat are computed
 * by the host with the same torch fp32 CPU ops as the reference and passed in, so scheduler arithmetic is bit-exact.
 * Builds the CFG-doubled network input: out act [2*BT, H, W, 64] channels-last, channels 0..3 = x * c_in,
 * 4..7 = concat cond (zeros for the unconditional half), 8..63 = 0. x: float32 NCHW [BT,4,H,W];
 * cond_concat: float32 NCHW [BT,4,H,W]; uc_concat likewise (may be NULL = zeros). */
int gcd_sampler_prep(const float* x, const float* uc_concat, const float* c_concat, int BT, int H, int W, float c_in,
                     void* out, void* stream);
/* net_out: float32 channels-last [2*BT, H, W, ld_net] (first 4 columns used), x updated IN PLACE (NCHW float32):
 *   den_k = net_k * c_out + x * c_skip ; den = den_u + scale[t](den_c - den_u) ; d = (x - den)/sigma ;
 *   x += d * dt.  scale: float32 [T] (frame index = bt % T). */
int gcd_sampler_update(float* x, const float* net_out, int ld_net, int BT, int T, int H, int W, float c_out,
                       float c_skip, float sigma, float dt, const float* scale, void* stream);

/* Experiments only (tools/autotune_tc.py): force the tile width (128 / 160 / 256) of the following gcd_tc_run calls; 0 = automatic.
 * `mode` is ignored (kept for ABI compatibility). Not thread-safe. */
void gcd_tc_override(int bn, int mode);

/* Evaluation-loop image metrics (gcd-model/scripts/test.py:346-496 calculate_metrics; SSIM = scikit-image 0.22.0
 * structural_similarity(data_range=1, channel_axis=0), masked form = gcd-model/scripts/eval_utils.py:571-664 masked_ssim).
 * pred, gt: float32 [frames, 3, H, W] in [0, 1]; mask: uint8 [frames, H, W] or NULL. out: float64 [frames, 8], zeroed here:
 *   {sum (pred-gt)^2, count, same over mask, count, sum SSIM map (3-pixel border cropped), count, same over the 3x eroded mask, count},
 * sums over the 3 channels. PSNR = 10 log10(count / sum) for data_range 1; SSIM = sum / count.
 * The per-pixel arithmetic is the reference's float32 arithmetic: (pred-gt)^2 squared in fp32; window means as scipy's
 * uniform_filter forms them (fp32 products, a vertical then a horizontal 7-tap pass, each summed in fp64 and rounded to fp32
 * once); the SSIM formula in fp32 in numpy's order without FMA contraction. Identical images give SSIM exactly 1. */
int gcd_frame_metrics(const float* pred, const float* gt, const uint8_t* mask, int frames, int H, int W, double* out, void* stream);

/* Point-cloud view synthesis of the evaluation clips (gcd-model/sgm/data/geometry.py:242-444 project_points_to_pixels +
 * spreaded_index_add + blur_into_black, then the bilinear resize and `* 2 - 1` of kubric_arbit.py:410-563 / pardom_arbit.py:585-738).
 * R renders in one call. Render r reads points [desc[r].p0, desc[r].p0 + desc[r].n) of frame desc[r].frame:
 *   xyz: fp16 [frames, P, 3] world coordinates (non-finite allowed: such points are dropped); rgb: uint8 [frames, P, 3];
 *   segm: uint8 [frames, P] semantic ids with palette float32 [256, 3], or both NULL. With segm, colour = (1 - a) rgb/255 + a palette[id]
 *   in fp32 with a = cams[r][21].
 *   desc: int32 [R, 4] = {frame, p0, n, blur kernel (odd, 1..31; sigma = k / 4)}, on the device; desc_host: the same array on the host.
 *   cams: fp64 [R, 24] on the device = {K (3x3 row-major, pixel units), RT[0:3, 0:3] (row-major), RT[0:3, 3], a, 0, 0}.
 * Render size H x W, output size Hp x Wp; spread_radius 0..8 (spreaded_index_add's offsets, weight x 0.02).
 * acc: fp64 [R, H*W, 4] workspace and maxd: fp64 [R], both zeroed here. On return maxd[r] is the largest depth of the render's valid
 * points, 0 when no point lands in the image (out is then the all-black render; the caller reports the error).
 * out: float32 [R, 3, Hp, Wp] in [-1, 1]. Errors: -2 bad arguments (null pointer, point range, kernel size, blur radius >= H or W). */
int gcd_render_views(const void* xyz, const uint8_t* rgb, const uint8_t* segm, const float* palette, int64_t P, int R,
                     const int32_t* desc_host, const int32_t* desc, const double* cams, int H, int W, int Hp, int Wp,
                     int spread_radius, double* acc, double* maxd, float* out, void* stream);

/* Input frames of gcd-model/scripts/infer.py (sgm/data/common.py:121-199 process_image / load_video_mp4 after decoding, then
 * infer.py:137 `(x + 1) / 2`). in: uint8 [n, H, W, C] decoded frames, C = 3 or 4 (the fourth channel is ignored); output channel c
 * reads input channel channel_map[c] (HOST int32 [3], entries 0..2: {0, 1, 2} for RGB, {2, 1, 0} for cv2's BGR). Crop box rows
 * [y0, y0 + ch), columns [x0, x0 + cw) (the host computes center_crop_numpy's box). p = u8 / 255 in fp32, resized from ch x cw
 * to Ho x Wo as cv2.resize(INTER_LINEAR) does on float32 images (scale = in / out in fp64, source coordinate
 * (d + 0.5) * scale - 0.5 rounded to fp32, floor, fraction 0 and index clamped at both borders, weights (1 - f, f) in fp32,
 * horizontal pass then vertical, unfused fp32 products and sums); no resize when the crop already has the output size.
 * out: float32 [frames, 3, Ho, Wo] in [0, 1], input frame f written to frame out_frame[f] (device int32 [n]) or f when out_frame is
 * NULL; value ((p * 2 - 1) + 1) / 2 in fp32. Errors: -2 bad arguments (null pointer, sizes, crop box outside the frame, map). */
int gcd_frames_prepare(const uint8_t* in, int n, int H, int W, int C, const int32_t* channel_map, int y0, int x0, int ch, int cw,
                       int Ho, int Wo, const int32_t* out_frame, float* out, void* stream);

/* RGB-D unprojection of the dataset conversion (data-gen/data_utils.py:91-138 unproject_pixels_to_points + camera_to_world; Kubric's
 * correct_depth_ball_plane_torch, convert_pcl_kubric.py:96-121; ParDom's clamp, convert_pcl_pardom.py:166). depth: float32 [n, H, W],
 * one image per (frame, view). cams: device float32 [n, GCD_UNPROJECT_CAM] = {fx, fy, cx, cy (pixels), R = RT[0:3, 0:3] row-major,
 * t = RT[0:3, 3]} as the reference builds them. mode GCD_UNPROJECT_BALL_TO_PLANE: z = depth / sqrt((tan(ax)^2 + tan(ay)^2) + 1) with
 * the pixel's angles from torch.linspace(-fov/2, fov/2) and fov = 2 atan(rcp(2 |f|) * size); mode GCD_UNPROJECT_CLAMP:
 * z = clamp(depth, 0, max_depth), NaN kept. x = ((u - cx) z) / fx, y = ((v - cy) z) / fy, world_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i,
 * every operation one fp32 rounding. out: fp16 [n, H*W, 3], point v*W + u, round-to-nearest-even (overflow -> +-inf).
 * Errors: -2 bad arguments (null pointer, n or H above 65535, unknown mode). */
#define GCD_UNPROJECT_CAM 16
#define GCD_UNPROJECT_CLAMP 0
#define GCD_UNPROJECT_BALL_TO_PLANE 1
int gcd_unproject_depth(const float* depth, int n, int H, int W, const float* cams, int mode, float max_depth, void* out, void* stream);

/* LPIPS perceptual metric, VGG16 variant (gcd-model/sgm/modules/autoencoding/lpips/loss/lpips.py; DiffusionEngine.validation_step,
 * models/diffusion.py:317-362). The 13 convolutions are gcd_tc_run ops with act = 3 (ReLU); these are the remaining stages.
 * Input stage: in float32 NCHW [n, 3, H, W] in [-1, 1]; shift, scale: device float32 [3] (ScalingLayer: (x - shift) / scale, fp32).
 * out: act [n*H*W, 64], row (f*H + y)*W + x: column (ky*3 + kx)*3 + c holds the scaled pixel (y + ky - 1, x + kx - 1, c), 0 outside
 * the image (zero padding of the scaled image); columns 27..63 are 0. conv1_1 is then one 1-tap K = 64 GEMM. */
int gcd_lpips_input(const float* in, int n, int H, int W, const float* shift, const float* scale, void* out, void* stream);
/* MaxPool2d(2, 2), floor mode: act [n, H, W, C] channels-last -> act [n, H/2, W/2, C] (odd H or W drop the last row or column).
 * C % 8 == 0, both tensors 16-byte aligned. */
int gcd_maxpool2x2(const void* in, int n, int H, int W, int C, void* out, void* stream);
/* LPIPS head of one tapped layer (relu1_2 .. relu5_3). feat: act [frames, HW, C] channels-last, C in {64, 128, 256, 512};
 * pairs: device int32 [n_pairs, 2] frame indices (input, target); w: device float32 [C] (lin<k>.model.1.weight).
 * out[p] = mean over the HW pixels of sum_c w[c] (a[c] / (|a| + 1e-10) - b[c] / (|b| + 1e-10))^2 with a, b the two frames'
 * features at the pixel (norms over channels, fp32), written as float64. The reduction order is fixed: same inputs, same bits.
 * partial: float64 [n_pairs * ceil(HW / GCD_LPIPS_HEAD_PIX)] workspace. count: uint32 [n_pairs], zero on entry; the kernel leaves
 * it zero, so it is zeroed once when allocated. */
#define GCD_LPIPS_HEAD_PIX 128
int gcd_lpips_head(const void* feat, int HW, int C, const int32_t* pairs, int n_pairs, const float* w, double* partial,
                   uint32_t* count, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
