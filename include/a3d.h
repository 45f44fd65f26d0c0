/* animate3d_b200 -- C ABI of the H100-native (sm_90a) hot path (liba3d.so).
 *
 * Plain pointers and sizes only; every pointer is a DEVICE pointer unless its name ends in _host.  All entry points
 * enqueue work on `stream` (a cudaStream_t passed as void*) and return 0 on success or a negative A3D_E* code; the
 * message of the last failure on the calling thread is available from a3d_last_error().  Nothing here allocates
 * device memory: the caller owns every buffer (workspace sizes are queried first), which is what makes the whole
 * UNet forward capturable in one CUDA graph.
 *
 * Which reference interface each entry point replaces (reference = yanqinJiang/Animate3D @ 033a1be):
 *   a3d_gemm            torch.nn.functional.linear / conv2d (cuBLAS / cuDNN) under diffusers ResnetBlock2D, Transformer2DModel,
 *                       TransformerTemporalModel, FeedForward/GEGLU -- called from animatediff/models/unet_motion_mv_model.py:768-859
 *   a3d_attention       xformers.ops.memory_efficient_attention at animatediff/models/attention_processor.py:103,233,268,405,416,656,691
 *   a3d_temporal_attn   Attention.get_attention_scores + torch.bmm at animatediff/models/attention_processor.py:634-635
 *   a3d_group_norm      torch GroupNorm(+SiLU) in ResnetBlock2D / Transformer2DModel / TransformerTemporalModel (5-D, over frames)
 *   a3d_layer_norm      torch LayerNorm in BasicTransformerBlock
 *   a3d_conv_in/out     unet_motion_mv_model.py:767-768 (permute + conv_in) and 859-862 (conv_out + permute back)
 *   a3d_ddim_cfg_step   animatediff/pipelines/pipeline.py:1023-1031 (CFG combine + DDIMScheduler.step + frame-0 re-injection)
 *   a3d_ddim_step       the same with eta > 0 (variance noise) and with guidance off (pipeline.py:580-590, 1008-1028)
 *   a3d_clip_preprocess .cpu() -> PIL -> CLIPImageProcessor -> patch embedding of the IP-Adapter image encoder at
 *                       custom/threestudio-animate3d/guidance/animatemv_guidance.py:546-555
 *   a3d_raster_*        diff_gaussian_rasterization._C.rasterize_gaussians / rasterize_gaussians_backward, called at
 *                       custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:161-170
 */
#ifndef A3D_H_
#define A3D_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define A3D_OK 0
#define A3D_EINVAL (-1)   /* bad argument / unsupported shape */
#define A3D_ECUDA (-2)    /* CUDA runtime or driver error     */
#define A3D_ENOTSUP (-3)  /* device is not sm_90              */

const char* a3d_last_error(void);
int a3d_version(void);
/* 0 when the current device is sm_90 and the driver entry points needed for TMA are available. */
int a3d_init(void);

/* ---------------------------------------------------------------- GEMM / implicit-GEMM convolution ----------- */
/* C[M,N] = epilogue( A[M,K] * B[N,K]^T ), fp16 operands, fp32 accumulation on the tensor cores (wgmma).
 * A operand modes: A3D_A_PLAIN  row-major [M, lda]
 *                  A3D_A_CONV3  NHWC image [n_img, H, W, C] gathered as a 3x3 (pad 1, stride 1|2) im2col, K = 9*C,
 *                               k index = (ky*3+kx)*C + c ; M = n_img*OH*OW
 * Epilogue:  v = acc + bias[n] + rowbias[((m / rb_div) % rb_mod) * rb_ld + n]
 *            v = acc_scale * v + r1_scale * R1[m, n] + R2[om, n]          (om = permuted output row, see below)
 *            GEGLU (geglu = 1): columns come in interleaved blocks of 32 (u | g); out[.., j] = u_j * gelu_erf(g_j), N_out = N/2
 *            GELU (geglu = 2): out[.., n] = gelu_erf(v) (CLIP's hidden_act="gelu" MLP); like GEGLU it takes bias / row-bias
 *            only and an fp16 output
 *            out[om, n] stored as fp16 (or fp32 when out_f32)
 * Row permutation (perm_a, perm_b > 0): om = (m / (a*b))*(a*b) + (m % b)*a + (m / b) % a   ("(x a b) -> (x b a)").
 */
enum { A3D_A_PLAIN = 0, A3D_A_CONV3 = 1 };
/* impl: A3D_GEMM_AUTO lets the library pick the kernel from the arguments; A3D_GEMM_TC forces the tensor-core (wgmma)
 * kernels and fails with A3D_EINVAL where they cannot run; A3D_GEMM_SIMT forces a3d_gemm's one-thread-per-element kernel,
 * which AUTO also picks for shapes and alignments the tensor cores cannot take. */
enum { A3D_GEMM_AUTO = 0, A3D_GEMM_TC = 1, A3D_GEMM_SIMT = 2 };

typedef struct a3d_gemm_args {
  const void* A;      /* fp16 */
  const void* B;      /* fp16 weights [N, K], K contiguous */
  void* C;            /* fp16 (or fp32) output */
  int64_t M, N, K;
  int64_t lda, ldc;   /* elements; lda ignored for CONV3 */
  int a_mode;
  int conv_n, conv_h, conv_w, conv_c, conv_stride; /* CONV3 geometry (input) */
  int conv_nopad_lo;          /* CONV3: 0 = zero padding 1 on every side (UNet); 1 = no padding in front of row / column 0 and 1 behind
                                 the last ones = F.pad(x, (0,1,0,1)) + conv(padding=0), the SD-VAE Downsample2D */
  const float* bias;          /* [N] or NULL */
  const float* rowbias;       /* [rb_rows, rb_ld] or NULL */
  int64_t rb_ld, rb_div, rb_mod;
  float acc_scale;            /* multiplies the accumulator: MUST be set (1.0 if unused; 0.0 is honoured, not remapped) */
  const void* R1; int64_t ldr1; float r1_scale;   /* fp16 or NULL; read at the unpermuted row m: it may alias C only
                                                     when perm_a == 0 (with a permutation another row's store can land
                                                     on R1[m, n] before it is read) */
  const void* R2; int64_t ldr2;                   /* fp16 or NULL; read at the output element om, n itself: may be C */
  int geglu;                  /* 0 = none, 1 = GEGLU, 2 = GELU */
  int out_f32;
  int64_t perm_a, perm_b;     /* 0,0 = identity */
  int impl;                   /* A3D_GEMM_AUTO / _TC / _SIMT */
} a3d_gemm_args;

/* Replaces every Linear / Conv2d(3x3) the reference's forward issues through torch: ResnetBlock2D conv1/conv2/
 * time_emb_proj/conv_shortcut, Down/Upsample2D convs, Transformer2DModel proj_in/proj_out + BasicTransformerBlock FF
 * (GEGLU) (diffusers 0.28, reached from animatediff/models/unet_motion_mv_model.py:768-859), and the processors'
 * to_q/to_k/to_v/to_out + *_i2v / *_ip / *_sp projections (animatediff/models/attention_processor.py:211-231, 383-403,
 * 425-441, 600-655, 686-717), with their bias, residual, positional-table and layout epilogues fused. */
int a3d_gemm(const a3d_gemm_args* args, void* stream);

/* Kernel queries: the kernel the matching call would launch for the same arguments, as a NUL-terminated name in name[n]
 * (names are shorter than 48 bytes; a buffer too small for the name is A3D_EINVAL).  They launch nothing, never touch the
 * device or dereference an operand pointer, need no a3d_init, and fail with the same A3D_EINVAL and a3d_last_error() as
 * the call.  A failure to encode a tensor map is reported by the call alone.
 *   a3d_gemm_kernel           "simt", or "tc BN{128|160|256} {plain|res|geglu|gelu|f32} {plain|conv-wide-rows|conv-row-block|
 *                             conv-image-block}": tile width, epilogue instance, A operand tiling
 *   a3d_attention_kernel      "fewkeys" (<= 8 keys), "shortkeys" (9..80 keys, operand rows aligned for it) or "tc"
 *   a3d_temporal_attn_kernel  "frames16" or "generic" */
int a3d_gemm_kernel(const a3d_gemm_args* args, char* name, size_t n);

/* ---------------------------------------------------------------- fused attention (wgmma) -------------------- */
/* O = softmax(scale * Q K^T) V per (batch, head); Q/K/V are read in place from projection outputs through rank-5
 * strided views so that the reference's "(b n f) l c -> (b f) (n l) c" regroupings never materialise.
 * A view addresses element (col, i1, i2, i3, i4) at base + col + i1*s1 + i2*s2 + i3*s3 + i4*s4 (element strides).
 * The sequence index l of a (batch) is l = i2*e1 + i1 (i1 < e1, i2 < e2); the batch index is qb = i4*e3 + i3.
 * Keys: batch kb = qb / kv_div; i3 is forced to 0 when kv_i3_zero (frame-0 keys of the I2V branch).
 * Head h reads Q/K columns [h*dqk, h*dqk+dqk) (dqk = roundup16(d), zero padded by the projection) and V columns
 * [h*dv, h*dv+dv) with dv = roundup16(d+1) whose column d holds 1.0 (the row sum then falls out of the PV product).
 * Output: fp16 [.., heads*d] written through the same view geometry as Q with row stride ldo:
 *   out = (accumulate ? out : 0) + out_scale * O.
 * Tensor-core tiles: 128 query rows.  e1 >= 128 that is not a multiple of 128 needs e2 == 1 (CLIP's 257 tokens per image):
 * the last tile's rows past e1 are zero-filled on load and never stored.  Keys come in tiles of 64 with the same rule.
 */
typedef struct a3d_view5 {
  const void* base;
  int64_t s1, s2, s3, s4;   /* element strides of dims 1..4 (dim 0 = columns, stride 1) */
  int64_t cols;             /* extent of dim 0 (total columns addressable from base) */
  int32_t e1, e2, e3, e4;   /* extents of dims 1..4 */
} a3d_view5;

typedef struct a3d_attn_args {
  a3d_view5 q, k, v;        /* k and v share extents */
  void* out;                /* fp16 */
  int64_t os1, os2, os3, os4; /* element strides of the output rows (same extents as q) */
  int heads, d;             /* true head dim (40/80/160) */
  float scale;
  int kv_div, kv_i3_zero;
  int accumulate; float out_scale;  /* MUST be set (1.0 if unused; 0.0 is honoured, not remapped: accumulate leaves out as is) */
  int impl;                 /* A3D_GEMM_AUTO: by key count (few-keys, short-keys or tensor-core kernel); A3D_GEMM_TC: the
                               tensor-core kernel at any key count.  Anything else is A3D_EINVAL. */
} a3d_attn_args;

/* Replaces the xformers.ops.memory_efficient_attention calls of the processors together with the einops regroups around
 * them: animatediff/models/attention_processor.py:233 (text keys) and 268 (IP-adapter image keys, accumulated with
 * `scale`), 405 (cross-view self-attention) and 416 (I2V branch, frame-0 keys: kv_i3_zero), 656 and 691 (spatio-temporal
 * processor's cross-view / image branches). */
int a3d_attention(const a3d_attn_args* args, void* stream);
int a3d_attention_kernel(const a3d_attn_args* args, char* name, size_t n);

/* Temporal attention over F frames for every (pixel, head): qkv [P, F, 3*C] fp16 (q | k | v), out [P, F, C].
 * Replaces the attention of the motion modules' temporal transformer blocks (diffusers TransformerTemporalModel reached
 * from unet_motion_mv_model.py:790-836) and the temporal branch of attention_processor.py:541-723 (line 103's call). */
int a3d_temporal_attn(const void* qkv, void* out, int64_t pixels, int frames, int heads, int d, float scale, int64_t ldo,
                      void* stream);   /* ldo: output row stride in halves (0 = C): lets the result land in a column block of a
                                          wider buffer, e.g. next to the cross-view branch for the merged output projection */
int a3d_temporal_attn_kernel(const void* out, int64_t pixels, int frames, int heads, int d, int64_t ldo, char* name, size_t n);

/* ---------------------------------------------------------------- normalisation / elementwise ---------------- */
/* Replaces nn.GroupNorm (+ SiLU) of ResnetBlock2D.norm1/norm2, Transformer2DModel.norm, TransformerTemporalModel.norm
 * (over frames) and conv_norm_out + conv_act (unet_motion_mv_model.py:262-266, 855-857).
 * GroupNorm over (rows_per_sample x C/groups) per sample, NHWC fp16.  x = concat(x1[C1], x2[C2]) along channels
 * (x2 may be NULL).  Optional SiLU.  Output rows may be permuted (perm_a, perm_b as in a3d_gemm).
 * Statistics are reduced without atomics in a fixed order ((n, mean, M2) partials merged with Chan's formula: per-thread
 * pivoted sums -> shared-memory tree -> warp-shuffle tree), so results are bit-reproducible and free of the
 * E[x^2]-E[x]^2 cancellation.  ws_stats: caller-owned scratch of a3d_group_norm_ws_bytes(samples, rows_per_sample, c1+c2,
 * groups) bytes (no initialisation needed). */
size_t a3d_group_norm_ws_bytes(int64_t samples, int64_t rows_per_sample, int c, int groups);
int a3d_group_norm(const void* x1, int c1, const void* x2, int c2, const float* gamma, const float* beta, void* y,
                   int64_t samples, int64_t rows_per_sample, int groups, float eps, int silu, int64_t perm_a,
                   int64_t perm_b, float* ws_stats, void* stream);
/* Input gradient of GroupNorm(+SiLU) for the VAE encoder on the SDS gradient path (animatemv_guidance.py:365-373; weights are
 * frozen, 301-302).  x / dy / dx: NHWC fp16 [samples * rows_per_sample, c]; fwd_ws_stats: the first 2*groups*samples floats of the
 * forward call's ws_stats ((mean, rstd) per (sample, group)); ws: scratch of a3d_group_norm_ws_bytes(...) bytes. */
int a3d_group_norm_backward(const void* x, int c, const float* gamma, const float* beta, const float* fwd_ws_stats, const void* dy,
                            void* dx, int64_t samples, int64_t rows_per_sample, int groups, int silu, float* ws, void* stream);
/* LayerNorm over C per row: BasicTransformerBlock.norm1/2/3 of the spatial and temporal transformers (diffusers). */
int a3d_layer_norm(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int c, float eps,
                   void* stream);
/* nearest x2 upsample NHWC: Upsample2D's F.interpolate in the up blocks (unet_motion_mv_model.py:838-850) */
int a3d_upsample2x(const void* x, void* y, int64_t n, int h, int w, int c, void* stream);
/* y[r, :] = silu(x[r / rep, :]) as fp16 (time-embedding broadcast for the time_emb_proj GEMM) */
int a3d_silu_rows(const float* x, void* y, int64_t rows, int c, int rep, void* stream);
/* conv_in: sample [BN, Cin, F, H, W] (fp32) -> NHWC fp16 [(BN F), H, W, Cout], 3x3 pad 1; w [Cout, Cin, 3, 3] fp32.
 * Replaces the permute/reshape + self.conv_in of unet_motion_mv_model.py:765-768. */
int a3d_conv_in(const float* sample, const float* w, const float* b, void* y, int bn, int cin, int f, int h, int wd,
                int cout, void* stream);
/* conv_out: NHWC fp16 [(BN F), H, W, Cin] -> [BN, Cout, F, H, W] fp32.  Replaces self.conv_out + the reshape/permute back
 * to [B, C, F, H, W] of unet_motion_mv_model.py:857-862. */
int a3d_conv_out(const void* x, const float* w, const float* b, float* y, int bn, int cin, int f, int h, int wd,
                 int cout, void* stream);
/* sinusoidal timestep projection: out[r, :] = [cos(t_r f_i), sin(t_r f_i)] fp32, dim = 2*half -- diffusers `Timesteps`
 * (flip_sin_to_cos=True, freq_shift=0) as called at unet_motion_mv_model.py:723, 734 (self.time_proj) */
int a3d_timestep_proj(const float* t, float* out, int rows, int half, void* stream);
/* small fp32 linear: y[M,N] = act(x[M,K]) W[N,K]^T + b  (act: 0 none, 1 silu);  add: y += previous y when accumulate.
 * The two TimestepEmbedding MLPs (time_embedding, camera_embedding; unet_motion_mv_model.py:730, 737, 742) and the IP-adapter
 * ImageProjection (encoder_hid_proj, 754-763). */
int a3d_linear_f32(const float* x, const float* w, const float* b, float* y, int m, int n, int k, int act_in,
                   int accumulate, void* stream);
/* fp32 -> fp16 cast with optional LayerNorm-free copy (utility) */
int a3d_cast_f32_f16(const float* x, void* y, int64_t n, void* stream);

/* ---------------------------------------------------------------- scheduler ---------------------------------- */
/* One DDIM (eta=0) update with classifier-free guidance and frame-0 re-injection (pipeline.py:1023-1031):
 *   eps = e_a + g * (e_b - e_a)   with (e_a, e_b) = (uncond, cond) halves of noise_pred when uncond_first, else the
 *   guidance ordering eps = e_text + g*(e_text - e_uncond);  x0 = (x - sqrt(1-a_t) eps)/sqrt(a_t);
 *   x' = sqrt(a_prev) x0 + sqrt(1-a_prev) eps;  frame 0 of x' := first_frame.
 * latents/noise_pred: fp32 [BN(,x2), C, F, H, W]. */
int a3d_ddim_cfg_step(float* latents, const float* noise_pred, const float* first_frame, int bn, int c, int f, int hw,
                      float guidance, float alpha_t, float alpha_prev, int uncond_first, void* stream);
/* One DDIM update with eta (diffusers 0.28.0 DDIMScheduler.step(..., eta, variance_noise), reached through
 * prepare_extra_step_kwargs at pipeline.py:580-590, 975, 1028), the optional CFG combine and frame-0 re-injection:
 *   eps = noise_pred                       cfg_mode 0 (no guidance: noise_pred holds bn samples)
 *   eps = e_u + g (e_c - e_u)              cfg_mode 1 ((uncond, cond) halves, pipeline.py:1023-1025)
 *   eps = e_c + g (e_c - e_u)              cfg_mode 2 ((cond, uncond) halves, the SDS guidance order)
 *   x0 = (x - sqrt(1-a_t) eps)/sqrt(a_t);  x' = sqrt(a_prev) x0 + dir_coef eps + std_dev z;  frame 0 of x' := first_frame.
 * The caller computes dir_coef = sqrt(1 - a_prev - std_dev^2) and std_dev = eta sqrt((1-a_prev)/(1-a_t) (1 - a_t/a_prev))
 * in fp32 (scheduler.py DDIMScheduler.step_coefficients).  variance_noise z: fp32 with the latents' shape [BN, C, F, H, W]
 * (frame 0 included and ignored); it may be NULL only when std_dev == 0.  first_frame may be NULL (no re-injection).
 * a3d_ddim_cfg_step(..., uncond_first) is this call with cfg_mode 1 / 2, dir_coef = sqrtf(1 - alpha_prev), std_dev 0. */
int a3d_ddim_step(float* latents, const float* noise_pred, const float* first_frame, const float* variance_noise, int bn, int c,
                  int f, int hw, int cfg_mode, float guidance, float alpha_t, float alpha_prev, float dir_coef, float std_dev,
                  void* stream);

/* One step of the DPM-Solver++ (orders 1 and 2) or Euler / Euler-ancestral scheduler (diffusers 0.28.0
 * DPMSolverMultistepScheduler / EulerDiscreteScheduler / EulerAncestralDiscreteScheduler .step, epsilon prediction) with the
 * CFG combine of a3d_ddim_step (`cfg_mode` 0 / 1 / 2) and the frame-0 re-injection.  One thread per latent element; the
 * caller computes every scalar in fp32 in diffusers' order (scheduler.py `next_step`).  Per element, in this fp32 order:
 *   eps = cfg(noise_pred)                                  as a3d_ddim_step
 *   A3D_SAMPLER_DPMPP:
 *     m0 = (x - sigma_s0 * eps) / alpha_s0                 sigma_s0 = sigma~ = sigma alpha of the current sigma
 *     history_out[i] = m0                                  when history_out is non-NULL
 *     x' = c_x * x - c_m0 * m0                             c_x = sigma~_t / sigma~_s0, c_m0 = alpha_t (e^-h - 1)
 *     order 2: x' = x' + c_d1 * (inv_r0 * (m0 - m1))       m1 = history_in[i], the previous step's m0;
 *                                                          c_d1 = -0.5 alpha_t (e^-h - 1) (midpoint) or
 *                                                          alpha_t ((e^-h - 1)/h + 1) (heun)
 *     (sigma_t = 0 on the last step gives c_x = 0, c_m0 = -1: x' = m0 exactly)
 *   A3D_SAMPLER_EULER:
 *     x0 = x - sigma * eps;  d = (x - x0) / sigma;  x' = x + d * dt
 *     x' = x' + noise[i] * sigma_up                        when sigma_up != 0 (ancestral: dt = sigma_down - sigma)
 *   frame 0 of x' := first_frame when first_frame is non-NULL (nothing else is read or written for frame 0).
 * latents, history_out, history_in, noise: fp32 [BN, C, F, H, W]; noise_pred [BN(,x2), C, F, H, W].  The history buffers are
 * caller-owned and must not alias each other: the caller swaps them between steps.  A3D_EINVAL: a bad kind or cfg_mode,
 * order not 1 or 2, order 2 without history_in, or sigma_up != 0 without noise. */
typedef struct a3d_sampler_step_args {
  float* latents;
  const float* noise_pred;
  const float* first_frame;   /* [BN, C, 1, H, W] or NULL */
  const float* noise;         /* Euler-ancestral z, or NULL */
  float* history_out;         /* DPM-Solver++: m0 of this step, or NULL */
  const float* history_in;    /* DPM-Solver++ order 2: m1 */
  int bn, c, f, hw;
  int cfg_mode;
  float guidance;
  int kind;                   /* A3D_SAMPLER_DPMPP or A3D_SAMPLER_EULER */
  int order;                  /* DPM-Solver++: 1 or 2 */
  float alpha_s0, sigma_s0, c_x, c_m0, inv_r0, c_d1;   /* DPM-Solver++ */
  float sigma, dt, sigma_up;                           /* Euler */
} a3d_sampler_step_args;
enum { A3D_SAMPLER_DPMPP = 0, A3D_SAMPLER_EULER = 1 };
int a3d_sampler_step(const a3d_sampler_step_args* args, void* stream);

/* ---------------------------------------------------------------- 4D-Gaussian rasterizer --------------------- */
typedef struct a3d_raster_cam {
  float viewmatrix[16];   /* row-vector convention, as passed by threestudio/utils/ops.py:344-359 */
  float projmatrix[16];
  float campos[3];
  float tanfovx, tanfovy;
} a3d_raster_cam;

typedef struct a3d_raster_args {
  int P;                     /* gaussians */
  int H, W;
  int num_cams;              /* cameras rendered by this call (batched) */
  const a3d_raster_cam* cams;/* device array [num_cams] */
  const float* means3D;      /* [cam_stride_geom ? num_cams : 1][P,3] */
  const float* scales;       /* [..][P,3] */
  const float* rotations;    /* [..][P,4] */
  const float* opacities;    /* [P,1] */
  const float* shs;          /* [P,(deg+1)^2,3] or NULL */
  const float* colors_precomp; /* [P,3] or NULL */
  int sh_degree, sh_coeffs;
  int per_cam_geometry;      /* 1: means/scales/rotations have a leading camera dim */
  float scale_modifier;
  float bg[3];
  int deterministic;         /* 1: the backward sums every gradient in a fixed order (bit-reproducible; needs the scratch of
                                a3d_raster_backward_scratch_bytes); 0: float atomics.  The forward is deterministic either way. */
} a3d_raster_args;

/* workspace bytes for a forward with at most max_rendered (tile,gaussian) pairs per camera */
size_t a3d_raster_workspace_bytes(int P, int H, int W, int num_cams, int64_t max_rendered);
/* forward: color [cams,3,H,W], depth [cams,1,H,W], alpha [cams,1,H,W], radii [cams,P] int32.
 * num_rendered_host (pinned, [cams]) receives the pair counts; returns A3D_EINVAL if a camera overflowed max_rendered. */
int a3d_raster_forward(const a3d_raster_args* args, float* color, float* depth, float* alpha, int32_t* radii,
                       void* workspace, size_t workspace_bytes, int64_t max_rendered, int64_t* num_rendered_host,
                       void* stream);
/* Byte offset (a multiple of 256) of the forward's pair counters inside its workspace: int64 [num_cams] per-camera pair
 * counts, then the total, then the overflow flag (1 when the total exceeded max_rendered).  a3d_raster_forward writes them on
 * the stream whether or not num_rendered_host is given, so a caller that cannot read the host copy (a CUDA-graph capture)
 * reads them here.  After an overflow the pairs past max_rendered are dropped (the render is incomplete but every access
 * stays inside the workspace, and a3d_raster_backward stays inside its scratch). */
size_t a3d_raster_counters_offset(int P, int H, int W, int num_cams, int64_t max_rendered);
/* Forward-only render straight to RGBA8, for test-view renders.  Replaces the per-camera test path of the reference:
 * rasterize_gaussians at custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:161-170, the clamp at
 * :180, and systems/animate3d.py:439-445, which saves cat(render, mask) as (rgba * 255).astype(np.uint8).
 * rgba [cams,H,W,4] uint8: per pixel (q(clamp(C + T*bg, 0, 1)), q(alpha)) with q(v) = (uint8)(int32)(v *rn 255) -- one
 * rounded fp32 multiply, truncation toward zero, the low 8 bits (numpy's cast on x86); alpha is not clamped.  The same
 * preprocess, binning and sort as a3d_raster_forward, so the bytes equal quantising that call's color / alpha.  radii may
 * be NULL.  No float planes and no backward state are written, so the workspace (a3d_raster_forward_rgba8_workspace_bytes)
 * is smaller than a3d_raster_workspace_bytes; it cannot serve a3d_raster_backward.  Counters and overflow behave as in
 * a3d_raster_forward (num_rendered_host: pinned [cams+2], optional). */
size_t a3d_raster_forward_rgba8_workspace_bytes(int P, int H, int W, int num_cams, int64_t max_rendered);
int a3d_raster_forward_rgba8(const a3d_raster_args* args, uint8_t* rgba, int32_t* radii, void* workspace, size_t workspace_bytes,
                             int64_t max_rendered, int64_t* num_rendered_host, void* stream);
/* Scratch bytes a3d_raster_backward needs: 0 when args->deterministic is 0, else 40 B per (tile, gaussian) pair slot of
 * max_rendered plus 4 B per (camera, gaussian). */
size_t a3d_raster_backward_scratch_bytes(const a3d_raster_args* args, int64_t max_rendered);
/* backward: grads w.r.t. means3D/scales/rotations ([cams or 1][P,*], accumulated over cameras when geometry is shared),
 * opacities [P,1], colors/shs, means2D [cams,P,3]. Needs the workspace of the matching forward untouched, and caller-owned
 * scratch of a3d_raster_backward_scratch_bytes (NULL when that returned 0).  With args->deterministic 0 the gradients are
 * accumulated with float atomics, like rasterize_gaussians_backward.  With args->deterministic set
 * (torch.use_deterministic_algorithms of the caller), the render backward reduces the 8 warp partials of a list entry in
 * warp order and stores one 10-float record per (camera, tile, gaussian) pair in the pair's pre-sort slot; a
 * per-(camera, gaussian) kernel sums its slots in slot (= tile) order, and a per-gaussian kernel pushes every camera's
 * gradients through the projection, summing cameras in camera order.  With SH colours (colors_precomp NULL),
 * dL_dmeans3D includes the colour's dependence on the mean through the view direction (mean - campos) / |mean - campos|,
 * whether or not dL_dshs is requested; channels clamped at 0 in the forward pass no gradient. */
int a3d_raster_backward(const a3d_raster_args* args, const float* dL_dcolor, const float* dL_ddepth,
                        const float* dL_dalpha, const int32_t* radii, void* workspace, size_t workspace_bytes,
                        int64_t max_rendered, float* dL_dmeans3D, float* dL_dscales, float* dL_drotations,
                        float* dL_dopacity, float* dL_dcolors, float* dL_dshs, float* dL_dmeans2D, void* scratch,
                        size_t scratch_bytes, void* stream);
/* debug/parity taps of the binning stage for one camera: sorted keys [n] uint64, point_list [n] uint32, ranges [tiles] uint2 */
int a3d_raster_binning_tap(const void* workspace, int P, int H, int W, int num_cams, int64_t max_rendered, int cam,
                           uint64_t* keys_out, uint32_t* point_list_out, uint32_t* ranges_out, void* stream);

/* ---------------------------------------------------------------- 4D deformation field (k-planes + MLPs) --------- */
/* Per (frame, gaussian): 32 k-planes features (num_scales x 16 channels, product over the 6 coordinate planes of
 * bilinear samples at (x,y,z,t)) -> three bias-free MLPs 32 -> 32 (ReLU) -> {3,4,3} -> means = xyz + d,
 * scales = exp(scaling + d) (d only when deform_scale), rotations = normalize(rotation + d).
 * Replaces Gaussian4DModel.interpolate_ms_features / get_xyz / get_scaling / get_rotation
 * (custom/threestudio-animate3d/geometry/gaussian_4d.py:450-548), without the optional global rot/trans branch.
 * planes[s*6+p] is a [channels, plane_h, plane_w] fp32 grid for coordinate pair p of (0,1),(0,2),(0,3),(1,2),(1,3),(2,3)
 * with the FIRST coordinate of the pair indexing W (grid_sample convention).  w1[m] [hidden, num_scales*channels],
 * w2[m] [out_m, hidden] for m = 0 (xyz, 3), 1 (rotation, 4), 2 (scaling, 3).  Outputs are [T, P, *].
 * backward accumulates (+=) into grad_planes / grad_w1 / grad_w2 (caller zeroes them). */
typedef struct a3d_deform_args {
  int P, T;
  const float* xyz;        /* [P,3] */
  const float* scaling;    /* [P,3] raw (log) scales */
  const float* rotation;   /* [P,4] raw quaternions */
  const float* times;      /* [T] timestamps in [-1,1] */
  int num_scales, channels, hidden;
  const float* planes[12];
  int plane_h[12], plane_w[12];
  const float* w1[3];
  const float* w2[3];
  int deform_scale;
  float* grad_planes[12];  /* backward only; entries may be NULL */
  float* grad_w1[3];
  float* grad_w2[3];
  /* `use_global_trans` support (gaussian_4d.py:499-511, 525-539); all optional (NULL = off) */
  const float* rot_base;      /* [T,P,4] per-frame base quaternions, replace `rotation` (forward and backward) */
  float* grad_rot_base;       /* backward: receives dL/d rot_base, [T,P,4] */
  const float* grad_featmean; /* backward: dL/d (per-frame mean feature), [T, num_scales*channels]; folded into grad_planes */
  int deterministic;          /* backward: 1 = fixed summation order (needs the scratch of a3d_deform_backward_scratch_bytes), 0 = atomics */
} a3d_deform_args;

int a3d_deform_forward(const a3d_deform_args* args, float* means, float* scales, float* rotations, void* stream);
/* per-frame mean over the P gaussians of the k-planes feature vector (`hidden_feats.mean(0)`, gaussian_4d.py:501, 527):
 * featmean [T, num_scales*channels].  Always summed in a fixed order (a cluster of 8 CTAs per frame, reduced through
 * distributed shared memory in rank order), so it is bit-reproducible and needs no scratch. */
int a3d_deform_featmean(const a3d_deform_args* args, float* featmean, void* stream);
/* Scratch bytes a3d_deform_backward needs: 0 when args->deterministic is 0.  Otherwise 768 B per (frame, gaussian) for
 * the stored upstream plane factors (0.61 GB at T = 16, P = 50 000), 16 B per (frame, gaussian) of sort buffers and the
 * per-CTA weight-gradient partials. */
size_t a3d_deform_backward_scratch_bytes(const a3d_deform_args* args);
/* The autograd backward of gaussian_4d.py:450-548.  Accumulates into args->grad_w1 / grad_w2 ([out, in] like the weights)
 * and args->grad_planes.  grad_planes[i] is a CHANNEL-LAST scratch [plane_h[i], plane_w[i], channels] (zero it first;
 * 16-byte aligned): transpose it into the [1, channels, H, W] parameter gradient afterwards.  scratch: caller-owned, of
 * a3d_deform_backward_scratch_bytes (NULL when that returned 0).  With args->deterministic 0 the texel gradients are written
 * with vector float atomics, like the reference's grid_sample backward.  With args->deterministic set: MLP weight gradients
 * are per-CTA partials reduced in CTA order; plane gradients are a gather: per plane, the (frame, gaussian) points are stably
 * radix-sorted by their lower-left cell, and every texel sums the stored factors (d loss / d feature x the other planes'
 * samples, grad_featmean folded in) of the points of its <= 4 adjacent cells in sorted order. */
int a3d_deform_backward(const a3d_deform_args* args, const float* dL_dmeans, const float* dL_dscales, const float* dL_drotations,
                        void* scratch, size_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------- ARAP regulariser (SURVEY 8f-3) -------------- */
/* Row i is positions 1..K of the order of all n points by (fp32 squared distance to point i, index), ascending:
 * pytorch3d.ops.knn_points(p, p, K=K+1)[..., 1:] as used by cal_connectivity_from_points
 * (custom/threestudio-animate3d/systems/util.py:79-82).  Position 0, the one dropped, is the lowest-index point coincident
 * with i: that is i itself unless a lower-index point shares its position, in which case that point is dropped and i appears
 * in its own row (after any other lower-index copies).  nbr [n,K] int32, dist2 [n,K]; 1 <= K <= 12, K < n. */
int a3d_knn_graph(const float* points, int n, int K, int32_t* nbr, float* dist2, void* stream);
/* cal_arap_error (util.py:183-215) with estimate_rotation (138-173) fused, all frames at once:
 *   err = sum_{t>=1} sum_{i in sample} sum_n w[i,n] | e_in(t) - R_i(t) e_in(0) |^2,   e_in(t) = x_t[i] - x_t[nbr[i,n]],
 * R_i(t) = the weighted Procrustes rotation of the node's frame-0 edges onto its frame-t edges (no gradient through R).
 * nodes [Nt,Nv,3]; nbr [Nv,K] (-1 = no edge); weight [Nv,K] or NULL (1 on existing edges, the reference's call);
 * sample [Ns] node indices or NULL (all nodes); an entry outside [0, Nv) contributes nothing (no energy, no gradient), and a
 * repeated entry contributes once per occurrence.  err: device scalar; grad [Nt,Nv,3] = d err / d nodes or NULL; both are
 * overwritten.  scratch: caller-owned, of a3d_arap_scratch_bytes (NULL when that returned 0).  With deterministic 0 one
 * kernel accumulates energy and gradient with float atomics.  With deterministic 1 every sum runs in a fixed order: the
 * energy from per-(frame, sample) partials reduced by one CTA; the gradient from per-(frame, sample, edge) 3-vector records
 * gathered per node after a stable sort of the (target node, record) pairs, so repeated samples add in sample order and the
 * frame-0 gradient adds frames in order.  Checked on the CPU (tests/test_arap_cpu.py) and on the GPU against the reference
 * goldens (tests/test_arap_gpu.py), and per element against the float64 oracle (tests/test_arap_abi_oracle_gpu.py). */
int a3d_arap(const float* nodes, int Nt, int Nv, const int32_t* nbr, int K, const float* weight, const int32_t* sample, int Ns,
             int deterministic, float* err, float* grad, void* scratch, size_t scratch_bytes, void* stream);
/* Scratch bytes a3d_arap needs for the same sizes (Ns of a NULL sample = Nv): 0 when deterministic is 0. */
size_t a3d_arap_scratch_bytes(int Nt, int Nv, int K, int Ns, int deterministic);

/* ---------------------------------------------------------------- mesh animation (SURVEY 8f-5) ---------------- */
/* The device mesh graph is CSR: row_ptr [V+1] and col [E] int32, one row per vertex, its unique neighbours (both directions
 * of every face edge) in ascending index order.  Nothing here uses atomics on an output: results are bit-identical per run. */
/* Vertex adjacency of a triangle mesh, the graph of compute_edge_distances / find_and_save_connected_vertices
 * (tools/mesh_animation/mesh2gaussian.py:36-63, 66-88): the 6 directed half-edges of every face as (src << 32 | dst) keys,
 * CUB radix-sorted, duplicates dropped by a flag pass and a scan, row offsets from the source boundaries.  faces [F,3];
 * a face with a corner outside [0, V) contributes no edge.  A repeated corner gives a self-edge, as in the reference.
 * col must hold 6F entries (the upper bound); num_edges_host (pinned) receives E once the stream reaches it. */
int a3d_mesh_adjacency(const int32_t* faces, int F, int V, int32_t* row_ptr, int32_t* col, int64_t* num_edges_host,
                       void* scratch, size_t scratch_bytes, void* stream);
/* Scratch bytes a3d_mesh_adjacency needs: 40 B per half-edge (6F) plus the CUB temporary.  0 for bad sizes. */
size_t a3d_mesh_adjacency_scratch_bytes(int V, int F);
/* mean_abs_edge [V,3]: the mean of |v_j - v_i| per axis over the CSR row of i, summed in CSR order (compute_edge_distances,
 * mesh2gaussian.py:36-63); 0 for an empty row.  With corner_rgb [F,3,3] (per face-corner colours) also vertex_rgb [V,3]:
 * the mean over the vertex's face corners with the count clamped to >= 1 (convert_to_textureVertex_with_average, 15-33),
 * summed through a stable vertex -> corner sort in the reference's order (corner slot 0 of every face, then slot 1, then 2).
 * corner_rgb NULL: faces / vertex_rgb / scratch are unused. */
int a3d_mesh_vertex_stats(const float* verts, int V, const int32_t* row_ptr, const int32_t* col, const int32_t* faces, int F,
                          const float* corner_rgb, float* mean_abs_edge, float* vertex_rgb, void* scratch, size_t scratch_bytes,
                          void* stream);
/* Scratch bytes a3d_mesh_vertex_stats needs (0 when with_rgb is 0). */
size_t a3d_mesh_vertex_stats_scratch_bytes(int V, int F, int with_rgb);
/* K <= 12 random neighbours per vertex without repetition, the per-step draw of the mesh-edge ARAP graph
 * (sample_matrix_vectorized, custom/threestudio-animate3d/systems/util.py:320-344, called at systems/animate3d.py:224):
 * slot j of row i gets the key = word 0 of Philox4x32-10 with counter (i, j, offset_lo, offset_hi) and key
 * (seed_lo, seed_hi); the K smallest keys (ties by j) are written in ascending key order.  nbr [V,K], -1 past the row's
 * degree: the ragged table a3d_arap reads.  A pure function of (seed, offset, CSR). */
int a3d_mesh_sample_neighbors(const int32_t* row_ptr, const int32_t* col, int V, int K, uint64_t seed, uint64_t offset,
                              int32_t* nbr, void* stream);
/* a3d_mesh_sample_neighbors with (seed, offset) read from device memory, state = uint64 [2] (seed, offset); once the draw
 * has read them, state[1] is advanced by one on the stream.  A CUDA graph that captured this call therefore draws new
 * neighbours on every replay: replay k writes the table of a3d_mesh_sample_neighbors(seed, offset0 + k). */
int a3d_mesh_sample_neighbors_state(const int32_t* row_ptr, const int32_t* col, int V, int K, uint64_t* state, int32_t* nbr,
                                    void* stream);

/* ---------------------------------------------------------------- CLIP image preprocessing (IP-Adapter encoder) ---- */
/* The frame-0 renders (or decoded condition images) -> the A operand of the ViT-H/14 patch-embedding GEMM, in one launch.
 * Replaces the host round trip at custom/threestudio-animate3d/guidance/animatemv_guidance.py:546-555 -- .cpu(),
 * (x*255).astype(np.uint8), PIL, CLIPImageProcessor (transformers 4.25-4.28: PIL bicubic resize of the short edge to 224,
 * centre crop 224, rescale 1/255, OpenAI CLIP mean / std) -- and the Conv2d(3, C, 14, 14) patchify of CLIPVisionEmbeddings
 * (reached from animatediff/utils/util.py:268-287, IPAdapterImageProcessor.encode_image).
 * Arithmetic (animate3d_b200/csrc/a3d_resize_math.h): u = trunc(fp32(x) * 255) clamped to [0, 255] for fp32 input; Pillow's
 * two-pass fixed-point bicubic resize (horizontal first); crop at floor((size - 224) / 2); v = (fp32(u) / 255 - mean) / std.
 * Sources: A3D_CLIP_SRC_F32_NCHW  fp32 [n, 3, h, w] in [0, 1]
 *          A3D_CLIP_SRC_U8_NHWC   uint8 [n, h, w, 3]
 *          A3D_CLIP_SRC_PIXELS    fp32 [n, 3, 224, 224], already normalised: only the patchify (h, w and the tables unused)
 * patches: fp16 [n * 257, 640]; row 0 of each image is zero (the class token comes from the GEMM's row-bias table), column
 *          k < 588 of patch row 1 + 16 py + px holds crop pixel (c, 14 py + ky, 14 px + kx) with k = (c * 14 + ky) * 14 + kx,
 *          columns 588..639 are zero.  May be NULL when pixel_values is given.
 * pixel_values: fp32 [n, 3, 224, 224] or NULL (resizing sources only).
 * The tables come from a3d_clip_resize_plan / a3d_clip_resize_coeffs (host functions) for this h, w, copied to the device. */
enum { A3D_CLIP_SRC_F32_NCHW = 0, A3D_CLIP_SRC_U8_NHWC = 1, A3D_CLIP_SRC_PIXELS = 2 };
typedef struct a3d_clip_prep_args {
  const void* src;
  int src_format;             /* A3D_CLIP_SRC_* */
  int n, h, w;
  int resize_h, resize_w;     /* the plan's resized size */
  const int32_t* bounds_y;    /* [resize_h, 2] (first row, taps) */
  const int32_t* coeffs_y;    /* [resize_h, ksize_y] 22-bit fixed point */
  int ksize_y;
  const int32_t* bounds_x;    /* [resize_w, 2] */
  const int32_t* coeffs_x;    /* [resize_w, ksize_x] */
  int ksize_x;
  void* patches;              /* fp16 [n * 257, 640] or NULL */
  float* pixel_values;        /* fp32 [n, 3, 224, 224] or NULL */
} a3d_clip_prep_args;
int a3d_clip_preprocess(const a3d_clip_prep_args* args, void* stream);
/* Host only: the resized size of an h x w image (short edge 224, long edge int(224 * long / short)) and the taps per output
 * sample of each axis. */
int a3d_clip_resize_plan(int h, int w, int* resize_h, int* resize_w, int* ksize_y, int* ksize_x);
/* Host only: Pillow's bicubic tables for in_size -> out_size: bounds_host [out_size, 2], coeffs_host [out_size, ksize]. */
int a3d_clip_resize_coeffs(int in_size, int out_size, int32_t* bounds_host, int32_t* coeffs_host);

/* debug hook: a device uint64 counter the tensor-core attention kernel bumps once per (warp, key step) that takes the
   lazy-rescale branch of the single-pass softmax (NULL = off; tests use it to prove adversarial inputs reach that branch). */
int a3d_debug_set_attn_trace(void* device_counter_u64);
/* measurement hooks of the rasterizer (bench.py's splat roofline): with timing enabled every forward / backward records CUDA
   events at its stage boundaries; a3d_debug_raster_stage_ms returns the milliseconds of the last forward's stages
   [0] preprocess [1] scan + counts + duplicate [2] radix sort [3] tile ranges [4] render and the last backward's [5] render
   backward [6] preprocess backward ([7] unused) */
int a3d_debug_raster_timing(int enable);
int a3d_debug_raster_stage_ms(float* out_host8);
/* same for the tensor-core GEMM: per-tile clock64 timestamps of CTA 0 (thread 0: tile start, main loop done, epilogue done) */
int a3d_debug_set_gemm_trace(void* device_buffer_1024_int64);

#ifdef __cplusplus
}
#endif
#endif /* A3D_H_ */
