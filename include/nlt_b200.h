/* nlt_b200.h -- C ABI of the NLT UV-space hot path (sm_90a).
 *
 * The reference (google/neural-light-transport) has NO native/FFI boundary:
 * its numerics live in pip wheels (tensorflow 2.2 / tensorflow-addons 0.10)
 * called from Keras layers.  Each entry point below therefore cites the
 * reference *call site* it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer to fp32, NHWC contiguous, owned by the
 *    caller (the library never allocates; workspace is queried, then passed)
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*)
 *  - return 0 on success; <0 on error, message via nlt_last_error()
 *      NLT_ERR_INVALID      bad shape / argument      (reference: ValueError/AssertionError)
 *      NLT_ERR_UNSUPPORTED  unsupported configuration (reference: NotImplementedError)
 *      NLT_ERR_CUDA         CUDA runtime failure
 *  - re-entrant for distinct streams; no global mutable state
 */
#ifndef NLT_B200_H_
#define NLT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NLT_MAX_SEG 4

#define NLT_OK 0
#define NLT_ERR_INVALID (-1)
#define NLT_ERR_UNSUPPORTED (-2)
#define NLT_ERR_CUDA (-3)

/* activation codes -- nlt/networks/elements.py:69-78 */
#define NLT_ACT_NONE 0
#define NLT_ACT_RELU 1
#define NLT_ACT_LEAKYRELU 2 /* alpha = 0.3 */
#define NLT_ACT_ELU 3       /* alpha = 1.0 */

/* One generalised convolution  out[p, n] = sum_{tap, c} A[map(p, tap), c] * W[tap, c, n]
 * over a *virtual channel concat* A of up to NLT_MAX_SEG NHWC tensors (the
 * tf.concat calls of nlt/models/nlt.py:95, :174, :190 are never materialised).
 *
 *   transposed == 0 : map(p,d) = p*stride + d - pad      (Conv2D 'same',          elements.py:26-31)
 *   transposed == 1 : map(p,d) = (p + pad - d) / stride  (Conv2DTranspose 'same', elements.py:34-39;
 *                     taps with a non-integer quotient are skipped)
 *
 * pad_t/pad_l are the TF-SAME pad_before of the underlying strided forward conv.
 * Weight element (tap=dy*kw+dx, c, n) lives at w[tap*w_tap_stride + c*w_c_stride + n*w_n_stride],
 * so that Keras Conv2D kernels (kh,kw,Ci,Co) and Conv2DTranspose kernels
 * (kh,kw,Co,Ci) are both consumed in place, and the adjoint (dgrad) of either
 * op is the other op on the same buffer with swapped strides.
 */
typedef struct nlt_gconv_desc {
  int32_t N;          /* batch */
  int32_t Hin, Win;   /* spatial size of the gathered operand A */
  int32_t Hout, Wout; /* spatial size of the output lattice */
  int32_t kh, kw, stride;
  int32_t pad_t, pad_l;
  int32_t transposed;
  int32_t nseg;                      /* 1..NLT_MAX_SEG */
  const float* seg_ptr[NLT_MAX_SEG]; /* [N or 1, Hin, Win, seg_C] */
  const float* seg_sub[NLT_MAX_SEG]; /* optional: A = seg_ptr - seg_sub (nn_rgb - nn_base, models/nlt.py:96) */
  int32_t seg_C[NLT_MAX_SEG];
  int32_t seg_bcast[NLT_MAX_SEG];    /* 1: tensor has batch 1 and is broadcast (tf.tile in nlt_test.py:84) */
  int32_t Cout;
  const float* w;
  int64_t w_tap_stride, w_c_stride, w_n_stride;
} nlt_gconv_desc;

const char* nlt_version(void);
/* process-wide switches: "tc" (1: wgmma 3xTF32 path where eligible [default], 0: fp32-FMA kernels only, 2: the wgmma
 * path for every shape it can run, ahead of the size heuristics and the stream kernels -- for A/B tests),
 * "tc_wgrad" (same for the weight-gradient kernel), "wgrad_rows" (1: row-run form of the warp-stream
 * weight-gradient kernel where float4 access allows it [default], 0: flat-pixel form), "dconv_wide" (1: the
 * pixel x 16-outputs stencil kernel for the 16-channel stencils, 0: the tiled implicit-GEMM kernel),
 * "dconv_wide32" (default 0 = off: the 32-output form of that kernel, validated but not faster;
 * 1 = one pixel per thread, 2 = two), "dconv_wide8" (default 1: the 8-output form, reached together
 * with "dconv_wide_first"), "dconv_wide_first" (routing, default 1: prefer the wide
 * stencil kernel over the quad-per-thread one for 16 / 8 outputs with K <= 32).
 * Environment defaults: NLT_DISABLE_TC=1, NLT_DISABLE_TC_WGRAD=1, NLT_DCONV_WIDE=0|1. */
int nlt_set_option(const char* name, int value);
const char* nlt_last_error(void);
/* number of CUDA kernels this library has launched so far in this process (diagnostic counter) */
uint64_t nlt_launch_count(void);
/* launches of one kernel so far, by the name the library reports it under (e.g. "pf_fwd_kernel"); 0 if never
 * launched (diagnostic counter: lets tests check which kernel a routing option selected) */
uint64_t nlt_kernel_launch_count(const char* name);
/* how many of those were wgmma tensor-core kernels (diagnostic counter) */
uint64_t nlt_tc_launch_count(void);

/* out = act(A*W + bias);   then  out = beta*out_old + out;  then out *= act'(mask_y)
 * Replaces Conv2D / Conv2DTranspose + LeakyReLU (elements.py:26-39, 69-78) and,
 * with the adjoint descriptor, their input-gradients (tape.gradient,
 * nlt/trainvali.py:279).  bias, mask_y may be NULL; beta is 0 or 1. */
int nlt_gconv_fwd(const nlt_gconv_desc* d, const float* bias, int act,
                  float beta, const float* mask_y, int mask_act,
                  float* out, void* stream);
/* Same op with caller-provided scratch: enables the wgmma (3xTF32 split,
 * fp32 accumulate in registers) tensor-core path where the shape allows it (all
 * sources with C % 16 == 0, Cout % 16 == 0, tileable lattice); the scratch holds
 * the per-call hi/lo TF32 weight planes.  Falls back to the fp32 kernels
 * otherwise.  Set NLT_DISABLE_TC=1 in the environment to force the fp32 path. */
int64_t nlt_gconv_fwd_workspace_bytes(const nlt_gconv_desc* d);
int nlt_gconv_fwd_ws(const nlt_gconv_desc* d, const float* bias, int act,
                     float beta, const float* mask_y, int mask_act, float* out,
                     void* workspace, int64_t workspace_bytes, void* stream);
/* The same op with the weight planes prepared AHEAD of time: the weights of a train step are final when the step
 * starts (tf.keras optimizers apply at its end, nlt/trainvali.py:279-281), so the caller can run every layer's
 * nlt_gconv_pack_weights on a separate stream that depends on nothing but the start of the step, and the per-layer
 * pack kernel leaves the critical path.  nlt_gconv_fwd_pack_bytes: size of the planes, 0 when the op (with this beta /
 * mask use) is not served by the tensor-core kernel, < 0 on error.  `packed` must stay untouched until the
 * nlt_gconv_fwd_packed call that reads it has finished. */
int64_t nlt_gconv_fwd_pack_bytes(const nlt_gconv_desc* d, float beta, int has_mask);
int nlt_gconv_pack_weights(const nlt_gconv_desc* d, void* packed, int64_t packed_bytes, void* stream);
int nlt_gconv_fwd_packed(const nlt_gconv_desc* d, const float* bias, int act,
                         float beta, const float* mask_y, int mask_act, float* out,
                         const void* packed, int64_t packed_bytes, void* stream);

/* A second, pointwise term fused into the epilogue of a pointwise op (1x1 stride-1 conv, or a
 * k == stride transposed conv in its depth-to-space form):
 *   out[n,y,x,c] = mask( act(conv_d(...)[n,y,x,c] + bias[c]) + sum_k x[n,y,x,k] * w[k*w_k_stride + c*w_n_stride]
 *                        + beta * out[n,y,x,c] )
 * x has the spatial shape of `out` and K <= 4 channels.  Use: the input gradient of the final 1x1 conv
 * (networks/convnet.py:65-70, 36 -> 3) w.r.t. the level-0 skip tensors rides on the launch of the level-1
 * down-conv's input gradient, which writes the same tensor -- one write + one read-modify-write pass over a
 * full-resolution 16-channel tensor less per skip.  _supported() returns 1 when the op is served by the
 * pointwise kernel with float4 stores (else 0); _fused() returns NLT_ERR_UNSUPPORTED in that case and the
 * caller issues the two ops separately. */
typedef struct nlt_pw_term {
  const float* x;
  int32_t K;
  const float* w;
  int64_t w_k_stride, w_n_stride;
} nlt_pw_term;
int nlt_gconv_fwd_fused_supported(const nlt_gconv_desc* d, const nlt_pw_term* term,
                                  const float* mask_y, const float* out);
int nlt_gconv_fwd_fused(const nlt_gconv_desc* d, const nlt_pw_term* term, const float* bias, int act,
                        float beta, const float* mask_y, int mask_act, float* out, void* stream);

/* Weight/bias gradient of the op described by d:
 *   dW[tap,c,n] (+)= sum_p A[map(p,tap),c] * G[p,n],   db[n] (+)= sum_p G[p,n]
 * written with the same strides as d->w.  Deterministic (two-stage split
 * reduction through `workspace`).  accumulate: 0 overwrite, 1 add.
 * Replaces tape.gradient w.r.t. trainable_variables (nlt/trainvali.py:279). */
int64_t nlt_gconv_wgrad_workspace_bytes(const nlt_gconv_desc* d);
int nlt_gconv_wgrad(const nlt_gconv_desc* d, const float* G, float* dW,
                    float* db, int accumulate, void* workspace,
                    int64_t workspace_bytes, void* stream);

/* mean over K observations: out[b] = (1/K) sum_k w[b,k] * in[k*B + b]
 * (tf.reduce_mean over the stacked observation axis, models/nlt.py:161-164).
 * weights may be NULL.  per_sample = H*W*C elements. */
int nlt_kmean_fwd(const float* in, const float* weights, int32_t K, int32_t B,
                  int64_t per_sample, float* out, void* stream);
/* d_in[k*B+b] = beta*d_in + w[b,k]/K * d_out[b]; then *= act'(mask_y) */
int nlt_kmean_bwd(const float* d_out, const float* weights, int32_t K,
                  int32_t B, int64_t per_sample, float beta,
                  const float* mask_y, int mask_act, float* d_in, void* stream);

/* UV -> camera tail of Model.call (nlt/models/nlt.py:99-120, 132-133):
 *   pred_uv = net_out (+ base if skip_connect_base); texel (0,0) of pred/base/fg zeroed;
 *   {fg,base,pred}_camspc = resampler(., warp * (uvw,uvh));  gt_camspc = rgb_camspc * fg_camspc.
 * warp [B,ih,iw,2] in [0,1].  Any output pointer may be NULL (skipped).
 * pred_uv [B,H,W,3] is always written. */
int nlt_uv2cam_fwd(const float* net_out, const float* base, const float* warp,
                   const float* rgb_camspc, int32_t B, int32_t H, int32_t W,
                   int32_t ih, int32_t iw, int32_t skip_connect_base,
                   float* pred_uv, float* pred_camspc, float* base_camspc,
                   float* fg_camspc, float* gt_camspc, void* stream);
/* d_net_out [B,H,W,3] = scatter-add of d_pred_camspc through the 4 bilinear
 * taps, texel (0,0) zeroed (gradient of tfa.image.resampler w.r.t. data).
 * d_net_out is fully overwritten. */
int nlt_uv2cam_bwd(const float* d_pred_camspc, const float* warp, int32_t B,
                   int32_t H, int32_t W, int32_t ih, int32_t iw,
                   float* d_net_out, void* stream);

/* The same gradient, bit-reproducible: contributions are accumulated as 64-bit fixed-point integers (order
 * independent), scaled by the largest |d_pred_camspc| of the call, then converted to fp32 once.
 * workspace: >= nlt_uv2cam_bwd_workspace_bytes(), 8-byte aligned, ZERO-FILLED by the caller before the first call;
 * every call leaves it zero-filled again (the conversion pass clears what the scatter touched). */
int64_t nlt_uv2cam_bwd_workspace_bytes(int32_t B, int32_t H, int32_t W);
int nlt_uv2cam_bwd_det(const float* d_pred_camspc, const float* warp, int32_t B,
                       int32_t H, int32_t W, int32_t ih, int32_t iw,
                       float* d_net_out, void* workspace, void* stream);

/* tf.image.resize bilinear, half-pixel centres (nlt/util/img.py:113-116) */
int nlt_resize_bilinear_fwd(const float* in, int32_t B, int32_t H, int32_t W,
                            int32_t C, int32_t oh, int32_t ow, float* out,
                            void* stream);
int nlt_resize_bilinear_bwd(const float* d_out, int32_t B, int32_t H, int32_t W,
                            int32_t C, int32_t oh, int32_t ow, float* d_in,
                            void* stream);

/* losses.L2 with keep_batch (nlt/losses.py:39-53) fused with its gradient:
 *   loss[b] = mean_{h,w,c} (gt-pred)^2 ;  d_pred = 2*(pred-gt)*loss_scale/(h*w*c)
 * loss_scale = 1/global_bs (tf.nn.compute_average_loss, trainvali.py:277-278).
 * d_pred may be NULL.  partial: >= nlt_l2_loss_workspace_bytes(). */
int64_t nlt_l2_loss_workspace_bytes(int32_t B, int64_t per_sample);
int nlt_l2_loss(const float* pred, const float* gt, int32_t B,
                int64_t per_sample, float loss_scale, float* loss,
                float* d_pred, void* workspace, void* stream);

/* losses.L1 (nlt/losses.py:27-36, MeanAbsoluteError then reduce_mean) per sample, fused with its gradient:
 *   loss[b] = mean_{h,w,c} |pred - gt| ;  d_pred = sign(pred - gt) * loss_scale / per_sample (exactly 0 on ties)
 * d_pred may be NULL.  Deterministic (per-block partials, fixed-order sum in double).
 * workspace: >= nlt_l1_loss_workspace_bytes() (< 0 for B <= 0 or per_sample <= 0). */
int64_t nlt_l1_loss_workspace_bytes(int32_t B, int64_t per_sample);
int nlt_l1_loss(const float* pred, const float* gt, int32_t B, int64_t per_sample, float loss_scale, float* loss,
                float* d_pred, void* workspace, void* stream);

/* losses.SSIM (nlt/losses.py:75-87) per sample, fused with its gradient: tf.image.ssim(gt, pred, max_val) of TF 2.2
 * (11 x 11 Gaussian window, sigma 1.5, VALID, k1 = 0.01, k2 = 0.03), averaged over channels and output pixels:
 *   loss[b] = (1 - ssim_b) / 2 ;  d_pred = d(sum_b loss[b] * loss_scale) / d(pred)
 * pred, gt: [B,H,W,3] with H, W >= 11 and B <= 65535; d_pred may be NULL (the loss is bit-identical either way).
 * Deterministic.  workspace: >= nlt_ssim_loss_workspace_bytes() (< 0 for B <= 0, H < 11 or W < 11). */
int64_t nlt_ssim_loss_workspace_bytes(int32_t B, int32_t H, int32_t W);
int nlt_ssim_loss(const float* pred, const float* gt, int32_t B, int32_t H, int32_t W, float max_val, float loss_scale,
                  float* loss, float* d_pred, void* workspace, void* stream);

/* SURVEY 8f row N1 (checked on the CPU and on hardware against the oracle pinned to the reference's wavelet
 * fixtures): losses.Barron with keep_batch (nlt/losses.py:90-121) fused with its gradient.
 *   r = (gt - pred) [* alpha]  ->  volume-preserving YUV  ->  `levels`-level CDF 9/7 analysis (reflecting
 *   boundaries)  ->  nll = sqrt((w/scale)^2 + 1) - 1 + log(scale) + log_z per coefficient
 *   loss[b] = mean_{h,w,c} nll ;  d_pred = d(sum_b loss[b] * loss_scale) / d(pred)
 * pred, gt: [B,H,W,3] with B <= 65535; alpha: [B,H,W,1] or NULL; log_z = log Z(1) = log(2 e K_1(1)) = 1.18549523...;
 * levels <= ceil(log2(min(H, W))) (the reference uses 5); d_pred may be NULL (the loss is bit-identical either way).
 * Deterministic: per-block partials summed per sample in a fixed order, in double.  workspace >= _workspace_bytes()
 * (the wavelet planes plus B x (blocks per sample) doubles), 8-byte aligned, contents on entry irrelevant. */
int64_t nlt_barron_loss_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t levels);
int nlt_barron_loss(const float* pred, const float* gt, const float* alpha, int32_t B, int32_t H, int32_t W,
                    int32_t levels, float scale, float log_z, float loss_scale, float* loss, float* d_pred,
                    void* workspace, void* stream);

/* tf.keras.optimizers.Adam(lr, amsgrad=True) dense update over a flat bucket
 * (nlt/trainvali.py:122-127, 280); step is 1-based; grad_scale multiplies g. */
int nlt_amsgrad_step(float* p, const float* g, float* m, float* v, float* vhat,
                     int64_t n, int32_t step, float lr, float beta1,
                     float beta2, float eps, float grad_scale, void* stream);

/* Normalisation layers of the conv blocks (conv -> norm -> act, nlt/networks/convnet.py:50-59, 67-76), each fused
 * with the activation that follows it.  x, y, dz, dx: [pixels or N*HW][C] NHWC rows, C % 4 == 0.
 *   pixel    (nlt/networks/elements.py:103-121): y = act(x * rsqrt(mean_c(x^2) + 1e-8)); no parameters.
 *            _bwd: dx from dz = d(loss)/d(norm output) (the activation's derivative is applied by the consumer
 *            from the saved output, as for every other op).
 *   instance (elements.py:97-100, tf.contrib.layers.instance_norm(center=True, scale=True, epsilon=1e-6)):
 *            y = act(gamma * (x - mean_hw) * rsqrt(var_hw + eps) + beta), statistics per sample and channel
 *            (biased variance); _fwd also returns mean / rstd [N*C] for the backward pass; _bwd writes dx and
 *            (accumulate ? adds to : overwrites) dgamma / dbeta [C].  Deterministic (fixed-order reductions).
 *            The variance is the centred second moment, taken per 1024-pixel chunk around the chunk's own mean and
 *            merged in double (Chan), so rstd does not degrade as |mean| / std grows.
 *            workspace >= nlt_instnorm_workspace_bytes() = (N * ceil(HW / 1024) * 3C + 2NC) floats; C <= 6144. */
int nlt_pixelnorm_fwd(const float* x, int64_t pixels, int32_t C, int act, float* y, void* stream);
int nlt_pixelnorm_bwd(const float* x, const float* dz, int64_t pixels, int32_t C, float* dx, void* stream);
int64_t nlt_instnorm_workspace_bytes(int32_t N, int32_t HW, int32_t C);
int nlt_instnorm_fwd(const float* x, const float* gamma, const float* beta, int32_t N, int32_t HW, int32_t C, int act,
                     float eps, float* y, float* mean, float* rstd, void* workspace, void* stream);
int nlt_instnorm_bwd(const float* x, const float* dz, const float* gamma, const float* mean, const float* rstd,
                     int32_t N, int32_t HW, int32_t C, float* dx, float* dgamma, float* dbeta, int accumulate,
                     void* workspace, void* stream);

/* The U-Net ops of `pool = max | avg` (nlt/networks/convnet.py:50-80).  x, y, d_x, d_y: [N,H,W,C] NHWC (any C; float4
 * rows when C % 4 == 0 and the pointers are 16-byte aligned).  Deterministic: no atomics.
 *   pool2x2      tf.keras.layers.{Max,Average}Pooling2D(2, 2, 'same') (elements.py:81-94): y [N,ceil(H/2),ceil(W/2),C];
 *                odd sizes clip the window at the right / bottom edge, avg divides by the valid taps.
 *                _bwd: d_x = (beta * d_x + g) * act'(mask_y), g = the window's d_y routed to the FIRST maximum of the
 *                window in row-major tap order (recomputed from x; 0 at the other taps) for max, d_y / valid taps for
 *                avg.  mask_y may be NULL; beta is 0 or 1.
 *   upsample2x   tf.keras.layers.UpSampling2D(2, interpolation='bilinear') (elements.py:42-48) = tf.image.resize to
 *                (2H, 2W), half-pixel centres: y [N,2H,2W,C].  A batch-1 x gives a batch-1 y (broadcast segment).
 *                _bwd: the exact adjoint, gathered per low-resolution pixel (<= 4 x 4 taps of d_y [N,2H,2W,C]),
 *                with the same beta / mask epilogue into d_x [N,H,W,C]. */
#define NLT_POOL_MAX 0
#define NLT_POOL_AVG 1
int nlt_pool2x2_fwd(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, int kind, float* y, void* stream);
int nlt_pool2x2_bwd(const float* x, const float* d_y, int32_t N, int32_t H, int32_t W, int32_t C, int kind, float beta,
                    const float* mask_y, int mask_act, float* d_x, void* stream);
int nlt_upsample2x_bilinear_fwd(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, float* y, void* stream);
int nlt_upsample2x_bilinear_bwd(const float* d_y, int32_t N, int32_t H, int32_t W, int32_t C, float beta,
                                const float* mask_y, int mask_act, float* d_x, void* stream);

/* uint8 image samples -> float32 in [0, 1] (v / 255, correctly rounded = the host pipeline's
 * float32(v / 255.0), nlt/datasets/nlt.py:134-139): lets a batch cross PCIe as bytes (SURVEY 8f N3). */
int nlt_u8_to_f32(const uint8_t* in, int64_t n, float* out, void* stream);

/* acc[i] += sum_k in[k*per_sample + i]  -- running per-level sum of the observation features over the samples
 * of a batch (the concat + tf.reduce_mean(axis=0) of nlt/nlt_test.py:114-124 without holding every sample). */
int nlt_ksum_acc(const float* in, int32_t K, int64_t per_sample, float* acc, void* stream);
/* x *= a   (the 1/count of that mean) */
int nlt_scale(float* x, int64_t n, float a, void* stream);
/* out = a * b elementwise (alpha_blend of the resized coverage, nlt/util/img.py:74-89, models/nlt.py:132-133) */
int nlt_mul(const float* a, const float* b, int64_t n, float* out, void* stream);

/* The same update with the 1-based step counter kept ON THE DEVICE (int32 *step_dev holds the number of updates
 * already applied; the call advances it by one first), so the optimiser launch can be part of a captured CUDA
 * graph of the whole train step (nlt/trainvali.py:267-290 runs as one tf.function). */
int nlt_amsgrad_step_dev(float* p, const float* g, float* m, float* v, float* vhat,
                         int64_t n, int32_t* step_dev, float lr, float beta1,
                         float beta2, float eps, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NLT_B200_H_ */
