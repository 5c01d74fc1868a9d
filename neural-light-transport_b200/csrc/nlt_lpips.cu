// losses.LPIPS (nlt/losses.py:143-169): the frozen LPIPS AlexNet graph (net-lin_alex_v0.1.pb) per sample, fused
// with its input gradient.  One call runs pred and gt through the network as one batch of 2B images:
//
//   prep     x = (2 v - 1) * scale_c + shift_c                          [2B, H, W, 3]     (pred: 0..B-1, gt: B..2B-1)
//   conv1    11x11 / s4, pad 2, 3 -> 64, ReLU      -> relu1 ; maxpool 3x3 / s2 VALID -> pool1
//   conv2    5x5, pad 2, 64 -> 192, ReLU           -> relu2 ; maxpool 3x3 / s2 VALID -> pool2
//   conv3-5  3x3, pad 1, 192 -> 384 -> 256 -> 256, ReLU -> relu3, relu4, relu5
//   head l   u = f / (sqrt(sum_c f^2) + 1e-10);  d = sum_c lin_l[c] (u_pred - u_gt)^2;  mean over the lattice
//   loss[b]  = sum_l mean_l
//
// The convs run on the generalised-conv machinery (gconv_run: bias and ReLU in the epilogue; conv2-5 on the wgmma
// kernel with partial edge tiles unless option tc = 0), reading the OIHW kernels in place through the descriptor
// strides.  The backward pass needs the input gradient of the pred half only: the head writes d relu_l for images
// 0..B-1, the conv input gradients of conv5 / conv4 accumulate onto d relu4 / d relu3 and apply their ReLU masks, the
// conv3 / conv2 input gradients write d pool2 / d pool1, whose gather-form adjoints accumulate onto d relu2 / d relu1
// and apply their masks, and conv1's input gradient (3 channels) is scaled by 2 scale_c in place in d_pred.
//
// Deterministic: the head's blocks write one double partial each to their own slot; lpips_loss_kernel adds each
// sample's partials layer by layer in a fixed order.  No atomics.
#include "nlt_common.cuh"

namespace nlt {
namespace {

constexpr int NL = 5;
constexpr int CONV_CO[NL] = {64, 192, 384, 256, 256};
constexpr int CONV_CI[NL] = {3, 64, 192, 384, 256};
constexpr int CONV_K[NL] = {11, 5, 3, 3, 3};
constexpr int CONV_S[NL] = {4, 1, 1, 1, 1};
constexpr int CONV_P[NL] = {2, 2, 1, 1, 1};
constexpr float LPIPS_EPS = 1e-10f;
constexpr int HEAD_WARPS = 8;
constexpr int HEAD_PIX = 256;        // lattice pixels per head block (32 per warp)
constexpr int SUM_T = 256;

__global__ void lpips_prep_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                  const float* __restrict__ scale, const float* __restrict__ shift, long long n_half,
                                  float* __restrict__ x) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < 2 * n_half;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = i < n_half ? pred[i] : gt[i - n_half];
    const int c = (int)(i % 3);
    // the graph's order: x * 2 - 1, the per-channel 1x1 conv, + shift (no contraction into FMAs)
    x[i] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(v, 2.f), 1.f), __ldg(scale + c)), __ldg(shift + c));
  }
}

// d_pred = d x * 2 scale_c, in place (d x: conv1's input gradient written into d_pred)
__global__ void lpips_prep_bwd_kernel(const float* __restrict__ scale, long long n, float* __restrict__ d) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    d[i] *= 2.f * __ldg(scale + (int)(i % 3));
}

// MaxPool 3x3 / s2 VALID, NHWC, C % 4 == 0: one thread per (output pixel, 4 channels)
__global__ void lpips_maxpool_kernel(const float* __restrict__ x, int N, int H, int W, int C, int Ho, int Wo,
                                     float* __restrict__ y) {
  const int C4 = C / 4;
  const long long total = (long long)N * Ho * Wo * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long p = i / C4;
    const int ox = (int)(p % Wo); p /= Wo;
    const int oy = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const float* base = x + (((long long)n * H + 2 * oy) * W + 2 * ox) * C + 4 * c4;
    float4 m = ld4(base);
    for (int t = 1; t < 9; ++t) {
      const float4 v = ld4(base + ((long long)(t / 3) * W + t % 3) * C);
      m.x = v.x > m.x ? v.x : m.x; m.y = v.y > m.y ? v.y : m.y;
      m.z = v.z > m.z ? v.z : m.z; m.w = v.w > m.w ? v.w : m.w;
    }
    reinterpret_cast<float4*>(y)[i] = m;
  }
}

// Adjoint of lpips_maxpool_kernel, gathered per input pixel: each of the <= 2 x 2 windows that contain (iy, ix) sends
// its d_y to the window's FIRST maximum in row-major tap order (recomputed from x).  Then
//   d_x = (d_x + g) * relu'(mask_y)      (accumulates onto the head's gradient of the pooled ReLU output)
__global__ void lpips_maxpool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, int N, int H, int W,
                                         int C, int Ho, int Wo, float* __restrict__ dx) {
  const int C4 = C / 4;
  const long long total = (long long)N * H * W * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long p = i / C4;
    const int ix = (int)(p % W); p /= W;
    const int iy = (int)(p % H);
    const int n = (int)(p / H);
    const int oy0 = iy >= 2 ? (iy - 1) / 2 : 0, oy1 = min(iy / 2, Ho - 1);
    const int ox0 = ix >= 2 ? (ix - 1) / 2 : 0, ox1 = min(ix / 2, Wo - 1);
    const float* img = x + (long long)n * H * W * C + 4 * c4;
    const int me = iy * W + ix;
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    for (int oy = oy0; oy <= oy1; ++oy) {
      for (int ox = ox0; ox <= ox1; ++ox) {
        const int w0 = 2 * oy * W + 2 * ox;
        float4 m = ld4(img + (long long)w0 * C);
        int am[4] = {w0, w0, w0, w0};
        for (int t = 1; t < 9; ++t) {
          const int q = w0 + (t / 3) * W + t % 3;
          const float4 v = ld4(img + (long long)q * C);
          if (v.x > m.x) { m.x = v.x; am[0] = q; }
          if (v.y > m.y) { m.y = v.y; am[1] = q; }
          if (v.z > m.z) { m.z = v.z; am[2] = q; }
          if (v.w > m.w) { m.w = v.w; am[3] = q; }
        }
        const float4 d = ld4(dy + (((long long)n * Ho + oy) * Wo + ox) * C + 4 * c4);
        if (am[0] == me) g[0] += d.x;
        if (am[1] == me) g[1] += d.y;
        if (am[2] == me) g[2] += d.z;
        if (am[3] == me) g[3] += d.w;
      }
    }
    const float4 y = ld4(img + (long long)me * C);
    float4 o = reinterpret_cast<float4*>(dx)[i];
    o.x = y.x > 0.f ? o.x + g[0] : 0.f;
    o.y = y.y > 0.f ? o.y + g[1] : 0.f;
    o.z = y.z > 0.f ? o.z + g[2] : 0.f;
    o.w = y.w > 0.f ? o.w + g[3] : 0.f;
    reinterpret_cast<float4*>(dx)[i] = o;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Distance head of one layer: one warp per lattice pixel, CPL = C / 32 channels per lane.  grid (blocks per sample,
// B); each block covers HEAD_PIX pixels of sample blockIdx.y and writes sum_pixels d (double) to part[blockIdx.y *
// gridDim.x + blockIdx.x].  With df != nullptr it also writes
//   df = gscale * (q / (r + eps) - f (f . q) / (r (r + eps)^2)),   q = 2 lin (u_pred - u_gt),  r = |f_pred|
// (the second term is 0 where r = 0), times relu'(f_pred) when mask_relu (relu5, which no later op masks).
template <int CPL>
__global__ void __launch_bounds__(HEAD_WARPS * 32)
lpips_head_kernel(const float* __restrict__ f, long long half, int HW, const float* __restrict__ lin, float gscale,
                  int mask_relu, double* __restrict__ part, float* __restrict__ df) {
  constexpr int C = CPL * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  float w[CPL];
#pragma unroll
  for (int j = 0; j < CPL; ++j) w[j] = __ldg(lin + lane + 32 * j);
  double acc = 0.0;
  const int p_end = min(HW, (blockIdx.x + 1) * HEAD_PIX);
  for (int pix = blockIdx.x * HEAD_PIX + warp; pix < p_end; pix += HEAD_WARPS) {
    const long long off = ((long long)b * HW + pix) * C + lane;
    float fp[CPL], fg[CPL];
    float sp = 0.f, sg = 0.f;
#pragma unroll
    for (int j = 0; j < CPL; ++j) {
      fp[j] = __ldg(f + off + 32 * j);
      fg[j] = __ldg(f + half + off + 32 * j);
      sp = fmaf(fp[j], fp[j], sp);
      sg = fmaf(fg[j], fg[j], sg);
    }
    const float rp = sqrtf(warp_sum(sp)), rg = sqrtf(warp_sum(sg));
    const float dp = rp + LPIPS_EPS, dg = rg + LPIPS_EPS;
    float a[CPL];
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < CPL; ++j) {
      a[j] = __fdiv_rn(fp[j], dp) - __fdiv_rn(fg[j], dg);
      d = fmaf(w[j] * a[j], a[j], d);
    }
    d = warp_sum(d);
    acc += (double)d;
    if (df != nullptr) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < CPL; ++j) s = fmaf(fp[j], 2.f * w[j] * a[j], s);
      s = warp_sum(s);
      const float t = rp > 0.f ? s / (rp * dp * dp) : 0.f;
#pragma unroll
      for (int j = 0; j < CPL; ++j) {
        float g = gscale * (2.f * w[j] * a[j] / dp - fp[j] * t);
        if (mask_relu && !(fp[j] > 0.f)) g = 0.f;
        df[off + 32 * j] = g;
      }
    }
  }
  __shared__ double sh[HEAD_WARPS];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < HEAD_WARPS; ++i) s += sh[i];
    part[(long long)b * gridDim.x + blockIdx.x] = s;
  }
}

// one block per sample: loss[b] = sum_l (1 / HW_l) sum_blocks part_l[b][blk], in a fixed order, in double
struct SumArgs {
  const double* part[NL];
  int nblk[NL];
  double inv_hw[NL];
};
__global__ void __launch_bounds__(SUM_T) lpips_loss_kernel(const SumArgs a, float* __restrict__ loss) {
  __shared__ double sh[SUM_T];
  double total = 0.0;
  for (int l = 0; l < NL; ++l) {
    const double* p = a.part[l] + (long long)blockIdx.x * a.nblk[l];
    double s = 0.0;
    for (int i = threadIdx.x; i < a.nblk[l]; i += SUM_T) s += p[i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int w = SUM_T / 2; w > 0; w >>= 1) {
      if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
      __syncthreads();
    }
    total += sh[0] * a.inv_hw[l];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[blockIdx.x] = (float)total;
}

// ---- shapes and workspace layout ----------------------------------------------------------------------------------
struct Plan {
  int B, H, W;
  int ch[NL], cw[NL];          // conv output lattices
  int ph[2], pw[2];            // pool outputs
  // float offsets (each a multiple of 64 floats = 256 bytes)
  size_t x0, relu[NL], pool[2], g[NL], gpool[2], part[NL], tc;
  int nblk[NL];
  size_t total_floats;
  int64_t tc_bytes;
};

inline int conv_out(int n, int l) { return (n + 2 * CONV_P[l] - CONV_K[l]) / CONV_S[l] + 1; }
inline int pool_out(int n) { return (n - 3) / 2 + 1; }

void conv_desc(const Plan& pl, int l, bool dgrad, const float* in, const float* w, nlt_gconv_desc* d) {
  memset(d, 0, sizeof(*d));
  const int hin = l == 0 ? pl.H : (l <= 2 ? pl.ph[l - 1] : pl.ch[l - 1]);
  const int win = l == 0 ? pl.W : (l <= 2 ? pl.pw[l - 1] : pl.cw[l - 1]);
  const int k = CONV_K[l], ci = CONV_CI[l], co = CONV_CO[l];
  d->kh = d->kw = k;
  d->stride = CONV_S[l];
  d->pad_t = d->pad_l = CONV_P[l];
  d->nseg = 1;
  d->seg_ptr[0] = in;
  d->w = w;
  d->w_tap_stride = 1;                       // OIHW: tap = ky * k + kx
  if (!dgrad) {                              // [2B, hin, win, ci] -> [2B, ch, cw, co]
    d->N = 2 * pl.B; d->Hin = hin; d->Win = win; d->Hout = pl.ch[l]; d->Wout = pl.cw[l];
    d->transposed = 0; d->seg_C[0] = ci; d->Cout = co;
    d->w_c_stride = (int64_t)k * k; d->w_n_stride = (int64_t)ci * k * k;
  } else {                                   // adjoint: [B, ch, cw, co] -> [B, hin, win, ci]
    d->N = pl.B; d->Hin = pl.ch[l]; d->Win = pl.cw[l]; d->Hout = hin; d->Wout = win;
    d->transposed = 1; d->seg_C[0] = co; d->Cout = ci;
    d->w_c_stride = (int64_t)ci * k * k; d->w_n_stride = (int64_t)k * k;
  }
}

bool make_plan(int B, int H, int W, Plan* pl) {
  if (B <= 0 || B > 65535 || H < 31 || W < 31 || (long long)H * W > (1ll << 28)) return false;
  pl->B = B; pl->H = H; pl->W = W;
  pl->ch[0] = conv_out(H, 0); pl->cw[0] = conv_out(W, 0);
  pl->ph[0] = pool_out(pl->ch[0]); pl->pw[0] = pool_out(pl->cw[0]);
  pl->ch[1] = conv_out(pl->ph[0], 1); pl->cw[1] = conv_out(pl->pw[0], 1);
  pl->ph[1] = pool_out(pl->ch[1]); pl->pw[1] = pool_out(pl->cw[1]);
  for (int l = 2; l < NL; ++l) {
    pl->ch[l] = conv_out(l == 2 ? pl->ph[1] : pl->ch[l - 1], l);
    pl->cw[l] = conv_out(l == 2 ? pl->pw[1] : pl->cw[l - 1], l);
  }
  if (pl->ph[1] < 1 || pl->pw[1] < 1) return false;
  size_t off = 0;
  auto take = [&](size_t floats) { const size_t o = off; off += (floats + 63) / 64 * 64; return o; };
  const size_t B2 = 2 * (size_t)B;
  pl->x0 = take(B2 * H * W * 3);
  for (int l = 0; l < NL; ++l) {
    pl->relu[l] = take(B2 * pl->ch[l] * pl->cw[l] * CONV_CO[l]);
    if (l < 2) pl->pool[l] = take(B2 * pl->ph[l] * pl->pw[l] * CONV_CO[l]);
  }
  for (int l = 0; l < NL; ++l) {
    pl->g[l] = take((size_t)B * pl->ch[l] * pl->cw[l] * CONV_CO[l]);
    if (l < 2) pl->gpool[l] = take((size_t)B * pl->ph[l] * pl->pw[l] * CONV_CO[l]);
  }
  for (int l = 0; l < NL; ++l) {
    pl->nblk[l] = (pl->ch[l] * pl->cw[l] + HEAD_PIX - 1) / HEAD_PIX;
    pl->part[l] = take(2 * (size_t)B * pl->nblk[l]);     // doubles
  }
  // scratch of the wgmma kernel (packed weight planes): one region, reused by the convs one after another
  const float* any = reinterpret_cast<const float*>((uintptr_t)256);   // stands for any 16-byte aligned buffer
  pl->tc_bytes = 0;
  for (int l = 1; l < NL; ++l) {
    for (int dg = 0; dg < 2; ++dg) {
      nlt_gconv_desc d;
      conv_desc(*pl, l, dg == 1, any, any, &d);
      const int64_t b = gconv_tc_workspace_bytes(&d, true);
      if (b < 0) return false;
      if (b > pl->tc_bytes) pl->tc_bytes = b;
    }
  }
  pl->tc = take((size_t)(pl->tc_bytes + 3) / 4);
  pl->total_floats = off;
  return true;
}

int grid_for(long long n) {
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

int launch_head(const Plan& pl, int l, const float* f, const float* lin, float gscale, double* part, float* df,
                cudaStream_t st) {
  const int HW = pl.ch[l] * pl.cw[l];
  const long long half = (long long)pl.B * HW * CONV_CO[l];
  const dim3 grid(pl.nblk[l], pl.B);
  const int mask = l == NL - 1 ? 1 : 0;
  switch (CONV_CO[l] / 32) {
    case 2: lpips_head_kernel<2><<<grid, HEAD_WARPS * 32, 0, st>>>(f, half, HW, lin, gscale, mask, part, df); break;
    case 6: lpips_head_kernel<6><<<grid, HEAD_WARPS * 32, 0, st>>>(f, half, HW, lin, gscale, mask, part, df); break;
    case 8: lpips_head_kernel<8><<<grid, HEAD_WARPS * 32, 0, st>>>(f, half, HW, lin, gscale, mask, part, df); break;
    default: lpips_head_kernel<12><<<grid, HEAD_WARPS * 32, 0, st>>>(f, half, HW, lin, gscale, mask, part, df); break;
  }
  NLT_CUDA_LAUNCH_CHECK("lpips_head_kernel");
  return NLT_OK;
}

}  // namespace
}  // namespace nlt

using namespace nlt;

extern "C" {

int64_t nlt_lpips_loss_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  Plan pl;
  if (!make_plan(B, H, W, &pl)) return -1;
  return (int64_t)pl.total_floats * 4 + 256;
}

int nlt_lpips_loss(const float* pred, const float* gt, const nlt_lpips_weights* wt, int32_t B, int32_t H, int32_t W,
                   float loss_scale, float* loss, float* d_pred, void* workspace, int64_t workspace_bytes,
                   void* stream) {
  Plan pl;
  NLT_CHECK_ARG(make_plan(B, H, W, &pl), "lpips loss: bad shape %dx%dx%d (images need H, W >= 31, B <= 65535)", B, H,
                W);
  NLT_CHECK_ARG(pred != nullptr && gt != nullptr && wt != nullptr && loss != nullptr && workspace != nullptr,
                "null pointer");
  NLT_CHECK_ARG(wt->scale != nullptr && wt->shift != nullptr, "null scaling-layer constants");
  for (int l = 0; l < NL; ++l)
    NLT_CHECK_ARG(wt->w[l] != nullptr && wt->b[l] != nullptr && wt->lin[l] != nullptr, "null constants of layer %d",
                  l + 1);
  const int64_t need = (int64_t)pl.total_floats * 4 + 256;
  NLT_CHECK_ARG(workspace_bytes >= need, "lpips workspace too small: need %lld bytes, got %lld", (long long)need,
                (long long)workspace_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  void* tcws = ws + pl.tc;
  const int64_t tcb = pl.tc_bytes;
  int rc;

  const long long n_half = (long long)B * H * W * 3;
  lpips_prep_kernel<<<grid_for(2 * n_half), 256, 0, st>>>(pred, gt, wt->scale, wt->shift, n_half, ws + pl.x0);
  NLT_CUDA_LAUNCH_CHECK("lpips_prep_kernel");
  // forward: both halves
  const float* in = ws + pl.x0;
  for (int l = 0; l < NL; ++l) {
    nlt_gconv_desc d;
    conv_desc(pl, l, false, in, wt->w[l], &d);
    rc = gconv_run(&d, wt->b[l], NLT_ACT_RELU, 0.f, nullptr, 0, ws + pl.relu[l], tcws, tcb, true, st);
    if (rc != NLT_OK) return rc;
    in = ws + pl.relu[l];
    if (l < 2) {
      const long long n = 2LL * B * pl.ph[l] * pl.pw[l] * CONV_CO[l] / 4;
      lpips_maxpool_kernel<<<grid_for(n), 256, 0, st>>>(ws + pl.relu[l], 2 * B, pl.ch[l], pl.cw[l], CONV_CO[l],
                                                        pl.ph[l], pl.pw[l], ws + pl.pool[l]);
      NLT_CUDA_LAUNCH_CHECK("lpips_maxpool_kernel");
      in = ws + pl.pool[l];
    }
  }
  // heads (and d relu_l of the pred half)
  const bool grad = d_pred != nullptr;
  for (int l = 0; l < NL; ++l) {
    rc = launch_head(pl, l, ws + pl.relu[l], wt->lin[l], loss_scale / (float)(pl.ch[l] * pl.cw[l]),
                     reinterpret_cast<double*>(ws + pl.part[l]), grad ? ws + pl.g[l] : nullptr, st);
    if (rc != NLT_OK) return rc;
  }
  SumArgs sa;
  for (int l = 0; l < NL; ++l) {
    sa.part[l] = reinterpret_cast<const double*>(ws + pl.part[l]);
    sa.nblk[l] = pl.nblk[l];
    sa.inv_hw[l] = 1.0 / ((double)pl.ch[l] * pl.cw[l]);
  }
  lpips_loss_kernel<<<B, SUM_T, 0, st>>>(sa, loss);
  NLT_CUDA_LAUNCH_CHECK("lpips_loss_kernel");
  if (!grad) return NLT_OK;

  // backward, pred half: d relu_l (+)= input gradient of conv_{l+1}, masked by relu_l
  for (int l = NL - 1; l >= 1; --l) {
    nlt_gconv_desc d;
    conv_desc(pl, l, true, ws + pl.g[l], wt->w[l], &d);
    if (l >= 3) {        // conv5 / conv4 -> d relu4 / d relu3
      rc = gconv_run(&d, nullptr, 0, 1.f, ws + pl.relu[l - 1], NLT_ACT_RELU, ws + pl.g[l - 1], tcws, tcb, true, st);
      if (rc != NLT_OK) return rc;
    } else {             // conv3 / conv2 -> d pool2 / d pool1 -> d relu2 / d relu1
      const int p = l - 1;
      rc = gconv_run(&d, nullptr, 0, 0.f, nullptr, 0, ws + pl.gpool[p], tcws, tcb, true, st);
      if (rc != NLT_OK) return rc;
      const long long n = (long long)B * pl.ch[p] * pl.cw[p] * CONV_CO[p] / 4;
      lpips_maxpool_bwd_kernel<<<grid_for(n), 256, 0, st>>>(ws + pl.relu[p], ws + pl.gpool[p], B, pl.ch[p], pl.cw[p],
                                                            CONV_CO[p], pl.ph[p], pl.pw[p], ws + pl.g[p]);
      NLT_CUDA_LAUNCH_CHECK("lpips_maxpool_bwd_kernel");
    }
  }
  nlt_gconv_desc d;
  conv_desc(pl, 0, true, ws + pl.g[0], wt->w[0], &d);
  rc = gconv_run(&d, nullptr, 0, 0.f, nullptr, 0, d_pred, tcws, tcb, true, st);
  if (rc != NLT_OK) return rc;
  lpips_prep_bwd_kernel<<<grid_for(n_half), 256, 0, st>>>(wt->scale, n_half, d_pred);
  NLT_CUDA_LAUNCH_CHECK("lpips_prep_bwd_kernel");
  return NLT_OK;
}

}  // extern "C"
