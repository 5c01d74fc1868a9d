// HBM-bound streaming kernels around the conv stack: observation mean,
// UV->camera tail (base add, corner zero, bilinear resample, alpha blend) and
// its scatter-add backward, bilinear resize, fused L2 / L1 loss + gradient, fused
// AMSGrad.  All of these are byte movers: vectorised where alignment allows,
// grids sized in multiples of the SM count with grid-stride loops.
#include "nlt_common.cuh"

namespace nlt {


static inline int grid_for(size_t n, int block, int per_sm = 8) {
  size_t b = (n + block - 1) / block;
  size_t cap = (size_t)sm_count() * per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// ---------------------------------------------------------------------------
// mean over K observations -- nlt/models/nlt.py:161-164
// ---------------------------------------------------------------------------
__global__ void kmean_fwd_kernel(const float* __restrict__ in, const float* __restrict__ wts, int K, int B,
                                 size_t per_sample, float* __restrict__ out) {
  const size_t total = (size_t)B * per_sample;
  const float invK = 1.f / (float)K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_sample);
    float s = 0.f;
    for (int k = 0; k < K; ++k) {
      float v = __ldg(in + (size_t)k * total + i);
      if (wts) v *= __ldg(wts + (size_t)b * K + k);
      s += v;
    }
    out[i] = s * invK;
  }
}

__global__ void kmean_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ wts, int K, int B,
                                 size_t per_sample, float beta, const float* __restrict__ mask_y, int mask_act,
                                 float* __restrict__ d_in) {
  const size_t total = (size_t)B * per_sample;
  const float invK = 1.f / (float)K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_sample);
    const float g = __ldg(d_out + i) * invK;
    for (int k = 0; k < K; ++k) {
      const size_t j = (size_t)k * total + i;
      float v = wts ? g * __ldg(wts + (size_t)b * K + k) : g;
      if (beta != 0.f) v += beta * d_in[j];
      if (mask_y) v *= act_bwd_from_y(__ldg(mask_y + j), mask_act);
      d_in[j] = v;
    }
  }
}

// ---------------------------------------------------------------------------
// UV -> camera tail -- nlt/models/nlt.py:99-120, 132-133
// ---------------------------------------------------------------------------
__global__ void pred_uv_kernel(const float* __restrict__ net_out, const float* __restrict__ base, int B, int H, int W,
                               int skip, float* __restrict__ pred_uv) {
  const size_t per = (size_t)H * W * 3;
  const size_t total = (size_t)B * per;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float v = __ldg(net_out + i);
    if (skip) v += __ldg(base + i);           // pred += base   (models/nlt.py:101-102)
    if (i % per < 3) v *= 0.f;                // set_left_top_corner(pred, 0) is a mask MULTIPLY (util/img.py:182-185)
    pred_uv[i] = v;
  }
}

struct Taps {
  float w[4];
  int idx[4];   // texel index (y*W+x) or -1 when the tap contributes zero
};

// tfa.image.resampler tap set for one sample point, in the reference's
// summation order: (fx,fy), (cx,cy), (fx,cy), (cx,fy)
__device__ __forceinline__ bool resampler_taps(float x, float y, int H, int W, Taps& t) {
  if (!(x > -1.f && y > -1.f && x < (float)W && y < (float)H)) return false;
  const float fx = floorf(x), fy = floorf(y);
  const float cx = fx + 1.f, cy = fy + 1.f;
  const float dx = cx - x, dy = cy - y;
  const int ifx = (int)fx, ify = (int)fy, icx = ifx + 1, icy = ify + 1;
  const bool fxok = ifx >= 0 && ifx <= W - 1, cxok = icx >= 0 && icx <= W - 1;
  const bool fyok = ify >= 0 && ify <= H - 1, cyok = icy >= 0 && icy <= H - 1;
  t.w[0] = dx * dy;                 t.idx[0] = (fxok && fyok) ? ify * W + ifx : -1;
  t.w[1] = (1.f - dx) * (1.f - dy); t.idx[1] = (cxok && cyok) ? icy * W + icx : -1;
  t.w[2] = dx * (1.f - dy);         t.idx[2] = (fxok && cyok) ? icy * W + ifx : -1;
  t.w[3] = (1.f - dx) * dy;         t.idx[3] = (cxok && fyok) ? ify * W + icx : -1;
  return true;
}

__global__ void uv2cam_fwd_kernel(const float* __restrict__ pred_uv, const float* __restrict__ base,
                                  const float* __restrict__ warp, const float* __restrict__ rgb_camspc, int B, int H,
                                  int W, int ih, int iw, float* __restrict__ pred_c, float* __restrict__ base_c,
                                  float* __restrict__ fg_c, float* __restrict__ gt_c) {
  const size_t npix = (size_t)B * ih * iw;
  const size_t per_cam = (size_t)ih * iw;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(p / per_cam);
    const float2 wv = __ldg(reinterpret_cast<const float2*>(warp) + p);
    const float x = wv.x * (float)W, y = wv.y * (float)H;   // warp * (uvw, uvh)  (models/nlt.py:104-106)
    float pr[3] = {0.f, 0.f, 0.f}, ba[3] = {0.f, 0.f, 0.f}, fg = 0.f;
    Taps t;
    if (resampler_taps(x, y, H, W, t)) {
      const float* pu = pred_uv + (size_t)b * H * W * 3;
      const float* bu = base + (size_t)b * H * W * 3;
      float tp[4][3], tb[4][3], tf[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int id = t.idx[k];
        const bool live = id > 0;   // id == 0 is texel (0,0): zeroed in fg/base/pred
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          tp[k][c] = live ? __ldg(pu + (size_t)id * 3 + c) : 0.f;
          tb[k][c] = live ? __ldg(bu + (size_t)id * 3 + c) : 0.f;
        }
        tf[k] = live ? 1.f : 0.f;
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        pr[c] = t.w[0] * tp[0][c] + t.w[1] * tp[1][c] + t.w[2] * tp[2][c] + t.w[3] * tp[3][c];
        ba[c] = t.w[0] * tb[0][c] + t.w[1] * tb[1][c] + t.w[2] * tb[2][c] + t.w[3] * tb[3][c];
      }
      fg = t.w[0] * tf[0] + t.w[1] * tf[1] + t.w[2] * tf[2] + t.w[3] * tf[3];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (pred_c) pred_c[p * 3 + c] = pr[c];
      if (base_c) base_c[p * 3 + c] = ba[c];
      if (fg_c) fg_c[p * 3 + c] = fg;
      if (gt_c) gt_c[p * 3 + c] = __ldg(rgb_camspc + p * 3 + c) * fg;   // alpha_blend (util/img.py:74-89)
    }
  }
}

__global__ void uv2cam_bwd_kernel(const float* __restrict__ d_pred_c, const float* __restrict__ warp, int B, int H,
                                  int W, int ih, int iw, float* __restrict__ d_uv) {
  const size_t npix = (size_t)B * ih * iw;
  const size_t per_cam = (size_t)ih * iw;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(p / per_cam);
    const float2 wv = __ldg(reinterpret_cast<const float2*>(warp) + p);
    const float x = wv.x * (float)W, y = wv.y * (float)H;
    Taps t;
    if (!resampler_taps(x, y, H, W, t)) continue;
    float g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = __ldg(d_pred_c + p * 3 + c);
    if (g[0] == 0.f && g[1] == 0.f && g[2] == 0.f) continue;
    float* du = d_uv + (size_t)b * H * W * 3;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int id = t.idx[k];
      if (id <= 0) continue;   // out of range, or texel (0,0) whose mask multiply kills the gradient
#pragma unroll
      for (int c = 0; c < 3; ++c) atomicAdd(du + (size_t)id * 3 + c, t.w[k] * g[c]);
    }
  }
}

// Deterministic form of the scatter: the four tap contributions are accumulated as 64-bit FIXED-POINT integers
// (integer addition is associative, so the result does not depend on the order in which the atomics land), then
// converted to fp32 in one pass that also re-zeroes the accumulator for the next call (no memset pass).
// Scale: 2^(37 - floor(log2(gmax))) with gmax = max |d_pred_camspc| of THIS call (a max-reduction, itself order
// independent): every contribution is below 2^38 in magnitude, a texel can collect all ih*iw <= 2^24 camera pixels of
// its image without overflowing 63 bits, and the quantum gmax * 2^-38 is 2^14 times finer than fp32's own
// resolution at gmax.
__global__ void absmax_kernel(const float* __restrict__ x, size_t n, unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(__ldg(x + i)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out_bits, __float_as_uint(m));   // non-negative floats order as uints
}

__device__ __forceinline__ double fixed_scale(unsigned int gmax_bits) {
  const int e = (int)((gmax_bits >> 23) & 0xffu) - 127;          // floor(log2(gmax)) for normal numbers
  return ldexp(1.0, 37 - e);
}

// Horizontally adjacent camera pixels usually share a texel column (the right taps of pixel i are the left taps of pixel
// i + 1 wherever the warp field advances about one texel per pixel): lanes hand their right-tap contributions to the next
// lane when the target texel is the same, which removes up to half of the 64-bit atomics.  Integer sums: the result
// does not depend on who adds what, so the gradient stays bit-reproducible (and bit-identical to the unmerged form).
__global__ void uv2cam_bwd_fixed_kernel(const float* __restrict__ d_pred_c, const float* __restrict__ warp, int B, int H,
                                        int W, int ih, int iw, const unsigned int* __restrict__ gmax_bits,
                                        unsigned long long* __restrict__ acc) {
  const size_t npix = (size_t)B * ih * iw;
  const size_t per_cam = (size_t)ih * iw;
  const size_t total = (npix + 31) / 32 * 32;                    // whole warps iterate together (shuffles below)
  const double scale = fixed_scale(*gmax_bits);
  const int lane = threadIdx.x & 31;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (size_t)gridDim.x * blockDim.x) {
    bool live = p < npix;
    Taps t;
    float g[3] = {0.f, 0.f, 0.f};
    int b = 0;
    if (live) {
      b = (int)(p / per_cam);
      const float2 wv = __ldg(reinterpret_cast<const float2*>(warp) + p);
      live = resampler_taps(wv.x * (float)W, wv.y * (float)H, H, W, t);
    }
    if (live) {
#pragma unroll
      for (int c = 0; c < 3; ++c) g[c] = __ldg(d_pred_c + p * 3 + c);
      live = !(g[0] == 0.f && g[1] == 0.f && g[2] == 0.f);
    }
    int id[4];
    long long q[4][3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // id <= 0: out of range, or texel (0,0) whose mask multiply kills the gradient
      id[k] = (live && t.idx[k] > 0) ? b * H * W + t.idx[k] : -1;
#pragma unroll
      for (int c = 0; c < 3; ++c) q[k][c] = id[k] >= 0 ? __double2ll_rn((double)(t.w[k] * g[c]) * scale) : 0ll;
    }
    // taps: 0 = (fx,fy), 1 = (cx,cy), 2 = (fx,cy), 3 = (cx,fy): right taps 3 / 1 go to the next lane's left taps 0 / 2
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      const int kr = pr == 0 ? 3 : 1, kl = pr == 0 ? 0 : 2;
      const int nid = __shfl_down_sync(0xffffffffu, id[kl], 1);
      const bool give = lane < 31 && id[kr] >= 0 && nid == id[kr];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const long long recv = __shfl_up_sync(0xffffffffu, give ? q[kr][c] : 0ll, 1);
        if (lane > 0) q[kl][c] += recv;
      }
      if (give) id[kr] = -1;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (id[k] < 0) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (q[k][c] != 0) atomicAdd(acc + (size_t)id[k] * 3 + c, (unsigned long long)q[k][c]);   // two's complement: signed sum
    }
  }
}

__global__ void fixed_to_float_kernel(unsigned long long* __restrict__ acc, size_t n,
                                      const unsigned int* __restrict__ gmax_bits, float* __restrict__ out) {
  const double inv = 1.0 / fixed_scale(*gmax_bits);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const long long v = (long long)acc[i];
    out[i] = (float)((double)v * inv);
    if (v != 0) acc[i] = 0ull;                 // leave the accumulator zeroed for the next call
  }
}

// ---------------------------------------------------------------------------
// tf.image.resize bilinear, half-pixel centres -- nlt/util/img.py:113-116
// ---------------------------------------------------------------------------
__device__ __forceinline__ void resize_coef(int o, float scale, int n_in, int& lo, int& hi, float& l) {
  const float src = ((float)o + 0.5f) * scale - 0.5f;
  const float f = floorf(src);
  lo = max((int)f, 0);
  hi = min((int)ceilf(src), n_in - 1);
  l = src - f;
}

__global__ void resize_fwd_kernel(const float* __restrict__ in, int B, int H, int W, int C, int oh, int ow,
                                  float* __restrict__ out) {
  const size_t total = (size_t)B * oh * ow * C;
  const float sy = (float)H / (float)oh, sx = (float)W / (float)ow;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int ox = (int)(r % ow); r /= ow;
    const int oy = (int)(r % oh);
    const int b = (int)(r / oh);
    int y0, y1, x0, x1; float ly, lx;
    resize_coef(oy, sy, H, y0, y1, ly);
    resize_coef(ox, sx, W, x0, x1, lx);
    const float* ib = in + (size_t)b * H * W * C + c;
    const float tl = __ldg(ib + ((size_t)y0 * W + x0) * C), tr = __ldg(ib + ((size_t)y0 * W + x1) * C);
    const float bl = __ldg(ib + ((size_t)y1 * W + x0) * C), br = __ldg(ib + ((size_t)y1 * W + x1) * C);
    const float top = tl * (1.f - lx) + tr * lx, bot = bl * (1.f - lx) + br * lx;
    out[i] = top * (1.f - ly) + bot * ly;
  }
}

__global__ void resize_bwd_kernel(const float* __restrict__ d_out, int B, int H, int W, int C, int oh, int ow,
                                  float* __restrict__ d_in) {
  const size_t total = (size_t)B * oh * ow * C;
  const float sy = (float)H / (float)oh, sx = (float)W / (float)ow;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int ox = (int)(r % ow); r /= ow;
    const int oy = (int)(r % oh);
    const int b = (int)(r / oh);
    int y0, y1, x0, x1; float ly, lx;
    resize_coef(oy, sy, H, y0, y1, ly);
    resize_coef(ox, sx, W, x0, x1, lx);
    const float g = __ldg(d_out + i);
    float* ib = d_in + (size_t)b * H * W * C + c;
    atomicAdd(ib + ((size_t)y0 * W + x0) * C, g * (1.f - ly) * (1.f - lx));
    atomicAdd(ib + ((size_t)y0 * W + x1) * C, g * (1.f - ly) * lx);
    atomicAdd(ib + ((size_t)y1 * W + x0) * C, g * ly * (1.f - lx));
    atomicAdd(ib + ((size_t)y1 * W + x1) * C, g * ly * lx);
  }
}

// ---------------------------------------------------------------------------
// L2 loss (keep_batch) + gradient -- nlt/losses.py:39-53, trainvali.py:277-278
// ---------------------------------------------------------------------------
constexpr int L2_BLOCKS_PER_SAMPLE = 64;
constexpr int L2_THREADS = 256;

__global__ void l2_partial_kernel(const float* __restrict__ pred, const float* __restrict__ gt, size_t per_sample,
                                  float dscale, float* __restrict__ partial, float* __restrict__ d_pred) {
  const int b = blockIdx.y;
  const float* pp = pred + (size_t)b * per_sample;
  const float* gg = gt + (size_t)b * per_sample;
  float* dp = d_pred ? d_pred + (size_t)b * per_sample : nullptr;
  float s = 0.f;
  if ((per_sample & 3) == 0 && ((((uintptr_t)pp) | ((uintptr_t)gg) | ((uintptr_t)dp)) & 15) == 0) {
    // 16-byte path (every shape of the model: 3 channels x an even image): four independent partial sums per thread
    const float4* p4 = reinterpret_cast<const float4*>(pp);
    const float4* g4 = reinterpret_cast<const float4*>(gg);
    float4* d4 = reinterpret_cast<float4*>(dp);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    const size_t n4 = per_sample >> 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      const float4 a = __ldg(p4 + i), b4 = __ldg(g4 + i);
      const float4 d = make_float4(a.x - b4.x, a.y - b4.y, a.z - b4.z, a.w - b4.w);
      s0 = fmaf(d.x, d.x, s0); s1 = fmaf(d.y, d.y, s1); s2 = fmaf(d.z, d.z, s2); s3 = fmaf(d.w, d.w, s3);
      if (dp) d4[i] = make_float4(d.x * dscale, d.y * dscale, d.z * dscale, d.w * dscale);
    }
    s = (s0 + s1) + (s2 + s3);
  } else {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_sample; i += (size_t)gridDim.x * blockDim.x) {
      const float d = __ldg(pp + i) - __ldg(gg + i);
      s = fmaf(d, d, s);
      if (dp) dp[i] = d * dscale;
    }
  }
  __shared__ float red[L2_THREADS];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = L2_THREADS / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[(size_t)b * gridDim.x + blockIdx.x] = red[0];
}

__global__ void l2_final_kernel(const float* __restrict__ partial, int B, int nblk, float inv_n,
                                float* __restrict__ loss) {
  // one thread per sample, fixed summation order -> deterministic
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float s = 0.f;
  for (int i = 0; i < nblk; ++i) s += partial[(size_t)b * nblk + i];
  loss[b] = s * inv_n;
}

// ---------------------------------------------------------------------------
// L1 loss (keep_batch) + gradient -- nlt/losses.py:27-36 (MeanAbsoluteError, then reduce_mean)
// Same grid as the L2 pair.  d_pred = sign(pred - gt) * dscale, exactly 0 on ties (TF's Abs gradient).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float l1_grad(float d, float dscale) {
  return d > 0.f ? dscale : (d < 0.f ? -dscale : d * dscale);    // d * dscale: 0 on ties, NaN stays NaN
}

__global__ void l1_partial_kernel(const float* __restrict__ pred, const float* __restrict__ gt, size_t per_sample,
                                  float dscale, float* __restrict__ partial, float* __restrict__ d_pred) {
  const int b = blockIdx.y;
  const float* pp = pred + (size_t)b * per_sample;
  const float* gg = gt + (size_t)b * per_sample;
  float* dp = d_pred ? d_pred + (size_t)b * per_sample : nullptr;
  float s = 0.f;
  if ((per_sample & 3) == 0 && ((((uintptr_t)pp) | ((uintptr_t)gg) | ((uintptr_t)dp)) & 15) == 0) {
    const float4* p4 = reinterpret_cast<const float4*>(pp);
    const float4* g4 = reinterpret_cast<const float4*>(gg);
    float4* d4 = reinterpret_cast<float4*>(dp);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    const size_t n4 = per_sample >> 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      const float4 a = __ldg(p4 + i), b4 = __ldg(g4 + i);
      const float4 d = make_float4(a.x - b4.x, a.y - b4.y, a.z - b4.z, a.w - b4.w);
      s0 += fabsf(d.x); s1 += fabsf(d.y); s2 += fabsf(d.z); s3 += fabsf(d.w);
      if (dp) d4[i] = make_float4(l1_grad(d.x, dscale), l1_grad(d.y, dscale), l1_grad(d.z, dscale), l1_grad(d.w, dscale));
    }
    s = (s0 + s1) + (s2 + s3);
  } else {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_sample; i += (size_t)gridDim.x * blockDim.x) {
      const float d = __ldg(pp + i) - __ldg(gg + i);
      s += fabsf(d);
      if (dp) dp[i] = l1_grad(d, dscale);
    }
  }
  __shared__ float red[L2_THREADS];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = L2_THREADS / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[(size_t)b * gridDim.x + blockIdx.x] = red[0];
}

__global__ void l1_final_kernel(const float* __restrict__ partial, int B, int nblk, double inv_n,
                                float* __restrict__ loss) {
  // one thread per sample, fixed summation order in double -> deterministic
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double s = 0.0;
  for (int i = 0; i < nblk; ++i) s += partial[(size_t)b * nblk + i];
  loss[b] = (float)(s * inv_n);
}

// ---------------------------------------------------------------------------
// AMSGrad -- tf.keras.optimizers.Adam(amsgrad=True), nlt/trainvali.py:122-127
// ---------------------------------------------------------------------------
__global__ void amsgrad_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                               float* __restrict__ v, float* __restrict__ vhat, size_t n, float lr_t, float b1,
                               float b2, float eps, float gscale) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    const float mi = m[i] + (gi - m[i]) * (1.f - b1);
    const float vi = v[i] + (gi * gi - v[i]) * (1.f - b2);
    const float vh = fmaxf(vhat[i], vi);
    m[i] = mi; v[i] = vi; vhat[i] = vh;
    p[i] = p[i] - lr_t * mi / (sqrtf(vh) + eps);
  }
}

// ---------------------------------------------------------------------------
// small streaming helpers of the test-time feature cache (nlt/nlt_test.py:97-127) and the resize branch
// ---------------------------------------------------------------------------
__global__ void ksum_acc_kernel(const float* __restrict__ in, int K, size_t per, float* __restrict__ acc) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (size_t)gridDim.x * blockDim.x) {
    float s = acc[i];
    for (int k = 0; k < K; ++k) s += __ldg(in + (size_t)k * per + i);   // fixed order: deterministic
    acc[i] = s;
  }
}
__global__ void scale_kernel(float* __restrict__ x, size_t n, float a) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] *= a;
}
__global__ void mul_kernel(const float* __restrict__ a, const float* __restrict__ b, size_t n, float* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __ldg(a + i) * __ldg(b + i);
}

// uint8 image bytes (PNG samples) -> float32 in [0, 1]: out = v / 255, correctly rounded -- bit-identical to the
// host pipeline's float32(v / 255.0) for all 256 values (nlt/datasets/nlt.py:134-139 via xiuminglib normalize_uint)
__global__ void u8_to_f32_kernel(const uint8_t* __restrict__ in, size_t n, float* __restrict__ out) {
  const size_t n16 = n / 16;
  const uint4* in16 = reinterpret_cast<const uint4*>(in);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(in16 + i);
    const unsigned int w[4] = {v.x, v.y, v.z, v.w};
    float4* o = reinterpret_cast<float4*>(out + i * 16);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      o[j] = make_float4(__fdiv_rn((float)(w[j] & 0xffu), 255.f), __fdiv_rn((float)((w[j] >> 8) & 0xffu), 255.f),
                         __fdiv_rn((float)((w[j] >> 16) & 0xffu), 255.f), __fdiv_rn((float)(w[j] >> 24), 255.f));
  }
  for (size_t i = n16 * 16 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __fdiv_rn((float)in[i], 255.f);
}

// Same update with the step counter ON THE DEVICE, so that the optimiser launch can live inside a captured CUDA
// graph (a host-computed bias-corrected learning rate would be frozen into the graph at capture time).
// `step` holds the number of updates applied so far; it is advanced by amsgrad_step_inc_kernel right before.
__global__ void amsgrad_step_inc_kernel(int* __restrict__ step) { *step += 1; }

__global__ void amsgrad_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                   float* __restrict__ v, float* __restrict__ vhat, size_t n,
                                   const int* __restrict__ step, float lr, float b1, float b2, float eps, float gscale) {
  __shared__ float lr_s;
  if (threadIdx.x == 0) {
    const int t = *step;
    lr_s = (float)((double)lr * sqrt(1.0 - pow((double)b2, (double)t)) / (1.0 - pow((double)b1, (double)t)));
  }
  __syncthreads();
  const float lr_t = lr_s;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    const float mi = m[i] + (gi - m[i]) * (1.f - b1);
    const float vi = v[i] + (gi * gi - v[i]) * (1.f - b2);
    const float vh = fmaxf(vhat[i], vi);
    m[i] = mi; v[i] = vi; vhat[i] = vh;
    p[i] = p[i] - lr_t * mi / (sqrtf(vh) + eps);
  }
}

}  // namespace nlt

using namespace nlt;

extern "C" {

int nlt_kmean_fwd(const float* in, const float* weights, int32_t K, int32_t B, int64_t per_sample, float* out,
                  void* stream) {
  NLT_CHECK_ARG(in && out && K > 0 && B > 0 && per_sample > 0, "kmean_fwd: bad argument");
  const size_t total = (size_t)B * per_sample;
  kmean_fwd_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, weights, K, B, (size_t)per_sample, out);
  NLT_CUDA_LAUNCH_CHECK("kmean_fwd_kernel");
  return NLT_OK;
}

int nlt_kmean_bwd(const float* d_out, const float* weights, int32_t K, int32_t B, int64_t per_sample, float beta,
                  const float* mask_y, int mask_act, float* d_in, void* stream) {
  NLT_CHECK_ARG(d_out && d_in && K > 0 && B > 0 && per_sample > 0, "kmean_bwd: bad argument");
  const size_t total = (size_t)B * per_sample;
  kmean_bwd_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(d_out, weights, K, B, (size_t)per_sample,
                                                                             beta, mask_y, mask_act, d_in);
  NLT_CUDA_LAUNCH_CHECK("kmean_bwd_kernel");
  return NLT_OK;
}

int nlt_uv2cam_fwd(const float* net_out, const float* base, const float* warp, const float* rgb_camspc, int32_t B,
                   int32_t H, int32_t W, int32_t ih, int32_t iw, int32_t skip_connect_base, float* pred_uv,
                   float* pred_camspc, float* base_camspc, float* fg_camspc, float* gt_camspc, void* stream) {
  NLT_CHECK_ARG(net_out && base && warp && pred_uv, "uv2cam_fwd: null pointer");
  NLT_CHECK_ARG(B > 0 && H > 0 && W > 0 && ih > 0 && iw > 0, "uv2cam_fwd: bad geometry");
  NLT_CHECK_ARG(gt_camspc == nullptr || rgb_camspc != nullptr, "uv2cam_fwd: gt_camspc needs rgb_camspc");
  NLT_CHECK_ARG((long long)H * W < (1ll << 30), "uv2cam_fwd: UV map too large");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_uv = (size_t)B * H * W * 3;
  pred_uv_kernel<<<grid_for(n_uv, 256), 256, 0, st>>>(net_out, base, B, H, W, skip_connect_base, pred_uv);
  NLT_CUDA_LAUNCH_CHECK("pred_uv_kernel");
  if (pred_camspc || base_camspc || fg_camspc || gt_camspc) {
    const size_t npix = (size_t)B * ih * iw;
    uv2cam_fwd_kernel<<<grid_for(npix, 256), 256, 0, st>>>(pred_uv, base, warp, rgb_camspc, B, H, W, ih, iw,
                                                            pred_camspc, base_camspc, fg_camspc, gt_camspc);
    NLT_CUDA_LAUNCH_CHECK("uv2cam_fwd_kernel");
  }
  return NLT_OK;
}

int nlt_uv2cam_bwd(const float* d_pred_camspc, const float* warp, int32_t B, int32_t H, int32_t W, int32_t ih,
                   int32_t iw, float* d_net_out, void* stream) {
  NLT_CHECK_ARG(d_pred_camspc && warp && d_net_out, "uv2cam_bwd: null pointer");
  NLT_CHECK_ARG(B > 0 && H > 0 && W > 0 && ih > 0 && iw > 0, "uv2cam_bwd: bad geometry");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(d_net_out, 0, (size_t)B * H * W * 3 * sizeof(float), st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "memset: %s", cudaGetErrorString(e));
  const size_t npix = (size_t)B * ih * iw;
  uv2cam_bwd_kernel<<<grid_for(npix, 256), 256, 0, st>>>(d_pred_camspc, warp, B, H, W, ih, iw, d_net_out);
  NLT_CUDA_LAUNCH_CHECK("uv2cam_bwd_kernel");
  return NLT_OK;
}

int64_t nlt_uv2cam_bwd_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0) return -1;
  return (int64_t)B * H * W * 3 * 8 + 256;
}

int nlt_uv2cam_bwd_det(const float* d_pred_camspc, const float* warp, int32_t B, int32_t H, int32_t W, int32_t ih,
                       int32_t iw, float* d_net_out, void* workspace, void* stream) {
  NLT_CHECK_ARG(d_pred_camspc && warp && d_net_out && workspace, "uv2cam_bwd_det: null pointer");
  NLT_CHECK_ARG(B > 0 && H > 0 && W > 0 && ih > 0 && iw > 0, "uv2cam_bwd_det: bad geometry");
  NLT_CHECK_ARG((long long)ih * iw <= (1ll << 24), "uv2cam_bwd_det: camera image too large for the fixed-point range");
  NLT_CHECK_ARG((((uintptr_t)workspace) & 7) == 0, "uv2cam_bwd_det: workspace must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* gmax = reinterpret_cast<unsigned int*>(workspace);            // first 256 bytes: the max scalar
  unsigned long long* acc = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(workspace) + 256);
  cudaError_t e = cudaMemsetAsync(gmax, 0, 4, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "memset: %s", cudaGetErrorString(e));
  const size_t npix = (size_t)B * ih * iw;
  absmax_kernel<<<grid_for(npix * 3, 256, 4), 256, 0, st>>>(d_pred_camspc, npix * 3, gmax);
  NLT_CUDA_LAUNCH_CHECK("absmax_kernel");
  uv2cam_bwd_fixed_kernel<<<grid_for(npix, 256), 256, 0, st>>>(d_pred_camspc, warp, B, H, W, ih, iw, gmax, acc);
  NLT_CUDA_LAUNCH_CHECK("uv2cam_bwd_fixed_kernel");
  const size_t n = (size_t)B * H * W * 3;
  fixed_to_float_kernel<<<grid_for(n, 256), 256, 0, st>>>(acc, n, gmax, d_net_out);
  NLT_CUDA_LAUNCH_CHECK("fixed_to_float_kernel");
  return NLT_OK;
}

int nlt_resize_bilinear_fwd(const float* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow,
                            float* out, void* stream) {
  NLT_CHECK_ARG(in && out && B > 0 && H > 0 && W > 0 && C > 0 && oh > 0 && ow > 0, "resize_fwd: bad argument");
  const size_t total = (size_t)B * oh * ow * C;
  resize_fwd_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, B, H, W, C, oh, ow, out);
  NLT_CUDA_LAUNCH_CHECK("resize_fwd_kernel");
  return NLT_OK;
}

int nlt_resize_bilinear_bwd(const float* d_out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow,
                            float* d_in, void* stream) {
  NLT_CHECK_ARG(d_out && d_in && B > 0 && H > 0 && W > 0 && C > 0 && oh > 0 && ow > 0, "resize_bwd: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(d_in, 0, (size_t)B * H * W * C * sizeof(float), st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "memset: %s", cudaGetErrorString(e));
  const size_t total = (size_t)B * oh * ow * C;
  resize_bwd_kernel<<<grid_for(total, 256), 256, 0, st>>>(d_out, B, H, W, C, oh, ow, d_in);
  NLT_CUDA_LAUNCH_CHECK("resize_bwd_kernel");
  return NLT_OK;
}

int64_t nlt_l2_loss_workspace_bytes(int32_t B, int64_t per_sample) {
  (void)per_sample;
  return (int64_t)B * L2_BLOCKS_PER_SAMPLE * sizeof(float);
}

int nlt_l2_loss(const float* pred, const float* gt, int32_t B, int64_t per_sample, float loss_scale, float* loss,
                float* d_pred, void* workspace, void* stream) {
  NLT_CHECK_ARG(pred && gt && loss && workspace && B > 0 && per_sample > 0, "l2_loss: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  float* partial = (float*)workspace;
  const float dscale = 2.f * loss_scale / (float)per_sample;
  dim3 grid(L2_BLOCKS_PER_SAMPLE, B);
  l2_partial_kernel<<<grid, L2_THREADS, 0, st>>>(pred, gt, (size_t)per_sample, dscale, partial, d_pred);
  NLT_CUDA_LAUNCH_CHECK("l2_partial_kernel");
  l2_final_kernel<<<(B + 31) / 32, 32, 0, st>>>(partial, B, L2_BLOCKS_PER_SAMPLE, 1.f / (float)per_sample, loss);
  NLT_CUDA_LAUNCH_CHECK("l2_final_kernel");
  return NLT_OK;
}

int64_t nlt_l1_loss_workspace_bytes(int32_t B, int64_t per_sample) {
  if (B <= 0 || per_sample <= 0) return -1;
  return (int64_t)B * L2_BLOCKS_PER_SAMPLE * sizeof(float);
}

int nlt_l1_loss(const float* pred, const float* gt, int32_t B, int64_t per_sample, float loss_scale, float* loss,
                float* d_pred, void* workspace, void* stream) {
  NLT_CHECK_ARG(pred && gt && loss && workspace && B > 0 && B <= 65535 && per_sample > 0, "l1_loss: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  float* partial = (float*)workspace;
  const float dscale = (float)((double)loss_scale / (double)per_sample);
  dim3 grid(L2_BLOCKS_PER_SAMPLE, B);
  l1_partial_kernel<<<grid, L2_THREADS, 0, st>>>(pred, gt, (size_t)per_sample, dscale, partial, d_pred);
  NLT_CUDA_LAUNCH_CHECK("l1_partial_kernel");
  l1_final_kernel<<<(B + 31) / 32, 32, 0, st>>>(partial, B, L2_BLOCKS_PER_SAMPLE, 1.0 / (double)per_sample, loss);
  NLT_CUDA_LAUNCH_CHECK("l1_final_kernel");
  return NLT_OK;
}

int nlt_amsgrad_step(float* p, const float* g, float* m, float* v, float* vhat, int64_t n, int32_t step, float lr,
                     float beta1, float beta2, float eps, float grad_scale, void* stream) {
  NLT_CHECK_ARG(p && g && m && v && vhat && n > 0 && step >= 1, "amsgrad: bad argument");
  const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, step)) / (1.0 - pow((double)beta1, step));
  amsgrad_kernel<<<grid_for((size_t)n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, vhat, (size_t)n, (float)lr_t,
                                                                              beta1, beta2, eps, grad_scale);
  NLT_CUDA_LAUNCH_CHECK("amsgrad_kernel");
  return NLT_OK;
}

int nlt_ksum_acc(const float* in, int32_t K, int64_t per_sample, float* acc, void* stream) {
  NLT_CHECK_ARG(in && acc && K > 0 && per_sample > 0, "ksum_acc: bad argument");
  ksum_acc_kernel<<<grid_for((size_t)per_sample, 256), 256, 0, (cudaStream_t)stream>>>(in, K, (size_t)per_sample, acc);
  NLT_CUDA_LAUNCH_CHECK("ksum_acc_kernel");
  return NLT_OK;
}

int nlt_scale(float* x, int64_t n, float a, void* stream) {
  NLT_CHECK_ARG(x && n > 0, "scale: bad argument");
  scale_kernel<<<grid_for((size_t)n, 256), 256, 0, (cudaStream_t)stream>>>(x, (size_t)n, a);
  NLT_CUDA_LAUNCH_CHECK("scale_kernel");
  return NLT_OK;
}

int nlt_mul(const float* a, const float* b, int64_t n, float* out, void* stream) {
  NLT_CHECK_ARG(a && b && out && n > 0, "mul: bad argument");
  mul_kernel<<<grid_for((size_t)n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, (size_t)n, out);
  NLT_CUDA_LAUNCH_CHECK("mul_kernel");
  return NLT_OK;
}

int nlt_u8_to_f32(const uint8_t* in, int64_t n, float* out, void* stream) {
  NLT_CHECK_ARG(in && out && n > 0, "u8_to_f32: bad argument");
  NLT_CHECK_ARG((((uintptr_t)in) & 15) == 0 && (((uintptr_t)out) & 15) == 0, "u8_to_f32: pointers must be 16-byte aligned");
  u8_to_f32_kernel<<<grid_for((size_t)n / 16 + 1, 256), 256, 0, (cudaStream_t)stream>>>(in, (size_t)n, out);
  NLT_CUDA_LAUNCH_CHECK("u8_to_f32_kernel");
  return NLT_OK;
}

int nlt_amsgrad_step_dev(float* p, const float* g, float* m, float* v, float* vhat, int64_t n, int32_t* step_dev,
                         float lr, float beta1, float beta2, float eps, float grad_scale, void* stream) {
  NLT_CHECK_ARG(p && g && m && v && vhat && step_dev && n > 0, "amsgrad_dev: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  amsgrad_step_inc_kernel<<<1, 1, 0, st>>>(step_dev);
  NLT_CUDA_LAUNCH_CHECK("amsgrad_step_inc_kernel");
  amsgrad_dev_kernel<<<grid_for((size_t)n, 256), 256, 0, st>>>(p, g, m, v, vhat, (size_t)n, step_dev, lr, beta1, beta2,
                                                               eps, grad_scale);
  NLT_CUDA_LAUNCH_CHECK("amsgrad_dev_kernel");
  return NLT_OK;
}

}  // extern "C"
