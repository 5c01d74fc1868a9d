// "ssim" training-loss term of NLT (nlt/losses.py:75-87: tf.image.ssim(gt, pred, max_val), loss = (1 - ssim) / 2)
// fused with its gradient w.r.t. pred.  TF 2.2 image_ops_impl: _fspecial_gauss(11, 1.5), _ssim_helper,
// _ssim_per_channel (depthwise VALID correlation, k1 = 0.01, k2 = 0.03, compensation 1).
//
// One CTA owns a 32 x 32 tile of input pixels of one sample and runs all three channels:
//   stage    [52 x 52 x 3] x and y (tile + 10-pixel halo on each side + 10 more for the window) by cp.async
//   rows     4 moment maps filtered along x        -> smem [4][52][42]
//   cols     ... along y, then L, CS and the adjoint coefficients A, Bc, Cc of every output pixel whose window
//            touches the tile (42 x 42, recomputed by the neighbouring tiles rather than exchanged through HBM)
//   gather   G^T applied to A, Bc, Cc (rows, then cols) -> d_pred = G^T A + x G^T Bc + 2 y G^T Cc
// Only the owned output pixels (window origin inside the tile) add to the tile's loss partial; a second kernel sums
// the partials of a sample in a fixed order in double, so the result does not depend on scheduling.
//
// Accuracy: Cd = Sxx + Syy - mx^2 - my^2 + c2 cancels badly in fp32 where the image is flat near 1.  The moments are
// therefore taken of x - kx and y - ky, with kx, ky the values of the tile's first pixel (variance and covariance
// are shift invariant; mx = mx' + kx).  The gradient uses the same shifted moments: the terms the shift moves out of
// G^T A are exactly the ones it moves into x' G^T Bc + 2 y' G^T Cc.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "nlt_b200.h"
#include "nlt_common.cuh"

namespace nlt {
namespace {

constexpr int TS = 32;             // input pixels per tile side
constexpr int WIN = 11;            // window (filter_size)
constexpr int O = TS + WIN - 1;    // output positions per side whose window touches the tile (42)
constexpr int R = O + WIN - 1;     // staged input pixels per side (52)
constexpr int NT = 256;
constexpr int HS = 6;              // row pass: outputs per thread (strip along x)
constexpr int VS = 7;              // column pass: outputs per thread (strip along y)
constexpr int GS = 4;              // gather passes: outputs per thread
constexpr int XY_FLOATS = R * R * 3;
constexpr int BUF_FLOATS = (4 * R * O > 3 * O * O + 3 * O * TS) ? 4 * R * O : 3 * O * O + 3 * O * TS;
constexpr size_t SMEM_BYTES = sizeof(float) * (2 * XY_FLOATS + BUF_FLOATS);
static_assert(O % HS == 0 && O % VS == 0 && TS % GS == 0, "strip sizes must divide the tile");
static_assert(O * (O / VS) <= NT && TS * (TS / GS) == NT, "one column-pass item / one output strip per thread");

struct Win { float g[WIN]; };      // normalised 1-D Gaussian; the 2-D window is its outer product

__device__ __forceinline__ void cp_async4_zfill(uint32_t dst, const float* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4 : 0) : "memory");
}

__global__ void __launch_bounds__(NT, 2)
ssim_tile_kernel(const float* __restrict__ pred, const float* __restrict__ gt, int H, int W, Win win, float c1,
                 float c2, float w, int grad, double* __restrict__ partial, float* __restrict__ d_pred) {
  extern __shared__ float smem[];
  float* xs = smem;                        // gt   [R][R][3]
  float* ys = smem + XY_FLOATS;            // pred [R][R][3]
  float* buf = smem + 2 * XY_FLOATS;
  const int tid = threadIdx.x;
  const int t0x = blockIdx.x * TS, t0y = blockIdx.y * TS, b = blockIdx.z;
  const size_t img = (size_t)b * H * W * 3;

  {  // stage: each region row is R * 3 contiguous floats of the NHWC image
    const uint32_t xs_u = (uint32_t)__cvta_generic_to_shared(xs), ys_u = (uint32_t)__cvta_generic_to_shared(ys);
    for (int e = tid; e < XY_FLOATS; e += NT) {
      const int r = e / (R * 3), q = e - r * (R * 3);
      const int gy = t0y - (WIN - 1) + r, gx = t0x - (WIN - 1) + q / 3;
      const bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
      const size_t off = ok ? img + ((size_t)gy * W + gx) * 3 + (q - (q / 3) * 3) : 0;
      cp_async4_zfill(xs_u + 4 * e, gt + off, ok);
      cp_async4_zfill(ys_u + 4 * e, pred + off, ok);
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    __syncthreads();
  }

  float lsum = 0.f;
  for (int c = 0; c < 3; ++c) {
    const int ref = ((WIN - 1) * R + (WIN - 1)) * 3 + c;    // the tile's first pixel, always inside the image
    const float kx = xs[ref], ky = ys[ref];

    // ---- rows: h[m][r][j] = sum_k g[k] f_m(r, j + k),  f = x', y', x'y', x'^2 + y'^2 ----
    for (int it = tid; it < R * (O / HS); it += NT) {
      const int r = it / (O / HS), j0 = (it - r * (O / HS)) * HS;
      float a[4][HS];
#pragma unroll
      for (int o = 0; o < HS; ++o) a[0][o] = a[1][o] = a[2][o] = a[3][o] = 0.f;
#pragma unroll
      for (int t = 0; t < HS + WIN - 1; ++t) {
        const int s = (r * R + j0 + t) * 3 + c;
        const float xv = xs[s] - kx, yv = ys[s] - ky;
        const float p = xv * yv, q = fmaf(xv, xv, yv * yv);
#pragma unroll
        for (int o = 0; o < HS; ++o) {
          const int k = t - o;
          if (k >= 0 && k < WIN) {
            a[0][o] = fmaf(win.g[k], xv, a[0][o]);
            a[1][o] = fmaf(win.g[k], yv, a[1][o]);
            a[2][o] = fmaf(win.g[k], p, a[2][o]);
            a[3][o] = fmaf(win.g[k], q, a[3][o]);
          }
        }
      }
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int o = 0; o < HS; ++o) buf[(m * R + r) * O + j0 + o] = a[m][o];
    }
    __syncthreads();

    // ---- columns + per-pixel terms.  Output (i, j) has its window origin at image (t0y - 10 + i, t0x - 10 + j) ----
    float cf[3][VS];
    const bool vt = tid < O * (O / VS);
    const int vj = tid % O, vi0 = (tid / O) * VS;
    if (vt) {
      float a[4][VS];
#pragma unroll
      for (int o = 0; o < VS; ++o) a[0][o] = a[1][o] = a[2][o] = a[3][o] = 0.f;
#pragma unroll
      for (int t = 0; t < VS + WIN - 1; ++t) {
        float hv[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) hv[m] = buf[(m * R + vi0 + t) * O + vj];
#pragma unroll
        for (int o = 0; o < VS; ++o) {
          const int k = t - o;
          if (k >= 0 && k < WIN) {
#pragma unroll
            for (int m = 0; m < 4; ++m) a[m][o] = fmaf(win.g[k], hv[m], a[m][o]);
          }
        }
      }
      const int oy0 = t0y - (WIN - 1) + vi0, ox = t0x - (WIN - 1) + vj;
      const bool col_ok = ox >= 0 && ox <= W - WIN;
#pragma unroll
      for (int o = 0; o < VS; ++o) {
        const int oy = oy0 + o;
        cf[0][o] = cf[1][o] = cf[2][o] = 0.f;
        if (!(col_ok && oy >= 0 && oy <= H - WIN)) continue;
        const float m0 = a[0][o], m1 = a[1][o];
        const float mx = m0 + kx, my = m1 + ky;
        const float ld = fmaf(mx, mx, fmaf(my, my, c1));
        const float lv = fmaf(2.f * mx, my, c1) / ld;
        const float cd = fmaf(-m0, m0, fmaf(-m1, m1, a[3][o])) + c2;     // sigma_x^2 + sigma_y^2 + c2
        const float cs = fmaf(2.f, fmaf(-m0, m1, a[2][o]), c2) / cd;    // (2 sigma_xy + c2) / cd
        if (vi0 + o >= WIN - 1 && vj >= WIN - 1) lsum = fmaf(lv, cs, lsum);
        if (grad) {
          cf[0][o] = w * (2.f * cs * fmaf(-lv, my, mx) / ld + 2.f * lv * fmaf(cs, m1, -m0) / cd);
          cf[1][o] = w * 2.f * lv / cd;
          cf[2][o] = -w * lv * cs / cd;
        }
      }
    }
    if (!grad) {
      __syncthreads();            // buf is rewritten by the next channel's row pass
      continue;
    }
    __syncthreads();
    float* cfs = buf;                      // [3][O][O]
    float* gh = buf + 3 * O * O;           // [3][O][TS]
    if (vt) {
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int o = 0; o < VS; ++o) cfs[(m * O + vi0 + o) * O + vj] = cf[m][o];
    }
    __syncthreads();

    // ---- gather along x: gh[m][i][u] = sum_{j = u .. u + 10} g[j - u] cf[m][i][j]  (input column u + 10) ----
    for (int it = tid; it < O * (TS / GS); it += NT) {
      const int i = it / (TS / GS), u0 = (it - i * (TS / GS)) * GS;
      float a[3][GS];
#pragma unroll
      for (int o = 0; o < GS; ++o) a[0][o] = a[1][o] = a[2][o] = 0.f;
#pragma unroll
      for (int t = 0; t < GS + WIN - 1; ++t) {
        float v[3];
#pragma unroll
        for (int m = 0; m < 3; ++m) v[m] = cfs[(m * O + i) * O + u0 + t];
#pragma unroll
        for (int o = 0; o < GS; ++o) {
          const int k = t - o;
          if (k >= 0 && k < WIN) {
#pragma unroll
            for (int m = 0; m < 3; ++m) a[m][o] = fmaf(win.g[k], v[m], a[m][o]);
          }
        }
      }
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int o = 0; o < GS; ++o) gh[(m * O + i) * TS + u0 + o] = a[m][o];
    }
    __syncthreads();

    // ---- gather along y and combine: one strip of GS input rows per thread, a warp per strip ----
    {
      const int u = tid % TS, s0 = (tid / TS) * GS;
      float a[3][GS];
#pragma unroll
      for (int o = 0; o < GS; ++o) a[0][o] = a[1][o] = a[2][o] = 0.f;
#pragma unroll
      for (int t = 0; t < GS + WIN - 1; ++t) {
        float v[3];
#pragma unroll
        for (int m = 0; m < 3; ++m) v[m] = gh[(m * O + s0 + t) * TS + u];
#pragma unroll
        for (int o = 0; o < GS; ++o) {
          const int k = t - o;
          if (k >= 0 && k < WIN) {
#pragma unroll
            for (int m = 0; m < 3; ++m) a[m][o] = fmaf(win.g[k], v[m], a[m][o]);
          }
        }
      }
      const int gx = t0x + u;
#pragma unroll
      for (int o = 0; o < GS; ++o) {
        const int gy = t0y + s0 + o;
        if (gx < W && gy < H) {
          const int s = ((s0 + o + WIN - 1) * R + u + WIN - 1) * 3 + c;
          const float xv = xs[s] - kx, yv = ys[s] - ky;
          d_pred[img + ((size_t)gy * W + gx) * 3 + c] = fmaf(xv, a[1][o], fmaf(2.f * yv, a[2][o], a[0][o]));
        }
      }
    }
    __syncthreads();
  }

  // ---- tile partial: fixed-order reduction in double ----
  double s = (double)lsum;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  __shared__ double red[NT / 32];
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int i = 0; i < NT / 32; ++i) t += red[i];
    partial[((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
  }
}

// loss[b] = (1 - mean L*CS) / 2: one CTA per sample, strided then tree sum in double (fixed order)
__global__ void __launch_bounds__(NT)
ssim_final_kernel(const double* __restrict__ partial, int ntiles, double inv_count, float* __restrict__ loss) {
  __shared__ double red[NT];
  const double* p = partial + (size_t)blockIdx.x * ntiles;
  double s = 0.0;
  for (int i = threadIdx.x; i < ntiles; i += NT) s += p[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[blockIdx.x] = (float)((1.0 - red[0] * inv_count) * 0.5);
}

bool ssim_shape_ok(int B, int H, int W) { return B > 0 && H >= WIN && W >= WIN; }

}  // namespace
}  // namespace nlt

using namespace nlt;

extern "C" {

int64_t nlt_ssim_loss_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (!ssim_shape_ok(B, H, W)) return -1;
  return (int64_t)B * ((H + TS - 1) / TS) * ((W + TS - 1) / TS) * (int64_t)sizeof(double);
}

int nlt_ssim_loss(const float* pred, const float* gt, int32_t B, int32_t H, int32_t W, float max_val, float loss_scale,
                  float* loss, float* d_pred, void* workspace, void* stream) {
  NLT_CHECK_ARG(ssim_shape_ok(B, H, W), "ssim loss: bad shape %dx%dx%d (the window needs H, W >= %d)", B, H, W, WIN);
  NLT_CHECK_ARG(pred != nullptr && gt != nullptr && loss != nullptr && workspace != nullptr, "ssim loss: null pointer");
  NLT_CHECK_ARG(max_val > 0.f, "ssim loss: max_val must be positive");
  NLT_CHECK_ARG(B <= 65535, "ssim loss: batch %d exceeds the grid's z limit", B);
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(ssim_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  // _fspecial_gauss(11, 1.5): softmax of -(i^2 + j^2) / (2 sigma^2) over the window == outer product of this
  Win win;
  double g[WIN], sum = 0.0;
  for (int i = 0; i < WIN; ++i) { const double d = i - WIN / 2; g[i] = exp(-d * d / 4.5); sum += g[i]; }
  for (int i = 0; i < WIN; ++i) win.g[i] = (float)(g[i] / sum);
  const float c1 = (0.01f * max_val) * (0.01f * max_val), c2 = (0.03f * max_val) * (0.03f * max_val);
  const long long P = (long long)(H - WIN + 1) * (W - WIN + 1);
  const float w = (float)(-(double)loss_scale / (2.0 * 3.0 * (double)P));    // d(loss_scale * loss_b) / d(L*CS)
  const dim3 grid((W + TS - 1) / TS, (H + TS - 1) / TS, B);
  double* partial = (double*)workspace;
  ssim_tile_kernel<<<grid, NT, SMEM_BYTES, st>>>(pred, gt, H, W, win, c1, c2, w, d_pred != nullptr, partial, d_pred);
  NLT_CUDA_LAUNCH_CHECK("ssim_tile_kernel");
  ssim_final_kernel<<<B, NT, 0, st>>>(partial, (int)(grid.x * grid.y), 1.0 / (3.0 * (double)P), loss);
  NLT_CUDA_LAUNCH_CHECK("ssim_final_kernel");
  return NLT_OK;
}

}  // extern "C"
