// "barron" training-loss term of NLT (nlt/losses.py:90-121) fused with its gradient -- SURVEY.md 8f, row N1.
// The per-element arithmetic (nlt_barron_core.h) is checked on the CPU against the pinned oracle, the kernels by
// tests/test_gpu_barron.py.
//
// Planar fp32 scratch ([3B planes][rows][cols]); per level l (image A x B):
//   rows pass : L[ceil(A/2)][B], H[floor(A/2)][B]
//   cols pass : LL -> next level's image;  LH, HL, HH -> loss sum + gradient stored in place of the coefficient
// backward walks the levels upwards with the exact adjoint (gather form), then maps the YUV gradient back to
// RGB, applies the alpha blend and the sign of d(gt - pred)/d(pred).
#include <cuda_runtime.h>
#include <stdint.h>

#include "nlt_b200.h"
#include "nlt_barron_core.h"
#include "nlt_common.cuh"

namespace nlt {
namespace {

using namespace nlt_barron;
constexpr int BT = 256;
constexpr int MAX_LEVELS = 12;

// Per-sample loss sums: a block is plane-major, so almost every block (and every warp) belongs to one sample ->
// shuffle-reduce per warp, combine the warps in shared memory, ONE atomic per block and sample.  EVERY thread of the
// block must call this (no early returns before it).
__device__ __forceinline__ void block_accumulate(float part, int sample, float* loss_acc) {
  __shared__ float sp[BT / 32];
  __shared__ int ss[BT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s0 = __shfl_sync(0xffffffffu, sample, 0);
  const bool uniform = __all_sync(0xffffffffu, sample == s0);
  float v = part;
  if (uniform) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  } else if (part != 0.f) {
    atomicAdd(loss_acc + sample, part);       // a warp straddling two samples (once per plane boundary at most)
    v = 0.f;
  }
  if (lane == 0) { sp[warp] = uniform ? v : 0.f; ss[warp] = s0; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float run = sp[0];
    int cur = ss[0];
    for (int w = 1; w < BT / 32; ++w) {
      if (ss[w] == cur) { run += sp[w]; continue; }
      if (run != 0.f) atomicAdd(loss_acc + cur, run);
      run = sp[w]; cur = ss[w];
    }
    if (run != 0.f) atomicAdd(loss_acc + cur, run);
  }
}

// residual -> scaled YUV planes
__global__ void __launch_bounds__(BT)
barron_prep_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ alpha,
                   int B, long long hw, float* __restrict__ x0) {
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= (long long)B * hw) return;
  const long long b = idx / hw, p = idx - b * hw;
  const float a = alpha ? __ldg(alpha + idx) : 1.f;
  const float r = (__ldg(gt + idx * 3 + 0) - __ldg(pred + idx * 3 + 0)) * a;
  const float g = (__ldg(gt + idx * 3 + 1) - __ldg(pred + idx * 3 + 1)) * a;
  const float bl = (__ldg(gt + idx * 3 + 2) - __ldg(pred + idx * 3 + 2)) * a;
  float y, u, v;
  rgb_to_syuv(r, g, bl, &y, &u, &v);
  x0[(b * 3 + 0) * hw + p] = y;
  x0[(b * 3 + 1) * hw + p] = u;
  x0[(b * 3 + 2) * hw + p] = v;
}

// analysis along axis 0 (rows): x [P][A][Bc] -> lo [P][ceil(A/2)][Bc], hi [P][floor(A/2)][Bc]
__global__ void __launch_bounds__(BT)
barron_rows_kernel(const float* __restrict__ x, int P, int A, int Bc, float* __restrict__ lo, float* __restrict__ hi) {
  const int nl = n_lo(A), nh = n_hi(A);
  const long long total = (long long)P * nl * Bc;
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % Bc);
  const int j = (int)((idx / Bc) % nl);
  const int p = (int)(idx / ((long long)Bc * nl));
  const float* col = x + (long long)p * A * Bc + c;
  lo[((long long)p * nl + j) * Bc + c] = analysis_lo(col, A, Bc, j);
  if (j < nh) hi[((long long)p * nh + j) * Bc + c] = analysis_hi(col, A, Bc, j);
}

// analysis along axis 1 (columns) of one row-pass output `src` [P][R][Bc]:
//   keep_lo != 0: the low-pass output is the next level's image (stored as is); else it is a band
//   bands: coefficient -> loss contribution (atomically summed per sample) and, in place, its gradient
__global__ void __launch_bounds__(BT)
barron_cols_kernel(const float* __restrict__ src, int P, int R, int Bc, float* __restrict__ out_lo,
                   float* __restrict__ out_hi, int keep_lo, float inv_scale, float gscale,
                   float* __restrict__ loss_acc) {
  const int nl = n_lo(Bc), nh = n_hi(Bc);
  const long long total = (long long)P * R * nl;
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  float part = 0.f;
  int sample = (P - 1) / 3;      // tail threads of the grid sit behind the last plane
  if (idx < total) {
    const int j = (int)(idx % nl);
    const int r = (int)((idx / nl) % R);
    const int p = (int)(idx / ((long long)nl * R));
    sample = p / 3;
    const float* row = src + ((long long)p * R + r) * Bc;
    const float l = analysis_lo(row, Bc, 1, j);
    if (keep_lo) {
      out_lo[((long long)p * R + r) * nl + j] = l;
    } else {
      part += charbonnier(l, inv_scale);
      out_lo[((long long)p * R + r) * nl + j] = gscale * charbonnier_grad(l, inv_scale);
    }
    if (j < nh) {
      const float h = analysis_hi(row, Bc, 1, j);
      part += charbonnier(h, inv_scale);
      out_hi[((long long)p * R + r) * nh + j] = gscale * charbonnier_grad(h, inv_scale);
    }
  }
  block_accumulate(part, sample, loss_acc);
}

// coarsest residual image: loss + gradient in place
__global__ void __launch_bounds__(BT)
barron_resid_kernel(float* __restrict__ img, int P, long long per_plane, float inv_scale, float gscale,
                    float* __restrict__ loss_acc) {
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= (long long)P * per_plane) return;
  const int p = (int)(idx / per_plane);
  const float w = img[idx];
  atomicAdd(loss_acc + p / 3, charbonnier(w, inv_scale));
  img[idx] = gscale * charbonnier_grad(w, inv_scale);
}

// adjoint of the columns pass: g_lo [P][R][ceil(Bc/2)], g_hi [P][R][floor(Bc/2)] -> out [P][R][Bc]
__global__ void __launch_bounds__(BT)
barron_cols_adj_kernel(const float* __restrict__ g_lo, const float* __restrict__ g_hi, int P, int R, int Bc,
                       float* __restrict__ out) {
  const int nl = n_lo(Bc), nh = n_hi(Bc);
  const long long total = (long long)P * R * Bc;
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= total) return;
  const int i = (int)(idx % Bc);
  const long long pr = idx / Bc;
  out[idx] = adjoint_at(g_lo + pr * nl, g_hi + pr * nh, Bc, 1, 1, i);
}

// adjoint of the rows pass: g_lo [P][ceil(A/2)][Bc], g_hi [P][floor(A/2)][Bc] -> out [P][A][Bc]
__global__ void __launch_bounds__(BT)
barron_rows_adj_kernel(const float* __restrict__ g_lo, const float* __restrict__ g_hi, int P, int A, int Bc,
                       float* __restrict__ out) {
  const int nl = n_lo(A), nh = n_hi(A);
  const long long total = (long long)P * A * Bc;
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= total) return;
  const int c = (int)(idx % Bc);
  const int i = (int)((idx / Bc) % A);
  const int p = (int)(idx / ((long long)Bc * A));
  out[idx] = adjoint_at(g_lo + (long long)p * nl * Bc + c, g_hi + (long long)p * nh * Bc + c, A, Bc, Bc, i);
}

// YUV-plane gradient -> d_pred (NHWC), and the per-sample loss values
__global__ void __launch_bounds__(BT)
barron_finish_kernel(const float* __restrict__ gx0, const float* __restrict__ alpha, int B, long long hw,
                     float* __restrict__ d_pred) {
  const long long idx = (long long)blockIdx.x * BT + threadIdx.x;
  if (idx >= (long long)B * hw) return;
  const long long b = idx / hw, p = idx - b * hw;
  float r, g, bl;
  syuv_to_rgb_transpose(gx0[(b * 3 + 0) * hw + p], gx0[(b * 3 + 1) * hw + p], gx0[(b * 3 + 2) * hw + p], &r, &g, &bl);
  const float a = alpha ? -__ldg(alpha + idx) : -1.f;       // residual = (gt - pred) * alpha
  d_pred[idx * 3 + 0] = a * r;
  d_pred[idx * 3 + 1] = a * g;
  d_pred[idx * 3 + 2] = a * bl;
}

__global__ void barron_loss_kernel(const float* __restrict__ loss_acc, int B, float inv_count, float constant,
                                   float* __restrict__ loss) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) loss[b] = loss_acc[b] * inv_count + constant;
}

struct Plan {
  int levels;
  int A[MAX_LEVELS + 1], Bc[MAX_LEVELS + 1];   // image size entering level l (A[levels] x Bc[levels] = residual)
  long long off_img[MAX_LEVELS + 1];           // image of level l (level 0 = the YUV planes)
  long long off_L[MAX_LEVELS], off_H[MAX_LEVELS];          // row-pass outputs
  long long off_LH[MAX_LEVELS], off_HL[MAX_LEVELS], off_HH[MAX_LEVELS];   // band gradients
  long long off_tmp;                            // one image-sized scratch for the backward pass
  long long off_loss;
  long long total_floats;
};

bool make_plan(int B, int H, int W, int levels, Plan* pl) {
  if (levels < 1 || levels > MAX_LEVELS || B < 1 || H < 1 || W < 1) return false;
  int mx = 0;
  while ((1 << mx) < (H < W ? H : W)) ++mx;      // ceil(log2(min side)), wavelet.get_max_num_levels
  if (levels > mx) return false;
  const long long P = 3LL * B;
  long long off = 0;
  auto take = [&](long long n) { const long long o = off; off += (n + 3) & ~3LL; return o; };
  pl->levels = levels;
  pl->A[0] = H; pl->Bc[0] = W;
  pl->off_img[0] = take(P * H * W);
  for (int l = 0; l < levels; ++l) {
    const int A = pl->A[l], Bc = pl->Bc[l];
    pl->off_L[l] = take(P * n_lo(A) * Bc);
    pl->off_H[l] = take(P * n_hi(A) * Bc);
    pl->off_LH[l] = take(P * n_lo(A) * n_hi(Bc));
    pl->off_HL[l] = take(P * n_hi(A) * n_lo(Bc));
    pl->off_HH[l] = take(P * n_hi(A) * n_hi(Bc));
    pl->A[l + 1] = n_lo(A); pl->Bc[l + 1] = n_lo(Bc);
    pl->off_img[l + 1] = take(P * n_lo(A) * n_lo(Bc));
  }
  pl->off_tmp = take(P * H * W);
  pl->off_loss = take(B);
  pl->total_floats = off;
  return true;
}

inline unsigned blocks(long long n) { return (unsigned)((n + BT - 1) / BT); }

}  // namespace
}  // namespace nlt

using namespace nlt;

extern "C" {

int64_t nlt_barron_loss_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t levels) {
  Plan pl;
  if (!make_plan(B, H, W, levels, &pl)) return -1;
  return (int64_t)(pl.total_floats * sizeof(float));
}

int nlt_barron_loss(const float* pred, const float* gt, const float* alpha, int32_t B, int32_t H, int32_t W,
                    int32_t levels, float scale, float log_z, float loss_scale, float* loss, float* d_pred,
                    void* workspace, void* stream) {
  Plan pl;
  NLT_CHECK_ARG(make_plan(B, H, W, levels, &pl), "barron loss: bad shape %dx%dx%d or levels %d", B, H, W, levels);
  NLT_CHECK_ARG(pred != nullptr && gt != nullptr && loss != nullptr && workspace != nullptr, "null pointer");
  NLT_CHECK_ARG(scale > 0.f, "scale must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const int P = 3 * B;
  const long long hw = (long long)H * W;
  const float inv_scale = 1.f / scale;
  const float inv_count = 1.f / (float)(hw * 3);                 // mean over H x W x 3 (nlt/losses.py:113-117)
  const float gscale = loss_scale * inv_count;                   // d(sum_b loss_b * loss_scale) / d(coefficient) factor
  float* loss_acc = ws + pl.off_loss;
  cudaMemsetAsync(loss_acc, 0, sizeof(float) * B, st);

  barron_prep_kernel<<<blocks((long long)B * hw), BT, 0, st>>>(pred, gt, alpha, B, hw, ws + pl.off_img[0]);
  NLT_CUDA_LAUNCH_CHECK("barron_prep_kernel");
  for (int l = 0; l < levels; ++l) {
    const int A = pl.A[l], Bc = pl.Bc[l];
    barron_rows_kernel<<<blocks((long long)P * n_lo(A) * Bc), BT, 0, st>>>(ws + pl.off_img[l], P, A, Bc,
                                                                          ws + pl.off_L[l], ws + pl.off_H[l]);
    NLT_CUDA_LAUNCH_CHECK("barron_rows_kernel");
    // low rows: LL (kept) + LH band;  high rows: HL + HH bands
    barron_cols_kernel<<<blocks((long long)P * n_lo(A) * n_lo(Bc)), BT, 0, st>>>(
        ws + pl.off_L[l], P, n_lo(A), Bc, ws + pl.off_img[l + 1], ws + pl.off_LH[l], 1, inv_scale, gscale, loss_acc);
    NLT_CUDA_LAUNCH_CHECK("barron_cols_kernel");
    if (n_hi(A) > 0) {
      barron_cols_kernel<<<blocks((long long)P * n_hi(A) * n_lo(Bc)), BT, 0, st>>>(
          ws + pl.off_H[l], P, n_hi(A), Bc, ws + pl.off_HL[l], ws + pl.off_HH[l], 0, inv_scale, gscale, loss_acc);
      NLT_CUDA_LAUNCH_CHECK("barron_cols_kernel");
    }
  }
  const long long rper = (long long)pl.A[levels] * pl.Bc[levels];
  barron_resid_kernel<<<blocks((long long)P * rper), BT, 0, st>>>(ws + pl.off_img[levels], P, rper, inv_scale, gscale,
                                                                 loss_acc);
  NLT_CUDA_LAUNCH_CHECK("barron_resid_kernel");
  barron_loss_kernel<<<(B + 127) / 128, 128, 0, st>>>(loss_acc, B, inv_count, logf(scale) + log_z, loss);
  NLT_CUDA_LAUNCH_CHECK("barron_loss_kernel");
  if (d_pred == nullptr) return NLT_OK;

  // ---- backward: off_img[l + 1] holds d(image l + 1); rebuild d(image l) level by level ----
  for (int l = levels - 1; l >= 0; --l) {
    const int A = pl.A[l], Bc = pl.Bc[l];
    // d(low rows) = colsT(dLL, dLH) ; d(high rows) = colsT(dHL, dHH)   (written over the row-pass outputs)
    barron_cols_adj_kernel<<<blocks((long long)P * n_lo(A) * Bc), BT, 0, st>>>(ws + pl.off_img[l + 1], ws + pl.off_LH[l], P,
                                                                               n_lo(A), Bc, ws + pl.off_L[l]);
    NLT_CUDA_LAUNCH_CHECK("barron_cols_adj_kernel");
    if (n_hi(A) > 0) {
      barron_cols_adj_kernel<<<blocks((long long)P * n_hi(A) * Bc), BT, 0, st>>>(ws + pl.off_HL[l], ws + pl.off_HH[l], P,
                                                                                 n_hi(A), Bc, ws + pl.off_H[l]);
      NLT_CUDA_LAUNCH_CHECK("barron_cols_adj_kernel");
    }
    float* dst = l == 0 ? ws + pl.off_tmp : ws + pl.off_img[l];
    barron_rows_adj_kernel<<<blocks((long long)P * A * Bc), BT, 0, st>>>(ws + pl.off_L[l], ws + pl.off_H[l], P, A, Bc, dst);
    NLT_CUDA_LAUNCH_CHECK("barron_rows_adj_kernel");
  }
  barron_finish_kernel<<<blocks((long long)B * hw), BT, 0, st>>>(ws + pl.off_tmp, alpha, B, hw, d_pred);
  NLT_CUDA_LAUNCH_CHECK("barron_finish_kernel");
  return NLT_OK;
}

}  // extern "C"
