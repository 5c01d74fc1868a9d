// "barron" training-loss term of NLT (nlt/losses.py:90-121) fused with its gradient -- SURVEY.md 8f, row N1.
// The per-element arithmetic (nlt_barron_core.h) is checked on the CPU against the pinned oracle, the kernels by
// tests/test_gpu_barron.py and, element by element against fp64, by tests/test_gpu_barron_census.py.
//
// Planar fp32 scratch ([3B planes][rows][cols]); per level l (image A x B):
//   rows pass : L[ceil(A/2)][B], H[floor(A/2)][B]
//   cols pass : LL -> next level's image;  LH, HL, HH -> per-block loss partials + gradient stored in place of the
//               coefficient (the partials are summed per sample in a fixed order: the loss is deterministic)
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

// Per-sample loss sums without atomics.  Every loss-producing launch runs a grid of (blocks per sample) x B, so each
// block holds terms of ONE sample (blockIdx.y); it shuffle-reduces per warp, adds the warps in double and writes one
// partial to its own slot.  barron_loss_kernel then adds each sample's partials in a fixed order, in double, so the
// loss is the same bits on every call.  EVERY thread of the block must call this (no early returns before it).
__device__ __forceinline__ void block_partial(float part, double* slot) {
  __shared__ double sp[BT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float v = part;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) sp[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < BT / 32; ++w) s += sp[w];
    *slot = s;
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

// analysis along axis 1 (columns) of one row-pass output `src` [3B][R][Bc], grid (blocks per sample) x B:
//   keep_lo != 0: the low-pass output is the next level's image (stored as is); else it is a band
//   bands: coefficient -> loss contribution (one partial per block in part[b * nparts + blockIdx.x]) and, in place,
//   its gradient
__global__ void __launch_bounds__(BT)
barron_cols_kernel(const float* __restrict__ src, int R, int Bc, float* __restrict__ out_lo,
                   float* __restrict__ out_hi, int keep_lo, float inv_scale, float gscale,
                   double* __restrict__ part_out, int nparts) {
  const int nl = n_lo(Bc), nh = n_hi(Bc);
  const long long per_sample = 3LL * R * nl;
  const long long local = (long long)blockIdx.x * BT + threadIdx.x;
  float part = 0.f;
  if (local < per_sample) {
    const long long idx = (long long)blockIdx.y * per_sample + local;
    const int j = (int)(idx % nl);
    const int r = (int)((idx / nl) % R);
    const int p = (int)(idx / ((long long)nl * R));
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
  block_partial(part, part_out + (long long)blockIdx.y * nparts + blockIdx.x);
}

// coarsest residual image [3B][per_plane]: loss + gradient in place, grid (blocks per sample) x B
__global__ void __launch_bounds__(BT)
barron_resid_kernel(float* __restrict__ img, long long per_plane, float inv_scale, float gscale,
                    double* __restrict__ part_out, int nparts) {
  const long long local = (long long)blockIdx.x * BT + threadIdx.x;
  float part = 0.f;
  if (local < 3 * per_plane) {
    const long long idx = (long long)blockIdx.y * 3 * per_plane + local;
    const float w = img[idx];
    part = charbonnier(w, inv_scale);
    img[idx] = gscale * charbonnier_grad(w, inv_scale);
  }
  block_partial(part, part_out + (long long)blockIdx.y * nparts + blockIdx.x);
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

// one block per sample: that sample's partials [nparts] added in a fixed order, in double
__global__ void __launch_bounds__(BT)
barron_loss_kernel(const double* __restrict__ part, int nparts, float inv_count, float constant,
                   float* __restrict__ loss) {
  __shared__ double sh[BT];
  const double* p = part + (long long)blockIdx.x * nparts;
  double s = 0.0;
  for (int i = threadIdx.x; i < nparts; i += BT) s += p[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = BT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[blockIdx.x] = (float)(sh[0] * (double)inv_count) + constant;
}

struct Plan {
  int levels;
  int A[MAX_LEVELS + 1], Bc[MAX_LEVELS + 1];   // image size entering level l (A[levels] x Bc[levels] = residual)
  long long off_img[MAX_LEVELS + 1];           // image of level l (level 0 = the YUV planes)
  long long off_L[MAX_LEVELS], off_H[MAX_LEVELS];          // row-pass outputs
  long long off_LH[MAX_LEVELS], off_HL[MAX_LEVELS], off_HH[MAX_LEVELS];   // band gradients
  long long off_tmp;                            // one image-sized scratch for the backward pass
  // per-sample loss partials: double [B][nparts]; the blocks of each loss-producing launch own a run of slots
  int slot_L[MAX_LEVELS], slot_H[MAX_LEVELS], slot_resid, nparts;
  long long off_part;
  long long total_floats;
};

inline unsigned blocks(long long n) { return (unsigned)((n + BT - 1) / BT); }

bool make_plan(int B, int H, int W, int levels, Plan* pl) {
  // B is the grid's y extent in the loss-producing launches
  if (levels < 1 || levels > MAX_LEVELS || B < 1 || B > 65535 || H < 1 || W < 1) return false;
  int mx = 0;
  while ((1 << mx) < (H < W ? H : W)) ++mx;      // ceil(log2(min side)), wavelet.get_max_num_levels
  if (levels > mx) return false;
  const long long P = 3LL * B;
  long long off = 0;
  auto take = [&](long long n) { const long long o = off; off += (n + 3) & ~3LL; return o; };
  long long slots = 0;
  pl->levels = levels;
  pl->A[0] = H; pl->Bc[0] = W;
  pl->off_img[0] = take(P * H * W);
  for (int l = 0; l < levels; ++l) {
    const int A = pl->A[l], Bc = pl->Bc[l];
    pl->slot_L[l] = (int)slots;
    slots += blocks(3LL * n_lo(A) * n_lo(Bc));
    pl->slot_H[l] = (int)slots;
    slots += n_hi(A) > 0 ? blocks(3LL * n_hi(A) * n_lo(Bc)) : 0;
    pl->off_L[l] = take(P * n_lo(A) * Bc);
    pl->off_H[l] = take(P * n_hi(A) * Bc);
    pl->off_LH[l] = take(P * n_lo(A) * n_hi(Bc));
    pl->off_HL[l] = take(P * n_hi(A) * n_lo(Bc));
    pl->off_HH[l] = take(P * n_hi(A) * n_hi(Bc));
    pl->A[l + 1] = n_lo(A); pl->Bc[l + 1] = n_lo(Bc);
    pl->off_img[l + 1] = take(P * n_lo(A) * n_lo(Bc));
  }
  pl->slot_resid = (int)slots;
  slots += blocks(3LL * pl->A[levels] * pl->Bc[levels]);
  if (slots > (1LL << 30)) return false;
  pl->nparts = (int)slots;
  pl->off_tmp = take(P * H * W);
  pl->off_part = take(2LL * B * slots);         // doubles; take() keeps 16-byte alignment
  pl->total_floats = off;
  return true;
}

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
  double* part = (double*)(ws + pl.off_part);                    // every slot is written below: no clearing

  barron_prep_kernel<<<blocks((long long)B * hw), BT, 0, st>>>(pred, gt, alpha, B, hw, ws + pl.off_img[0]);
  NLT_CUDA_LAUNCH_CHECK("barron_prep_kernel");
  for (int l = 0; l < levels; ++l) {
    const int A = pl.A[l], Bc = pl.Bc[l];
    barron_rows_kernel<<<blocks((long long)P * n_lo(A) * Bc), BT, 0, st>>>(ws + pl.off_img[l], P, A, Bc,
                                                                          ws + pl.off_L[l], ws + pl.off_H[l]);
    NLT_CUDA_LAUNCH_CHECK("barron_rows_kernel");
    // low rows: LL (kept) + LH band;  high rows: HL + HH bands
    barron_cols_kernel<<<dim3(blocks(3LL * n_lo(A) * n_lo(Bc)), B), BT, 0, st>>>(
        ws + pl.off_L[l], n_lo(A), Bc, ws + pl.off_img[l + 1], ws + pl.off_LH[l], 1, inv_scale, gscale,
        part + pl.slot_L[l], pl.nparts);
    NLT_CUDA_LAUNCH_CHECK("barron_cols_kernel");
    if (n_hi(A) > 0) {
      barron_cols_kernel<<<dim3(blocks(3LL * n_hi(A) * n_lo(Bc)), B), BT, 0, st>>>(
          ws + pl.off_H[l], n_hi(A), Bc, ws + pl.off_HL[l], ws + pl.off_HH[l], 0, inv_scale, gscale,
          part + pl.slot_H[l], pl.nparts);
      NLT_CUDA_LAUNCH_CHECK("barron_cols_kernel");
    }
  }
  const long long rper = (long long)pl.A[levels] * pl.Bc[levels];
  barron_resid_kernel<<<dim3(blocks(3 * rper), B), BT, 0, st>>>(ws + pl.off_img[levels], rper, inv_scale, gscale,
                                                                part + pl.slot_resid, pl.nparts);
  NLT_CUDA_LAUNCH_CHECK("barron_resid_kernel");
  barron_loss_kernel<<<B, BT, 0, st>>>(part, pl.nparts, inv_count, logf(scale) + log_z, loss);
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
