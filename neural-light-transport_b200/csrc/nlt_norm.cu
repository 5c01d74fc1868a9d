// Normalisation layers of the conv blocks (nlt/networks/elements.py:51-66): the two kinds that keep samples
// independent and are well defined in the reference --
//   'pixel'    (elements.py:103-121)  y = x * rsqrt(mean_c(x^2) + 1e-8), no parameters
//   'instance' (elements.py:97-100: tf.contrib.layers.instance_norm(center=True, scale=True, epsilon=1e-6))
//              y = gamma * (x - mean_hw) * rsqrt(var_hw + eps) + beta per sample and channel (biased variance)
// each fused with the activation that follows it in the block (conv -> norm -> act, convnet.py:50-59, 67-76).
// They are HBM streams: NHWC rows are read with float4 loads by groups of lanes that own one pixel, reductions are
// fixed-order (deterministic).  Shipped configs use norm = None, where none of this runs.
#include "nlt_common.cuh"

namespace nlt {


static inline int norm_grid(size_t n, int block, int per_sm = 8) {
  size_t b = (n + block - 1) / block;
  const size_t cap = (size_t)sm_count() * per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// lanes per pixel: power of two <= 32 covering C/4 float4 groups as evenly as possible
static inline int lanes_per_pixel(int C) {
  int g = 1;
  while (g < 32 && g * 4 < C) g <<= 1;
  return g;
}

// ---------------------------------------------------------------------------------------------
// pixel norm
// ---------------------------------------------------------------------------------------------
template <bool BWD>
__global__ void __launch_bounds__(256)
pixelnorm_kernel(const float* __restrict__ x, const float* __restrict__ dz, float* __restrict__ out, size_t P, int C,
                 int G, int act, float eps) {
  // group of G lanes = one pixel; C % 4 == 0
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;                       // lane inside the group
  const int ppw = 32 / G;                        // pixels per warp
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int C4 = C >> 2;
  const float invC = 1.f / (float)C;
  for (size_t pw = warp0; pw * ppw < P; pw += nwarps) {
    const size_t p = pw * ppw + lane / G;
    const bool live = p < P;
    const float4* xr = reinterpret_cast<const float4*>(x + p * C);
    const float4* dr = BWD ? reinterpret_cast<const float4*>(dz + p * C) : nullptr;
    float ss = 0.f, sd = 0.f;
    if (live)
      for (int q = gl; q < C4; q += G) {
        const float4 v = __ldg(xr + q);
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        if (BWD) {
          const float4 d = __ldg(dr + q);
          sd += v.x * d.x + v.y * d.y + v.z * d.z + v.w * d.w;
        }
      }
    for (int o = G >> 1; o > 0; o >>= 1) {       // butterfly inside the group: every lane ends with the group sum
      ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (BWD) sd += __shfl_xor_sync(0xffffffffu, sd, o);
    }
    if (!live) continue;
    const float r = rsqrtf(ss * invC + eps);
    float4* orow = reinterpret_cast<float4*>(out + p * C);
    if (!BWD) {
      for (int q = gl; q < C4; q += G) {
        const float4 v = __ldg(xr + q);
        orow[q] = make_float4(act_fwd(v.x * r, act), act_fwd(v.y * r, act), act_fwd(v.z * r, act), act_fwd(v.w * r, act));
      }
    } else {
      // dx_c = r * dz_c - x_c * r^3 * (sum_j dz_j x_j) / C
      const float k = r * r * r * sd * invC;
      for (int q = gl; q < C4; q += G) {
        const float4 v = __ldg(xr + q), d = __ldg(dr + q);
        orow[q] = make_float4(r * d.x - v.x * k, r * d.y - v.y * k, r * d.z - v.z * k, r * d.w - v.w * k);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// instance norm: per-(sample, channel) sums over H*W in two fixed-order stages
// ---------------------------------------------------------------------------------------------
constexpr int IN_CHUNK = 1024;                   // pixels per partial

// Thread layout of the two partial kernels.  C <= blockDim: thread = (row, channel), rows = blockDim / C pixel rows in
// flight (loads coalesced along channels); C > blockDim: one row, every thread walks several channels.

// Statistics pass: stat[(n * nchunk + chunk) * 3C + {c, C + c, 2C + c}] = (sum (x - a), sum (x - a)^2, a) over the
// chunk's pixels, where a is the chunk's own mean as a first fp32 sweep finds it.  The second sweep re-reads the chunk
// (1024 * C floats, cache resident at the channel counts of the large levels) around that shift, so neither sum
// cancels however far a channel's mean lies from zero: E[x^2] - mean^2 on the raw values loses
// (mean / std)^2 * 2^-24 of the variance.  sum (x - a) is the part of the chunk's sum the first sweep rounded away.
__global__ void __launch_bounds__(256)
instnorm_stats_partial_kernel(const float* __restrict__ x, int HW, int C, int nchunk, float* __restrict__ stat) {
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int p0 = chunk * IN_CHUNK, p1 = min(HW, p0 + IN_CHUNK);
  const float inv_cnt = 1.f / (float)(p1 - p0);
  extern __shared__ float sm[];                  // [rows][2C] partials of the thread rows
  const int rows = (int)blockDim.x / C > 0 ? (int)blockDim.x / C : 1;
  float* out = stat + ((size_t)n * nchunk + chunk) * 3 * C;
  auto sweep = [&](int row, int c, float a, float& r, float& q) {
    r = 0.f; q = 0.f;
    for (int p = p0 + row; p < p1; p += rows) {
      const float d = __ldg(x + ((size_t)n * HW + p) * C + c) - a;
      r += d; q += d * d;
    }
  };
  if (rows > 1) {                                // one (row, channel) per thread; the rows share the shift
    const int row = threadIdx.x / C, c = threadIdx.x - row * C;
    const bool live = row < rows;
    float r, q;
    if (live) { sweep(row, c, 0.f, r, q); sm[(size_t)row * 2 * C + c] = r; }
    __syncthreads();
    float a = 0.f;
    if (live) {
      for (int k = 0; k < rows; ++k) a += sm[(size_t)k * 2 * C + c];
      a *= inv_cnt;
    }
    __syncthreads();
    if (live) {
      sweep(row, c, a, r, q);
      sm[(size_t)row * 2 * C + c] = r;
      sm[(size_t)row * 2 * C + C + c] = q;
      if (row == 0) out[2 * C + c] = a;
    }
  } else {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float r, q;
      sweep(0, c, 0.f, r, q);
      const float a = r * inv_cnt;
      sweep(0, c, a, r, q);
      sm[c] = r;
      sm[C + c] = q;
      out[2 * C + c] = a;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * C; j += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < rows; ++k) s += sm[(size_t)k * 2 * C + j];
    out[j] = s;
  }
}

// Backward pass: partial[(n * nchunk + chunk) * 2C + {c, C + c}] = (sum dz, sum dz * xhat) over the chunk's pixels
// (xhat from mean / rstd)
__global__ void __launch_bounds__(256)
instnorm_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ dz, const float* __restrict__ mean,
                            const float* __restrict__ rstd, int HW, int C, int nchunk, float* __restrict__ partial) {
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int p0 = chunk * IN_CHUNK, p1 = min(HW, p0 + IN_CHUNK);
  extern __shared__ float sm[];                  // [rows][2C] partials of the thread rows
  const int rows = (int)blockDim.x / C > 0 ? (int)blockDim.x / C : 1;
  for (int idx = threadIdx.x; idx < rows * C; idx += blockDim.x) {
    const int row = idx / C, c = idx - row * C;
    float a = 0.f, b = 0.f;
    const float m = mean[(size_t)n * C + c], rs = rstd[(size_t)n * C + c];
    for (int p = p0 + row; p < p1; p += rows) {
      const size_t i = ((size_t)n * HW + p) * C + c;
      const float d = __ldg(dz + i);
      a += d;
      b += d * (__ldg(x + i) - m) * rs;
    }
    sm[(size_t)row * 2 * C + c] = a;
    sm[(size_t)row * 2 * C + C + c] = b;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * C; j += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < rows; ++r) s += sm[(size_t)r * 2 * C + j];
    partial[((size_t)n * nchunk + chunk) * 2 * C + j] = s;
  }
}

// mean / rstd per (n, c): the chunks' (count, mean, centred second moment) merged in double, in chunk order, with
// Chan's pairwise update
__global__ void instnorm_stats_kernel(const float* __restrict__ stat, int N, int HW, int C, int nchunk, float eps,
                                      float* __restrict__ mean, float* __restrict__ rstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  double cnt = 0.0, m = 0.0, m2 = 0.0;
  for (int k = 0; k < nchunk; ++k) {
    const float* s = stat + ((size_t)n * nchunk + k) * 3 * C;
    const double nk = (double)(min(HW, (k + 1) * IN_CHUNK) - k * IN_CHUNK);
    const double r = (double)s[c], q = (double)s[C + c];
    const double mk = (double)s[2 * C + c] + r / nk;
    double m2k = q - r * r / nk;
    if (m2k < 0.0) m2k = 0.0;
    const double d = mk - m, tot = cnt + nk;
    m += d * nk / tot;
    m2 += m2k + d * d * cnt * nk / tot;
    cnt = tot;
  }
  mean[i] = (float)m;
  rstd[i] = (float)(1.0 / sqrt(m2 / HW + (double)eps));
}

// per (n, c): sums of the backward partials -> (mean dz, mean dz*xhat); and the parameter gradients
__global__ void instnorm_bwd_reduce_kernel(const float* __restrict__ partial, int N, int HW, int C, int nchunk,
                                           float* __restrict__ mdz, float* __restrict__ mdzx,
                                           float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double gsum = 0.0, bsum = 0.0;
  for (int n = 0; n < N; ++n) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < nchunk; ++k) {
      a += (double)partial[((size_t)n * nchunk + k) * 2 * C + c];
      b += (double)partial[((size_t)n * nchunk + k) * 2 * C + C + c];
    }
    mdz[(size_t)n * C + c] = (float)(a / HW);
    mdzx[(size_t)n * C + c] = (float)(b / HW);
    bsum += a;
    gsum += b;
  }
  if (dgamma) dgamma[c] = (accumulate ? dgamma[c] : 0.f) + (float)gsum;
  if (dbeta) dbeta[c] = (accumulate ? dbeta[c] : 0.f) + (float)bsum;
}

// y = act(gamma * (x - mean) * rstd + beta)            (forward)
// dx = gamma * rstd * (dz - mdz - xhat * mdzx)         (backward)
template <bool BWD>
__global__ void __launch_bounds__(256)
instnorm_apply_kernel(const float* __restrict__ x, const float* __restrict__ dz, const float* __restrict__ mean,
                      const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ mdz, const float* __restrict__ mdzx, size_t total4, int HW, int C,
                      int act, float* __restrict__ out) {
  const int C4 = C >> 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % C4);
    const size_t p = i / C4;
    const int n = (int)(p / HW);
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    const float xv[4] = {v.x, v.y, v.z, v.w};
    float dv[4] = {0.f, 0.f, 0.f, 0.f};
    if (BWD) {
      const float4 d = __ldg(reinterpret_cast<const float4*>(dz) + i);
      dv[0] = d.x; dv[1] = d.y; dv[2] = d.z; dv[3] = d.w;
    }
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = q * 4 + e;
      const size_t s = (size_t)n * C + c;
      const float xh = (xv[e] - __ldg(mean + s)) * __ldg(rstd + s);
      if (!BWD) o[e] = act_fwd(__ldg(gamma + c) * xh + __ldg(beta + c), act);
      else o[e] = __ldg(gamma + c) * __ldg(rstd + s) * (dv[e] - __ldg(mdz + s) - xh * __ldg(mdzx + s));
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace nlt

using namespace nlt;

extern "C" {

int nlt_pixelnorm_fwd(const float* x, int64_t pixels, int32_t C, int act, float* y, void* stream) {
  NLT_CHECK_ARG(x && y && pixels > 0 && C > 0 && C % 4 == 0, "pixelnorm_fwd: bad argument (C %% 4 == 0 required)");
  NLT_CHECK_ARG(act >= 0 && act <= 3, "bad activation code");
  const int G = lanes_per_pixel(C);
  const size_t warps = ((size_t)pixels + (32 / G) - 1) / (32 / G);
  pixelnorm_kernel<false><<<norm_grid(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, nullptr, y, (size_t)pixels, C, G,
                                                                                       act, 1.0e-8f);
  NLT_CUDA_LAUNCH_CHECK("pixelnorm_fwd_kernel");
  return NLT_OK;
}

int nlt_pixelnorm_bwd(const float* x, const float* dz, int64_t pixels, int32_t C, float* dx, void* stream) {
  NLT_CHECK_ARG(x && dz && dx && pixels > 0 && C > 0 && C % 4 == 0, "pixelnorm_bwd: bad argument");
  const int G = lanes_per_pixel(C);
  const size_t warps = ((size_t)pixels + (32 / G) - 1) / (32 / G);
  pixelnorm_kernel<true><<<norm_grid(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, dz, dx, (size_t)pixels, C, G, 0,
                                                                                      1.0e-8f);
  NLT_CUDA_LAUNCH_CHECK("pixelnorm_bwd_kernel");
  return NLT_OK;
}

int64_t nlt_instnorm_workspace_bytes(int32_t N, int32_t HW, int32_t C) {
  if (N <= 0 || HW <= 0 || C <= 0) return -1;
  const int64_t nchunk = (HW + IN_CHUNK - 1) / IN_CHUNK;
  // forward: (sum, second moment, shift) per chunk and channel; backward: two sums per chunk and channel + mdz, mdzx
  return ((int64_t)N * nchunk * 3 * C + 2 * (int64_t)N * C) * (int64_t)sizeof(float);
}

// threads and shared memory of the two partial kernels (one [rows][2C] table)
static int instnorm_partial_smem(int C, size_t* smem) {
  const int rows = 256 / C > 0 ? 256 / C : 1;
  *smem = (size_t)rows * 2 * C * sizeof(float);
  NLT_CHECK_ARG(*smem <= 48 * 1024, "instance norm: too many channels (%d)", C);
  return NLT_OK;
}

int nlt_instnorm_fwd(const float* x, const float* gamma, const float* beta, int32_t N, int32_t HW, int32_t C, int act,
                     float eps, float* y, float* mean, float* rstd, void* workspace, void* stream) {
  NLT_CHECK_ARG(x && gamma && beta && y && mean && rstd && workspace, "instnorm_fwd: null pointer");
  NLT_CHECK_ARG(N > 0 && HW > 0 && C > 0 && C % 4 == 0, "instnorm_fwd: bad geometry (C %% 4 == 0 required)");
  NLT_CHECK_ARG(act >= 0 && act <= 3, "bad activation code");
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = (HW + IN_CHUNK - 1) / IN_CHUNK;
  float* partial = (float*)workspace;
  size_t smem;
  int rc = instnorm_partial_smem(C, &smem);
  if (rc != NLT_OK) return rc;
  instnorm_stats_partial_kernel<<<dim3(nchunk, N), 256, smem, st>>>(x, HW, C, nchunk, partial);
  NLT_CUDA_LAUNCH_CHECK("instnorm_stats_partial_kernel");
  instnorm_stats_kernel<<<(N * C + 127) / 128, 128, 0, st>>>(partial, N, HW, C, nchunk, eps, mean, rstd);
  NLT_CUDA_LAUNCH_CHECK("instnorm_stats_kernel");
  const size_t total4 = (size_t)N * HW * C / 4;
  instnorm_apply_kernel<false><<<norm_grid(total4, 256), 256, 0, st>>>(x, nullptr, mean, rstd, gamma, beta, nullptr, nullptr,
                                                                        total4, HW, C, act, y);
  NLT_CUDA_LAUNCH_CHECK("instnorm_apply_kernel");
  return NLT_OK;
}

int nlt_instnorm_bwd(const float* x, const float* dz, const float* gamma, const float* mean, const float* rstd, int32_t N,
                     int32_t HW, int32_t C, float* dx, float* dgamma, float* dbeta, int accumulate, void* workspace,
                     void* stream) {
  NLT_CHECK_ARG(x && dz && gamma && mean && rstd && dx && workspace, "instnorm_bwd: null pointer");
  NLT_CHECK_ARG(N > 0 && HW > 0 && C > 0 && C % 4 == 0, "instnorm_bwd: bad geometry");
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = (HW + IN_CHUNK - 1) / IN_CHUNK;
  float* partial = (float*)workspace;
  float* mdz = partial + (size_t)N * nchunk * 2 * C;
  float* mdzx = mdz + (size_t)N * C;
  size_t smem;
  int rc = instnorm_partial_smem(C, &smem);
  if (rc != NLT_OK) return rc;
  instnorm_bwd_partial_kernel<<<dim3(nchunk, N), 256, smem, st>>>(x, dz, mean, rstd, HW, C, nchunk, partial);
  NLT_CUDA_LAUNCH_CHECK("instnorm_bwd_partial_kernel");
  instnorm_bwd_reduce_kernel<<<(C + 63) / 64, 64, 0, st>>>(partial, N, HW, C, nchunk, mdz, mdzx, dgamma, dbeta, accumulate);
  NLT_CUDA_LAUNCH_CHECK("instnorm_bwd_reduce_kernel");
  const size_t total4 = (size_t)N * HW * C / 4;
  instnorm_apply_kernel<true><<<norm_grid(total4, 256), 256, 0, st>>>(x, dz, mean, rstd, gamma, nullptr, mdz, mdzx, total4,
                                                                       HW, C, 0, dx);
  NLT_CUDA_LAUNCH_CHECK("instnorm_apply_kernel");
  return NLT_OK;
}

}  // extern "C"
