// 2x2 pooling and the bilinear x2 upsampling of the U-Net built with `pool = max | avg`
// (nlt/networks/elements.py:81-94 and :42-48, nlt/networks/convnet.py:50-80):
//   pool      tf.keras.layers.MaxPooling2D / AveragePooling2D(pool_size=2, strides=2, padding='same')
//   upsample  tf.keras.layers.UpSampling2D(size=2, interpolation='bilinear') = tf.image.resize to 2H x 2W
//             (half-pixel centres, no antialias): out[2i] = .25 x[i-1] + .75 x[i], out[2i+1] = .75 x[i] + .25 x[i+1],
//             the index clamped at the edges
// and their adjoints.  All four ops are HBM streams over NHWC rows: one thread owns one pixel and V channels (float4
// when C % 4 == 0 and the pointers are 16-byte aligned), a block row of threads walks one image row, so loads and
// stores are coalesced along W * C.  No atomics: the 2x2 / stride-2 windows do not overlap, so the pool adjoint writes
// each input pixel from exactly one thread, and the upsample adjoint gathers each low-resolution pixel's <= 4 x 4
// high-resolution taps.  Every result is therefore deterministic.  The bilinear sums and the average are formed in
// double and rounded once.
#include "nlt_common.cuh"

namespace nlt {

constexpr int POOL_THREADS = 256;

template <int V> struct VecT;
template <> struct VecT<1> { typedef float T; };
template <> struct VecT<4> { typedef float4 T; };

template <int V>
__device__ __forceinline__ void ldv(const float* p, float (&v)[V]) {
  if (V == 4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; if (V > 1) { v[1 % V] = q.y; v[2 % V] = q.z; v[3 % V] = q.w; }
  } else {
    v[0] = __ldg(p);
  }
}

template <int V>
__device__ __forceinline__ void stv(float* p, const float (&v)[V]) {
  if (V == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1 % V], v[2 % V], v[3 % V]);
  else *p = v[0];
}

// out = (beta != 0 ? g + beta * out_old : g) * act'(mask_y), the epilogue of every engine.contribute writer
template <int V>
__device__ __forceinline__ void epilogue_store(float* out, float (&g)[V], float beta, const float* mask_y,
                                               int mask_act) {
  if (beta != 0.f) {
    float o[V];
    if (V == 4) {
      const float4 q = *reinterpret_cast<const float4*>(out);
      o[0] = q.x; if (V > 1) { o[1 % V] = q.y; o[2 % V] = q.z; o[3 % V] = q.w; }
    } else {
      o[0] = *out;
    }
#pragma unroll
    for (int e = 0; e < V; ++e) g[e] += beta * o[e];
  }
  if (mask_y) {
    float m[V];
    ldv<V>(mask_y, m);
#pragma unroll
    for (int e = 0; e < V; ++e) g[e] *= act_bwd_from_y(m[e], mask_act);
  }
  stv<V>(out, g);
}

// ---------------------------------------------------------------------------------------------
// pool: one thread per (output pixel, V channels); rows = N * Ho output rows
// ---------------------------------------------------------------------------------------------
template <int V, bool AVG>
__global__ void __launch_bounds__(POOL_THREADS)
pool2x2_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int C, int Ho, int Wo, float* __restrict__ y) {
  const int CV = C / V;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= Wo * CV) return;
  const int ox = j / CV, c = (j - ox * CV) * V;
  const int ix = 2 * ox, nx = min(2, W - ix);
  for (int r = blockIdx.y; r < N * Ho; r += gridDim.y) {
    const int n = r / Ho, oy = r - n * Ho;
    const int iy = 2 * oy, ny = min(2, H - iy);
    const float* p = x + (((size_t)n * H + iy) * W + ix) * C + c;
    float best[V];
    double sum[V];
    ldv<V>(p, best);
#pragma unroll
    for (int e = 0; e < V; ++e) sum[e] = best[e];
    // taps in row-major order; max keeps the first maximum (strict >)
    for (int t = 1; t < 4; ++t) {
      const int dy = t >> 1, dx = t & 1;
      if (dy >= ny || dx >= nx) continue;
      float v[V];
      ldv<V>(p + ((size_t)dy * W + dx) * C, v);
#pragma unroll
      for (int e = 0; e < V; ++e) {
        if (AVG) sum[e] += (double)v[e];
        else if (v[e] > best[e]) best[e] = v[e];
      }
    }
    if (AVG) {
      const double inv = 1.0 / (double)(ny * nx);     // SAME average pool: divide by the valid taps only
#pragma unroll
      for (int e = 0; e < V; ++e) best[e] = (float)(sum[e] * inv);
    }
    stv<V>(y + (((size_t)n * Ho + oy) * Wo + ox) * C + c, best);
  }
}

// adjoint: the thread of window (oy, ox) writes the window's <= 4 input pixels (windows are disjoint).
//   max: the whole d_y goes to the FIRST maximum of the window in row-major tap order (recomputed from x), 0 elsewhere
//   avg: every valid tap receives d_y / (valid taps)
template <int V, bool AVG>
__global__ void __launch_bounds__(POOL_THREADS)
pool2x2_bwd_kernel(const float* x, const float* __restrict__ d_y, int N, int H, int W, int C, int Ho, int Wo,
                   float beta, const float* mask_y, int mask_act, float* d_x) {
  const int CV = C / V;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= Wo * CV) return;
  const int ox = j / CV, c = (j - ox * CV) * V;
  const int ix = 2 * ox, nx = min(2, W - ix);
  for (int r = blockIdx.y; r < N * Ho; r += gridDim.y) {
    const int n = r / Ho, oy = r - n * Ho;
    const int iy = 2 * oy, ny = min(2, H - iy);
    const size_t p0 = (((size_t)n * H + iy) * W + ix) * C + c;
    float g[V];
    ldv<V>(d_y + (((size_t)n * Ho + oy) * Wo + ox) * C + c, g);
    int arg[V];
    if (AVG) {
      const float inv = 1.f / (float)(ny * nx);
#pragma unroll
      for (int e = 0; e < V; ++e) g[e] *= inv;
    } else {
      float best[V];
      ldv<V>(x + p0, best);
#pragma unroll
      for (int e = 0; e < V; ++e) arg[e] = 0;
      for (int t = 1; t < 4; ++t) {
        const int dy = t >> 1, dx = t & 1;
        if (dy >= ny || dx >= nx) continue;
        float v[V];
        ldv<V>(x + p0 + ((size_t)dy * W + dx) * C, v);
#pragma unroll
        for (int e = 0; e < V; ++e)
          if (v[e] > best[e]) { best[e] = v[e]; arg[e] = t; }
      }
    }
    for (int t = 0; t < 4; ++t) {
      const int dy = t >> 1, dx = t & 1;
      if (dy >= ny || dx >= nx) continue;
      const size_t p = p0 + ((size_t)dy * W + dx) * C;
      float v[V];
#pragma unroll
      for (int e = 0; e < V; ++e) v[e] = (AVG || arg[e] == t) ? g[e] : 0.f;
      epilogue_store<V>(d_x + p, v, beta, mask_y ? mask_y + p : nullptr, mask_act);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// bilinear x2: one thread per (low-resolution pixel, V channels); rows = N * H input rows
// ---------------------------------------------------------------------------------------------
// forward: the thread of input pixel (i, j) writes the output quad (2i..2i+1, 2j..2j+1) from the clamped 3 x 3
// neighbourhood: per row h_l = .25 x[j-1] + .75 x[j], h_r = .75 x[j] + .25 x[j+1], then the same along the column
template <int V>
__global__ void __launch_bounds__(POOL_THREADS)
upsample2x_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int C, float* __restrict__ y) {
  const int CV = C / V;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= W * CV) return;
  const int ix = j / CV, c = (j - ix * CV) * V;
  const int xl = max(ix - 1, 0), xr = min(ix + 1, W - 1);
  const int Wo = 2 * W;
  for (int r = blockIdx.y; r < N * H; r += gridDim.y) {
    const int n = r / H, iy = r - n * H;
    const int ys[3] = {max(iy - 1, 0), iy, min(iy + 1, H - 1)};
    double hl[3][V], hr[3][V];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float* row = x + ((size_t)n * H + ys[k]) * W * C + c;
      float a[V], b[V], d[V];
      ldv<V>(row + (size_t)xl * C, a);
      ldv<V>(row + (size_t)ix * C, b);
      ldv<V>(row + (size_t)xr * C, d);
#pragma unroll
      for (int e = 0; e < V; ++e) {
        hl[k][e] = 0.25 * (double)a[e] + 0.75 * (double)b[e];
        hr[k][e] = 0.75 * (double)b[e] + 0.25 * (double)d[e];
      }
    }
    float o[4][V];
#pragma unroll
    for (int e = 0; e < V; ++e) {
      o[0][e] = (float)(0.25 * hl[0][e] + 0.75 * hl[1][e]);
      o[1][e] = (float)(0.25 * hr[0][e] + 0.75 * hr[1][e]);
      o[2][e] = (float)(0.75 * hl[1][e] + 0.25 * hl[2][e]);
      o[3][e] = (float)(0.75 * hr[1][e] + 0.25 * hr[2][e]);
    }
    float* out = y + (((size_t)n * 2 * H + 2 * iy) * Wo + 2 * ix) * C + c;
    stv<V>(out, o[0]);
    stv<V>(out + C, o[1]);
    stv<V>(out + (size_t)Wo * C, o[2]);
    stv<V>(out + (size_t)Wo * C + C, o[3]);
  }
}

// weight of high-resolution tap 2i - 1 + t (t = 0..3) in the adjoint of low-resolution pixel i of n: the two taps the
// pixel feeds with .75, the two neighbours' taps with .25, and a clamped edge tap (out[0] = x[0], out[2n-1] = x[n-1])
// adds the .25 its missing neighbour would have taken
__device__ __forceinline__ double adj_weight(int i, int n, int t) {
  if (t == 0) return i > 0 ? 0.25 : 0.0;
  if (t == 1) return i == 0 ? 1.0 : 0.75;
  if (t == 2) return i == n - 1 ? 1.0 : 0.75;
  return i < n - 1 ? 0.25 : 0.0;
}

template <int V>
__global__ void __launch_bounds__(POOL_THREADS)
upsample2x_bwd_kernel(const float* __restrict__ d_y, int N, int H, int W, int C, float beta, const float* mask_y,
                      int mask_act, float* d_x) {
  const int CV = C / V;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= W * CV) return;
  const int ix = j / CV, c = (j - ix * CV) * V;
  const int Wo = 2 * W;
  double wx[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) wx[t] = adj_weight(ix, W, t);
  for (int r = blockIdx.y; r < N * H; r += gridDim.y) {
    const int n = r / H, iy = r - n * H;
    double acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.0;
#pragma unroll
    for (int ty = 0; ty < 4; ++ty) {
      const double wy = adj_weight(iy, H, ty);
      if (wy == 0.0) continue;
      const float* row = d_y + ((size_t)n * 2 * H + (2 * iy - 1 + ty)) * Wo * C + c;
      double h[V];
#pragma unroll
      for (int e = 0; e < V; ++e) h[e] = 0.0;
#pragma unroll
      for (int tx = 0; tx < 4; ++tx) {
        if (wx[tx] == 0.0) continue;
        float v[V];
        ldv<V>(row + (size_t)(2 * ix - 1 + tx) * C, v);
#pragma unroll
        for (int e = 0; e < V; ++e) h[e] += wx[tx] * (double)v[e];
      }
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] += wy * h[e];
    }
    float g[V];
#pragma unroll
    for (int e = 0; e < V; ++e) g[e] = (float)acc[e];
    const size_t p = (((size_t)n * H + iy) * W + ix) * C + c;
    epilogue_store<V>(d_x + p, g, beta, mask_y ? mask_y + p : nullptr, mask_act);
  }
}

static inline dim3 row_grid(int cols, int rows) {
  return dim3((unsigned)((cols + POOL_THREADS - 1) / POOL_THREADS), (unsigned)(rows < 65535 ? rows : 65535));
}

static inline bool vec4(int C, const void* a, const void* b, const void* c = nullptr, const void* d = nullptr) {
  return C % 4 == 0 && aligned16(a) && aligned16(b) && (c == nullptr || aligned16(c)) && (d == nullptr || aligned16(d));
}

}  // namespace nlt

using namespace nlt;

extern "C" {

int nlt_pool2x2_fwd(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, int kind, float* y, void* stream) {
  NLT_CHECK_ARG(x && y && N > 0 && H > 0 && W > 0 && C > 0, "pool2x2_fwd: bad argument");
  NLT_CHECK_ARG(kind == NLT_POOL_MAX || kind == NLT_POOL_AVG, "pool2x2_fwd: bad pool kind %d", kind);
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  NLT_CHECK_ARG((long long)Wo * C < (1ll << 31) && (long long)N * Ho < (1ll << 31), "pool2x2_fwd: too large");
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = vec4(C, x, y);
  const dim3 grid = row_grid(Wo * (v4 ? C / 4 : C), N * Ho);
  if (v4) {
    if (kind == NLT_POOL_AVG) pool2x2_fwd_kernel<4, true><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, Ho, Wo, y);
    else pool2x2_fwd_kernel<4, false><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, Ho, Wo, y);
  } else {
    if (kind == NLT_POOL_AVG) pool2x2_fwd_kernel<1, true><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, Ho, Wo, y);
    else pool2x2_fwd_kernel<1, false><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, Ho, Wo, y);
  }
  NLT_CUDA_LAUNCH_CHECK("pool2x2_fwd_kernel");
  return NLT_OK;
}

int nlt_pool2x2_bwd(const float* x, const float* d_y, int32_t N, int32_t H, int32_t W, int32_t C, int kind, float beta,
                    const float* mask_y, int mask_act, float* d_x, void* stream) {
  NLT_CHECK_ARG(x && d_y && d_x && N > 0 && H > 0 && W > 0 && C > 0, "pool2x2_bwd: bad argument");
  NLT_CHECK_ARG(kind == NLT_POOL_MAX || kind == NLT_POOL_AVG, "pool2x2_bwd: bad pool kind %d", kind);
  NLT_CHECK_ARG(mask_act >= 0 && mask_act <= 3, "bad activation code");
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  NLT_CHECK_ARG((long long)Wo * C < (1ll << 31) && (long long)N * Ho < (1ll << 31), "pool2x2_bwd: too large");
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = vec4(C, x, d_y, d_x, mask_y);
  const dim3 grid = row_grid(Wo * (v4 ? C / 4 : C), N * Ho);
  if (v4) {
    if (kind == NLT_POOL_AVG)
      pool2x2_bwd_kernel<4, true><<<grid, POOL_THREADS, 0, st>>>(x, d_y, N, H, W, C, Ho, Wo, beta, mask_y, mask_act, d_x);
    else
      pool2x2_bwd_kernel<4, false><<<grid, POOL_THREADS, 0, st>>>(x, d_y, N, H, W, C, Ho, Wo, beta, mask_y, mask_act, d_x);
  } else {
    if (kind == NLT_POOL_AVG)
      pool2x2_bwd_kernel<1, true><<<grid, POOL_THREADS, 0, st>>>(x, d_y, N, H, W, C, Ho, Wo, beta, mask_y, mask_act, d_x);
    else
      pool2x2_bwd_kernel<1, false><<<grid, POOL_THREADS, 0, st>>>(x, d_y, N, H, W, C, Ho, Wo, beta, mask_y, mask_act, d_x);
  }
  NLT_CUDA_LAUNCH_CHECK("pool2x2_bwd_kernel");
  return NLT_OK;
}

int nlt_upsample2x_bilinear_fwd(const float* x, int32_t N, int32_t H, int32_t W, int32_t C, float* y, void* stream) {
  NLT_CHECK_ARG(x && y && N > 0 && H > 0 && W > 0 && C > 0, "upsample2x_bilinear_fwd: bad argument");
  NLT_CHECK_ARG((long long)W * C < (1ll << 30) && (long long)N * H < (1ll << 30), "upsample2x_bilinear_fwd: too large");
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = vec4(C, x, y);
  const dim3 grid = row_grid(W * (v4 ? C / 4 : C), N * H);
  if (v4) upsample2x_fwd_kernel<4><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, y);
  else upsample2x_fwd_kernel<1><<<grid, POOL_THREADS, 0, st>>>(x, N, H, W, C, y);
  NLT_CUDA_LAUNCH_CHECK("upsample2x_fwd_kernel");
  return NLT_OK;
}

int nlt_upsample2x_bilinear_bwd(const float* d_y, int32_t N, int32_t H, int32_t W, int32_t C, float beta,
                                const float* mask_y, int mask_act, float* d_x, void* stream) {
  NLT_CHECK_ARG(d_y && d_x && N > 0 && H > 0 && W > 0 && C > 0, "upsample2x_bilinear_bwd: bad argument");
  NLT_CHECK_ARG(mask_act >= 0 && mask_act <= 3, "bad activation code");
  NLT_CHECK_ARG((long long)W * C < (1ll << 30) && (long long)N * H < (1ll << 30), "upsample2x_bilinear_bwd: too large");
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = vec4(C, d_y, d_x, mask_y);
  const dim3 grid = row_grid(W * (v4 ? C / 4 : C), N * H);
  if (v4) upsample2x_bwd_kernel<4><<<grid, POOL_THREADS, 0, st>>>(d_y, N, H, W, C, beta, mask_y, mask_act, d_x);
  else upsample2x_bwd_kernel<1><<<grid, POOL_THREADS, 0, st>>>(d_y, N, H, W, C, beta, mask_y, mask_act, d_x);
  NLT_CUDA_LAUNCH_CHECK("upsample2x_bwd_kernel");
  return NLT_OK;
}

}  // extern "C"
