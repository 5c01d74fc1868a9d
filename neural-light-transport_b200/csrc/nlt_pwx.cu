// Wide pointwise (1x1, stride 1) convolution into 16 channels over a virtual channel concat of 17..128 inputs:
// the level-0 layer of the 64-channel query stack (BASELINE.json "1024^2 x 64ch": base 3 + cvis 60 + lvis 1 -> 16,
// nlt/models/nlt.py:95 + nlt/networks/convnet.py:44) -- forward and weight gradient.
//
// Both are streams of [pixels x K] rows against a tiny [K x 16] matrix (AI ~ 6 FLOP/B), so the design goal is:
// every input byte crosses HBM once, arrives in shared memory by cp.async (16-byte pieces for float4-able
// sources, 4-byte pieces for the 3- and 1-channel ones -- no register staging, two tiles in flight), and the math
// runs as float2 FMA pairs over (even, odd) channels with constant-bank weights so that the CUDA-core issue rate
// stays below the HBM time per tile:
//
//   tile = 256 consecutive pixels (1x1 conv: each source's tile is one contiguous run of bytes)
//   smem row of a pixel = [float4-able sources ...][scalar sources ...][zero pad], stride KROW = K4*4 + 4 floats
//   (an odd number of 16-byte chunks: thread-per-pixel LDS.128 over consecutive rows is bank-conflict free)
//
//   forward : thread = pixel, 16 outputs as 16 float2 accumulators over (even, odd) channel pairs; the weight
//             pairs (W[c][n], W[c+1][n]) sit in constant memory (see pwx_cw)
//   wgrad   : warp = pixel, lane = (channel quad group cg, output quad ng); dz is staged duplicated
//             (d, d) so that x pairs (c, c+1) times a broadcast pair accumulate dW[c..c+1][n] in one FMA pair;
//             one fp32 partial per CTA goes to the workspace in the k-group layout of WgradK, the fixed-order
//             reduce kernel of nlt_gconv.cu finishes (deterministic).
#include <type_traits>
#include "nlt_common.cuh"

namespace nlt {

// Tile = 128 pixels per CTA of 128 threads, ONE shared-memory stage per CTA (45-51 KB): four to five CTAs share an SM and
// cover each other's copy latency (one 8-warp CTA per SM with double-buffered 256-pixel tiles could not hide the
// load latency in front of the FMA chains).
constexpr int PWX_T = 128;          // pixels per tile
constexpr int PWX_THREADS = 128;
constexpr int PWX_WARPS = PWX_THREADS / 32;
constexpr int PWX_CTAS_PER_SM = 4;
constexpr int PWX_N = 16;           // output channels
constexpr int PWX_KMAX = 128;

struct PwxSeg {
  const float* ptr;
  int C;         // channels
  int off;       // first smem column
  int vec;       // 1: 16-byte pieces
  FastDiv div;   // division of the float4 index by C/4 (vec) or of the element index by C (scalar)
};

struct PwxParams {
  PwxSeg seg[NLT_MAX_SEG];
  int nseg;
  int K, K4;           // channels, float4 groups per smem row (incl. zero padding up to a multiple of 8 groups for wgrad)
  int krow;            // smem row stride in floats
  int kpad0;           // first zero-padded smem column (== K4 * 4 when there is none)
  int ct, lw;          // depth-to-space forward: true output channels per tap, log2(row tiles) unused otherwise
  uint32_t M;          // pixels
  uint32_t ntiles;
  int16_t col_c[PWX_KMAX];    // smem column -> concat channel (weight row), -1 pad
  int16_t col_row[PWX_KMAX];  // smem column -> workspace row of the wgrad partial (k-group layout), -1 pad
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }
__device__ __forceinline__ uint32_t pwx_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// stage the x rows of tile `t` into xs (row stride p.krow floats); rows beyond M are zero-filled by the caller once
__device__ __forceinline__ void pwx_stage_x(const PwxParams& p, uint32_t t, float* xs, const uint32_t nthr = PWX_THREADS) {
  const uint32_t pix0 = t * PWX_T;
  const uint32_t npx = min((uint32_t)PWX_T, p.M - pix0);
  const uint32_t xs_u = pwx_smem_u32(xs);
#pragma unroll 1
  for (int s = 0; s < p.nseg; ++s) {
    const PwxSeg sg = p.seg[s];
    if (sg.vec) {
      const uint32_t c4 = (uint32_t)sg.C >> 2;
      const uint32_t n4 = npx * c4;
      const float4* src = reinterpret_cast<const float4*>(sg.ptr + (size_t)pix0 * sg.C);
      for (uint32_t i = threadIdx.x; i < n4; i += nthr) {
        const uint32_t px = fdiv(i, sg.div);
        const uint32_t j = i - px * c4;
        cp_async16(xs_u + (px * p.krow + sg.off + 4 * j) * 4, src + i);
      }
    } else {
      const uint32_t n = npx * (uint32_t)sg.C;
      const float* src = sg.ptr + (size_t)pix0 * sg.C;
      for (uint32_t i = threadIdx.x; i < n; i += nthr) {
        const uint32_t px = fdiv(i, sg.div);
        const uint32_t c = i - px * (uint32_t)sg.C;
        cp_async4(xs_u + (px * p.krow + sg.off + c) * 4, src + i);
      }
    }
  }
}

// zero the rows [from, PWX_T) of an x stage
__device__ __forceinline__ void pwx_zero_rows(const PwxParams& p, float* xs, uint32_t from, const uint32_t nthr = PWX_THREADS) {
  for (uint32_t i = from * p.krow + threadIdx.x; i < (uint32_t)PWX_T * p.krow; i += nthr) xs[i] = 0.f;
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
constexpr int PWX_OROW = 20;        // floats per staged output row (16 + 4: conflict-free STS.128 per pixel)

// The [K x 16] weight matrix lives in CONSTANT memory as (even, odd) channel pairs: every lane of a warp needs the same
// weight at the same time, so it is a constant-bank operand of the FMA and costs neither an LSU slot nor a
// shared-memory wavefront (the shared-memory form needed 272 broadcast LDS.128 per pixel).
constexpr int PWX_CW_PAIRS = 64;                                   // K <= 128
__constant__ float2 pwx_cw[PWX_CW_PAIRS * 32];                     // [pair][n] = (W[c_even][n], W[c_odd][n]); n < 16 (or 32: d2s form)
__device__ float2 pwx_cw_stage[PWX_CW_PAIRS * 32];                 // written by the pack kernel, copied into pwx_cw

__global__ void pwx_pack_w_kernel(const PwxParams p, const float* __restrict__ w, long long wc, long long wn) {
  const int npair = p.K4 * 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npair * 16; i += gridDim.x * blockDim.x) {
    const int cp = i >> 4, n = i & 15;
    const int c0 = p.col_c[2 * cp], c1 = p.col_c[2 * cp + 1];
    pwx_cw_stage[i] = make_float2(c0 >= 0 ? __ldg(w + (long long)c0 * wc + (long long)n * wn) : 0.f,
                                  c1 >= 0 ? __ldg(w + (long long)c1 * wc + (long long)n * wn) : 0.f);
  }
}

// K4 x NO FMA-pair block of one thread: x row from shared memory, weights [pair][NOUT] from the constant bank at the
// COMPILE-TIME column offset H * NO (a thread-derived offset, even a warp-uniform one, turns the constant-bank operands
// into per-thread loads)
template <int K4, int NOUT, int NO, int H>
__device__ __forceinline__ void pwx_row_mac(const float4* __restrict__ xrow, float2 (&acc)[NO]) {
#pragma unroll
  for (int n = 0; n < NO; ++n) acc[n] = make_float2(0.f, 0.f);
#pragma unroll
  for (int q = 0; q < K4; ++q) {
    const float4 xv = xrow[q];
    const float2 xa = make_float2(xv.x, xv.y), xb = make_float2(xv.z, xv.w);
#pragma unroll
    for (int n = 0; n < NO; ++n) {
      acc[n] = ffma2(xa, pwx_cw[(2 * q) * NOUT + H * NO + n], acc[n]);
      acc[n] = ffma2(xb, pwx_cw[(2 * q + 1) * NOUT + H * NO + n], acc[n]);
    }
  }
}

template <int NO>
__device__ __forceinline__ void pwx_row_out(const float2 (&acc)[NO], const float* __restrict__ bias, const int act,
                                            float* __restrict__ dst) {
#pragma unroll
  for (int j = 0; j < NO / 4; ++j) {
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = 4 * j + e;
      o[e] = act_fwd(acc[n].x + acc[n].y + (bias ? __ldg(bias + n) : 0.f), act);
    }
    reinterpret_cast<float4*>(dst)[j] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// NS threads per pixel, each owning 16 / NS outputs (warp-uniform split: the constant-bank weights stay uniform
// operands); the output stage aliases the x stage, so that the CTA needs 35 KB at K = 64 and 4 CTAs x 8 warps fit.
template <int K4, int NS>
__global__ void __launch_bounds__(PWX_THREADS * NS, NS == 1 ? (K4 <= 16 ? 6 : (K4 <= 24 ? 4 : 3)) : (K4 <= 16 ? 4 : 3))
pwx_fwd_kernel(const PwxParams p, const float* __restrict__ bias, const int act, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  constexpr int KROW = K4 * 4 + 4;
  constexpr int THR = PWX_THREADS * NS, NO = 16 / NS;
  float* xs = smem;
  float* so = smem;                                            // [PWX_T][PWX_OROW], aliases xs (KROW >= PWX_OROW)
  const int tid = threadIdx.x;
  const int px_t = tid % PWX_T, half = tid / PWX_T;

  pwx_zero_rows(p, xs, 0, THR);
  __syncthreads();

  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    pwx_stage_x(p, t, xs, THR);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();                                           // tile t has landed for every thread

    const float4* xrow = reinterpret_cast<const float4*>(xs + px_t * KROW);
    float2 acc[NO];
    if (NS == 1 || half == 0) pwx_row_mac<K4, 16, NO, 0>(xrow, acc);                      // warp-uniform branch
    else pwx_row_mac<K4, 16, NO, NS - 1>(xrow, acc);
    __syncthreads();                                           // every row of xs has been read
    pwx_row_out<NO>(acc, bias ? bias + half * NO : nullptr, act, so + px_t * PWX_OROW + half * NO);
    __syncthreads();                                           // outputs staged
    // coalesced 16-byte stores: the tile's outputs are one contiguous run of PWX_T*16 floats
    const uint32_t pix0 = t * PWX_T;
    const uint32_t npx = min((uint32_t)PWX_T, p.M - pix0);
    float4* dst = reinterpret_cast<float4*>(out + (size_t)pix0 * 16);
#pragma unroll
    for (int i = 0; i < 4 / NS; ++i) {
      const uint32_t qi = tid + i * THR;                       // float4 index inside the tile
      const uint32_t px = qi >> 2, j = qi & 3;
      if (px < npx) dst[qi] = *reinterpret_cast<const float4*>(so + px * PWX_OROW + 4 * j);
    }
    __syncthreads();                                           // so is xs: the next tile's copies wait for these reads
    // the staged outputs overlay the first PWX_T * PWX_OROW floats of the x stage, zero-pad columns included: re-zero
    // those (rows beyond M of a partial tile may hold anything: their results are never stored)
    const int npad = K4 * 4 - p.kpad0;
    if (npad > 0) {
      constexpr int DIRTY = (PWX_T * PWX_OROW + KROW - 1) / KROW;
      for (int i = tid; i < DIRTY * npad; i += THR) xs[(i / npad) * KROW + p.kpad0 + i % npad] = 0.f;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// weight gradient
// ---------------------------------------------------------------------------------------------
template <int NG>                  // float4 channel groups per lane (K4 <= 8*NG)
__global__ void __launch_bounds__(PWX_THREADS, PWX_CTAS_PER_SM)
pwx_wgrad_kernel(const PwxParams p, const float* __restrict__ G, float* __restrict__ ws, const int kd_pad,
                 const int bias_row, const int ld, const int coff, const int gmode, const int Win, const int gsub) {
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;
  float* gs = xs + PWX_T * p.krow;                             // [PWX_T][32]: dz duplicated (d, d)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cg = lane & 7, ng = lane >> 3;

  pwx_zero_rows(p, xs, 0);
  __syncthreads();

  float2 acc[NG][2][4];
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int g = 0; g < NG; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[g][h][n] = make_float2(0.f, 0.f);

  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    if (p.M - t * PWX_T < (uint32_t)PWX_T) pwx_zero_rows(p, xs, p.M - t * PWX_T);
    pwx_stage_x(p, t, xs);
    cp_async_commit();
    {   // dz of the tile: PWX_T*16 floats = 512 float4, 4 per thread, stored duplicated (d, d)
      const uint32_t pix0 = t * PWX_T;
      const uint32_t nq = min((uint32_t)PWX_T, p.M - pix0) * 4;
      const float4* src = reinterpret_cast<const float4*>(G + (size_t)pix0 * 16);
      // up-convs (gmode 1 / 2): the tile is 128 pixels of input row r; its 16 gradient columns are
      //   gmode 1 (4 output channels): the pixel's whole 2x2 block, float4 (dy, dx) at G4[(2r + dy) * 2W + 2x + dx]
      //   gmode 2 (8 output channels), pass gsub = dy: the 16 contiguous floats of pixels (2x, 2x + 1) of row 2r + dy
      uint32_t r = 0, x0 = 0;
      if (gmode != 0) { r = pix0 / (uint32_t)Win; x0 = pix0 - r * (uint32_t)Win; }
      if (gmode == 2) src = reinterpret_cast<const float4*>(G + ((size_t)(2 * r + gsub) * (2 * (size_t)Win) + 2 * x0) * 8);
      const float4* g4 = reinterpret_cast<const float4*>(G);
      float4 r4[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t qi = tid + i * PWX_THREADS;
        if (gmode == 1) {
          const uint32_t px = qi >> 2, dy = (qi >> 1) & 1, dx = qi & 1;
          r4[i] = __ldg(g4 + (size_t)(2 * r + dy) * (2 * (size_t)Win) + 2 * (x0 + px) + dx);
        } else {
          r4[i] = qi < nq ? __ldg(src + qi) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t qi = tid + i * PWX_THREADS;             // pixel = qi / 4, output quad = qi % 4
        float4* d = reinterpret_cast<float4*>(gs + (qi >> 2) * 32 + (qi & 3) * 8);
        d[0] = make_float4(r4[i].x, r4[i].x, r4[i].y, r4[i].y);
        d[1] = make_float4(r4[i].z, r4[i].z, r4[i].w, r4[i].w);
      }
    }
    cp_async_wait<0>();
    __syncthreads();                                           // x and dz of tile t are visible

#pragma unroll 2
    for (int i = 0; i < PWX_T / PWX_WARPS; ++i) {
      const int px = warp + PWX_WARPS * i;
      const float4* xr = reinterpret_cast<const float4*>(xs + px * p.krow);
      const float4* gq = reinterpret_cast<const float4*>(gs + px * 32 + ng * 8);
      const float4 g0 = gq[0], g1 = gq[1];                     // (d0,d0,d1,d1), (d2,d2,d3,d3)
      const float2 gd[4] = {make_float2(g0.x, g0.y), make_float2(g0.z, g0.w), make_float2(g1.x, g1.y),
                            make_float2(g1.z, g1.w)};
      bs[0] += g0.x; bs[1] += g0.z; bs[2] += g1.x; bs[3] += g1.z;
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const float4 xv = xr[cg + 8 * g];
        const float2 xa = make_float2(xv.x, xv.y), xb = make_float2(xv.z, xv.w);
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          acc[g][0][n] = ffma2(xa, gd[n], acc[g][0][n]);
          acc[g][1][n] = ffma2(xb, gd[n], acc[g][1][n]);
        }
      }
    }
    __syncthreads();                                           // everyone is done with xs / gs of tile t
  }

  // ---- cross-warp reduction in fixed order, one partial per CTA ----
  float* red = smem;                                           // [warps][8*NG*4 columns][16]
  const int ncol = 8 * NG * 4;
#pragma unroll
  for (int g = 0; g < NG; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int col = (cg + 8 * g) * 4 + 2 * h;
      float* r0 = red + ((size_t)warp * ncol + col) * 16 + ng * 4;
      *reinterpret_cast<float4*>(r0) = make_float4(acc[g][h][0].x, acc[g][h][1].x, acc[g][h][2].x, acc[g][h][3].x);
      *reinterpret_cast<float4*>(r0 + 16) = make_float4(acc[g][h][0].y, acc[g][h][1].y, acc[g][h][2].y, acc[g][h][3].y);
    }
  float* redb = red + (size_t)PWX_WARPS * ncol * 16;           // [warps][16] bias partials
  if (cg == 0) *reinterpret_cast<float4*>(redb + warp * 16 + ng * 4) = make_float4(bs[0], bs[1], bs[2], bs[3]);
  __syncthreads();
  float* dst = ws + (size_t)blockIdx.x * kd_pad * ld + coff;
  for (int i = tid; i < ncol * 16; i += PWX_THREADS) {
    const int col = i >> 4, n = i & 15;
    float s = 0.f;
#pragma unroll
    for (int wv = 0; wv < PWX_WARPS; ++wv) s += red[((size_t)wv * ncol + col) * 16 + n];
    const int row = col < PWX_KMAX ? p.col_row[col] : -1;
    if (row >= 0) dst[(size_t)row * ld + n] = s;
  }
  if (tid < 16) {
    float s = 0.f;
#pragma unroll
    for (int wv = 0; wv < PWX_WARPS; ++wv) s += redb[wv * 16 + tid];
    dst[(size_t)bias_row * ld + tid] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static bool pwx_shape_ok(const GConvK& k) {
  if (k.d2s || k.M == 0 || k.Cout != PWX_N || k.cout_true != PWX_N) return false;
  if (k.ay.nu != 1 || k.ax.nu != 1 || k.ay.it != 1 || k.ax.it != 1 || k.ay.i0 != 0 || k.ax.i0 != 0) return false;
  if (k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0) return false;
  if (k.Hin != k.Hout || k.Win != k.Wout || k.ay.nt != k.Hout || k.ax.nt != k.Wout) return false;
  int K = 0;
  for (int s = 0; s < k.nseg; ++s) {
    if (k.seg[s].sub != nullptr || k.seg[s].bcast) return false;
    K += k.seg[s].C;
  }
  return K > 16 && K <= PWX_KMAX - 8 && k.M >= 4 * PWX_T;
}

static bool pwx_build(const GConvK& k, bool for_wgrad, PwxParams* p, int* kd_pad, int* bias_row, int* GS_out,
                      bool k4_even = false) {
  memset(p, 0, sizeof(*p));
  for (int i = 0; i < PWX_KMAX; ++i) { p->col_c[i] = -1; p->col_row[i] = -1; }
  int gbase[NLT_MAX_SEG], GS = 0;
  for (int s = 0; s < k.nseg; ++s) { gbase[s] = GS; GS += (k.seg[s].C + 3) / 4; }
  int off = 0, K = 0;
  p->nseg = k.nseg;
  // float4-able sources first (their rows start on 16-byte columns), scalar ones behind
  for (int pass = 0; pass < 2; ++pass)
    for (int s = 0; s < k.nseg; ++s) {
      const Seg& sg = k.seg[s];
      if ((sg.vec ? 0 : 1) != pass) continue;
      PwxSeg& d = p->seg[s];
      d.ptr = sg.ptr; d.C = sg.C; d.off = off; d.vec = sg.vec;
      d.div = make_fastdiv(sg.vec ? (uint32_t)sg.C / 4 : (uint32_t)sg.C);
      for (int c = 0; c < sg.C; ++c) {
        if (off + c >= PWX_KMAX) return false;
        p->col_c[off + c] = (int16_t)(sg.coff + c);
        p->col_row[off + c] = (int16_t)((gbase[s] + c / 4) * 4 + (c & 3));
      }
      off += sg.C;
      K += sg.C;
    }
  p->K = K;
  int K4 = (off + 3) / 4;
  // wgrad: lanes cover 8 groups per step; forward: instantiated for 8, 16, 24, 32; depth-to-space forward
  // (k4_even): any even count (an even K4 keeps the LDS.128 row stride K4*4 + 4 conflict-free)
  K4 = k4_even ? (K4 + 1) / 2 * 2 : (K4 + 7) / 8 * 8;
  p->kpad0 = off;
  (void)for_wgrad;
  if (K4 * 4 > PWX_KMAX) return false;
  p->K4 = K4;
  p->krow = K4 * 4 + 4;
  p->M = k.M;
  p->ntiles = (k.M + PWX_T - 1) / PWX_T;
  if (kd_pad) *kd_pad = (GS + 1) * 4;
  if (bias_row) *bias_row = GS * 4;
  if (GS_out) *GS_out = GS;
  return true;
}

static size_t pwx_fwd_smem(const PwxParams& p) {       // the output stage aliases the x stage (krow >= PWX_OROW)
  return (size_t)PWX_T * (p.krow > PWX_OROW ? p.krow : PWX_OROW) * sizeof(float);
}
static size_t pwx_wgrad_smem(const PwxParams& p) {
  const size_t stage = ((size_t)PWX_T * p.krow + (size_t)PWX_T * 32) * sizeof(float);
  const size_t red = ((size_t)PWX_WARPS * p.K4 * 4 * 16 + PWX_WARPS * 16) * sizeof(float);
  return stage > red ? stage : red;
}
constexpr size_t PWX_SMEM_MAX = 56 * 1024;      // four CTAs per SM
constexpr size_t PWX_WGRAD_SMEM_MAX = 72 * 1024; // three CTAs per SM (K = 65 .. 96: the level-11 up-conv)

bool pwx_fwd_applicable(const GConvK& k, float beta, const float* mask_y, const float* out) {
  if (!pwx_shape_ok(k) || beta != 0.f || mask_y != nullptr || !aligned16(out)) return false;
  PwxParams p;
  return pwx_build(k, false, &p, nullptr, nullptr, nullptr) && pwx_fwd_smem(p) <= PWX_SMEM_MAX;
}

template <int K4, int NS>
static int pwx_fwd_launch(const PwxParams& p, const float* bias, int act, float* out, size_t smem, cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pwx_fwd_kernel<K4, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PWX_SMEM_MAX);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const unsigned per_sm = NS == 1 ? (K4 <= 16 ? 6u : (K4 <= 24 ? 4u : 3u)) : (K4 <= 16 ? 4u : 3u);
  const unsigned grid = p.ntiles < (unsigned)sm_count() * per_sm ? p.ntiles : (unsigned)sm_count() * per_sm;
  pwx_fwd_kernel<K4, NS><<<grid, PWX_THREADS * NS, smem, st>>>(p, bias, act, out);
  NLT_CUDA_LAUNCH_CHECK("pwx_fwd_kernel");
  return NLT_OK;
}

// NOTE: the constant-memory weight table is one per device: launches of this forward on DIFFERENT streams of the
// same device must not overlap (the model issues it from its main stream only).
int launch_pwx_fwd(const GConvK& k, const float* bias, int act, float* out, cudaStream_t st) {
  PwxParams p;
  if (!pwx_build(k, false, &p, nullptr, nullptr, nullptr)) return set_err(NLT_ERR_INVALID, "pwx_fwd not applicable");
  const size_t smem = pwx_fwd_smem(p);
  pwx_pack_w_kernel<<<4, 256, 0, st>>>(p, k.w, k.wc, k.wn);
  NLT_CUDA_LAUNCH_CHECK("pwx_pack_w_kernel");
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, pwx_cw_stage);
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbolAsync(pwx_cw, stage, (size_t)p.K4 * 2 * 16 * sizeof(float2), 0, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "pwx weight table: %s", cudaGetErrorString(e));
  const int ns = opt(Opt::PWX_NS);     // threads per pixel (default 1; 2 = the output split)
#define PWX_GO(K4_) do { if (ns == 1) return pwx_fwd_launch<K4_, 1>(p, bias, act, out, smem, st); \
                         return pwx_fwd_launch<K4_, 2>(p, bias, act, out, smem, st); } while (0)
  switch (p.K4) {
    case 8: PWX_GO(8);
    case 16: PWX_GO(16);
    case 24: PWX_GO(24);
    default: PWX_GO(32);
  }
#undef PWX_GO
}

// ---------------------------------------------------------------------------------------------
// forward of a 2x2 / stride-2 transposed convolution into 4 or 8 channels (levels 11-12 of the decoder,
// nlt/networks/convnet.py:67-76): a pointwise [K] -> [4 taps x CT] product per INPUT pixel whose four CT-channel
// groups land on the 2x2 output block of that pixel ("depth-to-space").  Same staging and constant-bank weights as
// pwx_fwd_kernel, NOUT = 4 * CT columns; a tile is 128 consecutive pixels of one input row, so that each of its two
// output rows is one contiguous run of 128 * 2 * CT floats.
// ---------------------------------------------------------------------------------------------
__global__ void pwx_pack_w_d2s_kernel(const PwxParams p, const float* __restrict__ w, long long wt, long long wc,
                                      long long wn, int nout) {
  const int npair = p.K4 * 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npair * nout; i += gridDim.x * blockDim.x) {
    const int cp = i / nout, n = i - cp * nout;
    const int tap = n / p.ct, nn = n - tap * p.ct;
    const int c0 = p.col_c[2 * cp], c1 = p.col_c[2 * cp + 1];
    const float* wb = w + (long long)tap * wt + (long long)nn * wn;
    pwx_cw_stage[i] = make_float2(c0 >= 0 ? __ldg(wb + (long long)c0 * wc) : 0.f, c1 >= 0 ? __ldg(wb + (long long)c1 * wc) : 0.f);
  }
}

template <int K4, int NOUT>
__global__ void __launch_bounds__(PWX_THREADS, NOUT == 16 ? 4 : 3)
pwx_d2s_fwd_kernel(const PwxParams p, const float* __restrict__ bias, const int act, float* __restrict__ out,
                   const int Win) {
  extern __shared__ __align__(16) float smem[];
  constexpr int KROW = K4 * 4 + 4;
  constexpr int OROW = NOUT + 4;
  constexpr int CT = NOUT / 4;
  float* xs = smem;
  float* so = smem;                                            // aliases xs: written after every thread has consumed its row
  const int tid = threadIdx.x;
  pwx_zero_rows(p, xs, 0);
  __syncthreads();

  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    pwx_stage_x(p, t, xs);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    float2 acc[NOUT];
#pragma unroll
    for (int n = 0; n < NOUT; ++n) acc[n] = make_float2(0.f, 0.f);
    const float4* xrow = reinterpret_cast<const float4*>(xs + tid * KROW);
#pragma unroll
    for (int q = 0; q < K4; ++q) {
      const float4 xv = xrow[q];
      const float2 xa = make_float2(xv.x, xv.y), xb = make_float2(xv.z, xv.w);
#pragma unroll
      for (int n = 0; n < NOUT; ++n) {
        acc[n] = ffma2(xa, pwx_cw[(2 * q) * NOUT + n], acc[n]);
        acc[n] = ffma2(xb, pwx_cw[(2 * q + 1) * NOUT + n], acc[n]);
      }
    }
    __syncthreads();                                           // every row of xs has been read
    float4* srow = reinterpret_cast<float4*>(so + tid * OROW);
#pragma unroll
    for (int j = 0; j < NOUT / 4; ++j) {
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = 4 * j + e;
        o[e] = act_fwd(acc[n].x + acc[n].y + (bias ? __ldg(bias + (n % CT)) : 0.f), act);
      }
      srow[j] = make_float4(o[0], o[1], o[2], o[3]);
    }
    __syncthreads();
    // tile = pixels [x0, x0 + 128) of input row r = n * Hin + y; output rows 2r and 2r + 1 (Hout = 2 Hin), columns from 2 x0
    const uint32_t pix0 = t * PWX_T;
    const uint32_t r = pix0 / (uint32_t)Win, x0 = pix0 - r * (uint32_t)Win;
    constexpr int Q = 2 * CT / 4;                              // float4 per input pixel per output row
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      float4* dst = reinterpret_cast<float4*>(out + ((size_t)(2 * r + dy) * (2 * (size_t)Win) + 2 * x0) * CT);
#pragma unroll
      for (int i = 0; i < Q; ++i) {
        const uint32_t qi = tid + i * PWX_THREADS;
        const uint32_t px = qi / Q, j = qi % Q;
        dst[qi] = *reinterpret_cast<const float4*>(so + px * OROW + dy * 2 * CT + 4 * j);
      }
    }
    __syncthreads();                                           // so is xs: the next tile's copies must wait for these reads
    if (p.kpad0 < K4 * 4)
      for (int c = p.kpad0; c < K4 * 4; ++c) xs[tid * KROW + c] = 0.f;      // the zero pad held outputs
  }
}

static size_t pwx_d2s_smem(const PwxParams& p, int nout) {
  const int row = p.krow > nout + 4 ? p.krow : nout + 4;
  return (size_t)PWX_T * row * sizeof(float);
}

static int pwx_d2s_k4(int k4) {          // instantiated widths
  const int opts[] = {6, 10, 12, 16, 20, 24, 28};
  for (int o : opts) if (k4 <= o) return o;
  return 0;
}

static bool pwx_d2s_build(const GConvK& k, PwxParams* p) {
  if (!pwx_build(k, false, p, nullptr, nullptr, nullptr, /*k4_even=*/true)) return false;
  const int k4 = pwx_d2s_k4(p->K4);
  if (k4 == 0) return false;
  p->K4 = k4;
  p->krow = k4 * 4 + 4;
  p->ct = k.cout_true;
  return true;
}

bool pwx_d2s_fwd_applicable(const GConvK& k, float beta, const float* mask_y, const float* out) {
  if (!k.d2s || k.d2s_s != 2 || k.M == 0 || beta != 0.f || mask_y != nullptr || !aligned16(out)) return false;
  if ((k.cout_true != 4 && k.cout_true != 8) || k.Cout != 4 * k.cout_true) return false;
  if (k.ax.nt != k.Win || k.ay.nt != k.Hin || k.Hout != 2 * k.Hin || k.Wout != 2 * k.Win || k.Win % PWX_T != 0) return false;
  int K = 0;
  for (int s = 0; s < k.nseg; ++s) {
    if (k.seg[s].sub != nullptr || k.seg[s].bcast || !k.seg[s].vec) return false;
    K += k.seg[s].C;
  }
  if (K < k.Cout || K > 112) return false;
  PwxParams p;
  return pwx_d2s_build(k, &p) && pwx_d2s_smem(p, k.Cout) <= PWX_SMEM_MAX;
}

template <int K4, int NOUT>
static int pwx_d2s_launch(const PwxParams& p, const float* bias, int act, float* out, int Win, size_t smem, cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pwx_d2s_fwd_kernel<K4, NOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PWX_SMEM_MAX);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const unsigned per_sm = NOUT == 16 ? 4u : 3u;
  const unsigned grid = p.ntiles < (unsigned)sm_count() * per_sm ? p.ntiles : (unsigned)sm_count() * per_sm;
  pwx_d2s_fwd_kernel<K4, NOUT><<<grid, PWX_THREADS, smem, st>>>(p, bias, act, out, Win);
  NLT_CUDA_LAUNCH_CHECK("pwx_d2s_fwd_kernel");
  return NLT_OK;
}

template <int NOUT>
static int pwx_d2s_dispatch(const PwxParams& p, const float* bias, int act, float* out, int Win, size_t smem, cudaStream_t st) {
  switch (p.K4) {
    case 6: return pwx_d2s_launch<6, NOUT>(p, bias, act, out, Win, smem, st);
    case 10: return pwx_d2s_launch<10, NOUT>(p, bias, act, out, Win, smem, st);
    case 12: return pwx_d2s_launch<12, NOUT>(p, bias, act, out, Win, smem, st);
    case 16: return pwx_d2s_launch<16, NOUT>(p, bias, act, out, Win, smem, st);
    case 20: return pwx_d2s_launch<20, NOUT>(p, bias, act, out, Win, smem, st);
    case 24: return pwx_d2s_launch<24, NOUT>(p, bias, act, out, Win, smem, st);
    default: return pwx_d2s_launch<28, NOUT>(p, bias, act, out, Win, smem, st);
  }
}

// main-stream only (shares pwx_cw with the forward above)
int launch_pwx_d2s_fwd(const GConvK& k, const float* bias, int act, float* out, cudaStream_t st) {
  PwxParams p;
  if (!pwx_d2s_build(k, &p)) return set_err(NLT_ERR_INVALID, "pwx_d2s_fwd not applicable");
  const size_t smem = pwx_d2s_smem(p, k.Cout);
  pwx_pack_w_d2s_kernel<<<4, 256, 0, st>>>(p, k.w, k.wt, k.wc, k.wn, k.Cout);
  NLT_CUDA_LAUNCH_CHECK("pwx_pack_w_d2s_kernel");
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, pwx_cw_stage);
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbolAsync(pwx_cw, stage, (size_t)p.K4 * 2 * k.Cout * sizeof(float2), 0, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "pwx weight table: %s", cudaGetErrorString(e));
  if (k.Cout == 16) return pwx_d2s_dispatch<16>(p, bias, act, out, k.Win, smem, st);
  return pwx_d2s_dispatch<32>(p, bias, act, out, k.Win, smem, st);
}

// ---------------------------------------------------------------------------------------------
// forward of the 2x2 / stride-2 convolutions of levels 1-2 (nlt/networks/convnet.py:50-59): 16- or 32-channel sources
// into 16 or 32 channels, K = 4 * sum C = 64 or 128.  Per output pixel this is the pointwise product above with the
// pixel's K-vector gathered from its 2x2 input patch: a tile is TP output pixels of one output row, whose input is, per
// source and patch row, ONE contiguous run of TP * 2 * C floats; cp.async scatters it into the padded per-pixel rows
// (columns in (source, dy, dx, c) order).  No padding case: H_in = 2 H_out exactly.
// ---------------------------------------------------------------------------------------------
struct PfParams {
  const float* seg_ptr[NLT_MAX_SEG];
  int seg_C[NLT_MAX_SEG], seg_col[NLT_MAX_SEG], seg_coff[NLT_MAX_SEG], seg_l[NLT_MAX_SEG];   // l = log2(C / 2)
  int nseg, K;
  int Hin, Win, Wout;
  int tiles_per_row;
  uint32_t ntiles;
  int s1;                        // 1: stride-1 2x2 stencil (one 16-channel source): input pixel = output pixel + tap offset
  int iuy, i0y, iux, i0x;        // tap offsets of the stride-1 form: iy = y + uy * iuy + i0y
  int Hout;
};

__global__ void pf_pack_w_kernel(const PfParams p, const float* __restrict__ w, long long wt, long long wc, long long wn,
                                 int nout, int4 tapmap) {        // weight tap = (d0y + dsy * dy) * 2 + d0x + dsx * dx
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (p.K / 2) * nout; i += gridDim.x * blockDim.x) {
    const int cp = i / nout, n = i - cp * nout;
    float v[2];
    for (int h = 0; h < 2; ++h) {
      const int col = 2 * cp + h;
      int s = 0;
      while (s + 1 < p.nseg && col >= p.seg_col[s + 1]) ++s;
      const int r = col - p.seg_col[s], C = p.seg_C[s];
      const int pt = r / C, c = r - pt * C;                    // patch position dy * 2 + dx
      const int tap = (tapmap.x + tapmap.y * (pt >> 1)) * 2 + tapmap.z + tapmap.w * (pt & 1);
      v[h] = __ldg(w + (long long)tap * wt + (long long)(p.seg_coff[s] + c) * wc + (long long)n * wn);
    }
    pwx_cw_stage[i] = make_float2(v[0], v[1]);
  }
}

// NS threads share a pixel, each owning NOUT / NS outputs (the split is warp-uniform, so the constant-bank weights stay
// uniform operands): twice the resident warps for the same tile, at the price of every x row being read NS times from
// shared memory.
template <int K4, int NOUT, int TP, int NS>
struct PfCfg {
  static constexpr int THR = TP * NS;
  static constexpr int NO = NOUT / NS;                         // outputs per thread
  static constexpr int ROW = K4 * 4 + 4 > NOUT + 4 ? K4 * 4 + 4 : NOUT + 4;
  static constexpr size_t SMEM = (size_t)TP * ROW * sizeof(float);
  static constexpr int MB_S = (int)((220u * 1024u) / (SMEM + 1024));
  static constexpr int MB_T = (NO <= 8 ? 1024 : (NO <= 16 ? 768 : 512)) / THR;
  static constexpr int MB = MB_S < MB_T ? (MB_S < 1 ? 1 : MB_S) : (MB_T < 1 ? 1 : MB_T);
};

template <int K4, int NOUT, int TP, int NS>
__global__ void __launch_bounds__(TP * NS, (PfCfg<K4, NOUT, TP, NS>::MB))
pf_fwd_kernel(const PfParams p, const float* __restrict__ bias, const int act, float* __restrict__ out,
              const float beta, const float* __restrict__ mask_y, const int mask_act) {
  extern __shared__ __align__(16) float smem[];
  constexpr int KROW = K4 * 4 + 4;
  constexpr int OROW = NOUT + 4;
  float* xs = smem;
  float* so = smem;                                            // aliases xs
  constexpr int THR = TP * NS, NO = NOUT / NS;
  const int tid = threadIdx.x;
  const int px_t = tid % TP, half = tid / TP;                  // warp-uniform split index
  const uint32_t xs_u = pwx_smem_u32(xs);

  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    const uint32_t orow = t / (uint32_t)p.tiles_per_row;       // n * Hout + y; input rows 2 * orow + dy (Hin = 2 Hout)
    const uint32_t x0 = (t - orow * (uint32_t)p.tiles_per_row) * TP;
    if (p.s1) {
      // stride-1 stencil: every input pixel of the two tap rows lands in the K-rows of the (up to) two output pixels
      // that see it; rows / columns outside the image (SAME padding) are stored as zeros
      const int C = p.seg_C[0], c4 = C >> 2, l = p.seg_l[0] - 1;         // l = log2(C / 4)
      const uint32_t n = orow / (uint32_t)p.Hout, y = orow - n * (uint32_t)p.Hout;
#pragma unroll
      for (int uy = 0; uy < 2; ++uy) {
        const int iy = (int)y + uy * p.iuy + p.i0y;
        const bool rowok = (unsigned)iy < (unsigned)p.Hin;
        const float4* src = reinterpret_cast<const float4*>(p.seg_ptr[0] + ((size_t)n * p.Hin + (rowok ? iy : 0)) * p.Win * C);
#pragma unroll
        for (int ux = 0; ux < 2; ++ux) {
          const int xoff = (int)x0 + ux * p.iux + p.i0x;
          const uint32_t col = (uint32_t)(uy * 2 + ux) * C;
          for (int i = tid; i < TP * c4; i += THR) {
            const uint32_t px = (uint32_t)i >> l, j = (uint32_t)i & ((uint32_t)c4 - 1u);
            const int ix = xoff + (int)px;
            const uint32_t dst = px * KROW + col + 4 * j;
            if (rowok && (unsigned)ix < (unsigned)p.Win) cp_async16(xs_u + dst * 4, src + (size_t)ix * c4 + j);
            else *reinterpret_cast<float4*>(xs + dst) = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
    } else {
#pragma unroll
      for (int s = 0; s < NLT_MAX_SEG; ++s) {
        if (s >= p.nseg) break;
        const int C = p.seg_C[s], l = p.seg_l[s];
        const int n4 = TP << l;                                  // float4 per patch row of the tile: TP * 2C / 4
  #pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
          const float4* src = reinterpret_cast<const float4*>(p.seg_ptr[s] + ((size_t)(2 * orow + dy) * p.Win + 2 * x0) * C);
          const uint32_t col = p.seg_col[s] + dy * 2 * C;
          for (int i = tid; i < n4; i += THR) {
            const uint32_t px = (uint32_t)i >> l, j = (uint32_t)i & ((1u << l) - 1u);
            cp_async16(xs_u + (px * KROW + col + 4 * j) * 4, src + i);
          }
        }
      }
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    const float4* xrow = reinterpret_cast<const float4*>(xs + px_t * KROW);
    float2 acc[NO];
    if (NS == 1 || half == 0) pwx_row_mac<K4, NOUT, NO, 0>(xrow, acc);                    // warp-uniform branch
    else pwx_row_mac<K4, NOUT, NO, NS - 1>(xrow, acc);
    __syncthreads();                                           // every row of xs has been read
    pwx_row_out<NO>(acc, bias ? bias + half * NO : nullptr, act, so + px_t * OROW + half * NO);
    __syncthreads();
    const size_t o4 = ((size_t)orow * p.Wout + x0) * (NOUT / 4);
    float4* dst = reinterpret_cast<float4*>(out) + o4;
    constexpr int Q = NOUT / 4;
    constexpr int QT = Q / NS;                                 // float4 per thread: TP * Q over THR threads
    // input-gradient use: + beta * (what the buffer holds), * activation derivative of the source (from its output y)
    constexpr int CH = QT < 4 ? QT : 4;                        // float4 in flight per thread
#pragma unroll
    for (int i0 = 0; i0 < QT; i0 += CH) {
      float4 oldv[CH], yv[CH];
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const uint32_t qi = tid + (i0 + i) * THR;
        if (beta != 0.f) oldv[i] = dst[qi];
        if (mask_y != nullptr) yv[i] = __ldg(reinterpret_cast<const float4*>(mask_y) + o4 + qi);
      }
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        const uint32_t qi = tid + (i0 + i) * THR;
        float4 v = *reinterpret_cast<const float4*>(so + (qi / Q) * OROW + 4 * (qi % Q));
        if (beta != 0.f) { v.x += beta * oldv[i].x; v.y += beta * oldv[i].y; v.z += beta * oldv[i].z; v.w += beta * oldv[i].w; }
        if (mask_y != nullptr) {
          v.x *= act_bwd_from_y(yv[i].x, mask_act); v.y *= act_bwd_from_y(yv[i].y, mask_act);
          v.z *= act_bwd_from_y(yv[i].z, mask_act); v.w *= act_bwd_from_y(yv[i].w, mask_act);
        }
        dst[qi] = v;
      }
    }
    __syncthreads();                                           // so is xs
  }
}

static bool pf_build(const GConvK& k, PfParams* p, int* tp) {
  memset(p, 0, sizeof(*p));
  if (k.d2s || k.M == 0) return false;
  if (k.Cout != k.cout_true || (k.Cout != 16 && k.Cout != 32)) return false;
  if (k.ay.nu != 2 || k.ax.nu != 2 || k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0) return false;
  const bool s1 = k.ay.it == 1 && k.ax.it == 1;
  if (s1) {
    // stride-1 2x2 stencil 16 -> 16 (second convs of level 1 / 10 and their adjoints), option "pf_s1"
    if (k.nseg != 1 || k.seg[0].C != 16 || k.Cout != 16) return false;
    if (k.Hin != k.Hout || k.Win != k.Wout || k.ay.nt != k.Hout || k.ax.nt != k.Wout) return false;
    if ((k.ay.iu != 1 && k.ay.iu != -1) || (k.ax.iu != 1 && k.ax.iu != -1)) return false;
  } else {
    if (k.ay.iu != 1 || k.ax.iu != 1 || k.ay.i0 != 0 || k.ax.i0 != 0 || k.ay.it != 2 || k.ax.it != 2) return false;
    if (k.ay.nt != k.Hout || k.ax.nt != k.Wout || k.Hin != 2 * k.Hout || k.Win != 2 * k.Wout) return false;
  }
  if (k.kw != 2 || (k.ay.d0 + k.ay.ds) < 0 || (k.ay.d0 + k.ay.ds) > 1 || (k.ax.d0 + k.ax.ds) < 0 || (k.ax.d0 + k.ax.ds) > 1 ||
      k.ay.d0 < 0 || k.ay.d0 > 1 || k.ax.d0 < 0 || k.ax.d0 > 1) return false;
  int col = 0;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    if (!sg.vec || sg.sub != nullptr || sg.bcast || (sg.C != 4 && sg.C != 8 && sg.C != 16 && sg.C != 32)) return false;
    p->seg_ptr[s] = sg.ptr; p->seg_C[s] = sg.C; p->seg_col[s] = col; p->seg_coff[s] = sg.coff;
    p->seg_l[s] = sg.C == 4 ? 1 : (sg.C == 8 ? 2 : (sg.C == 16 ? 3 : 4));
    col += 4 * sg.C;
  }
  // (K = 16 -- the input gradient of the up-conv into 4 channels -- is left to the wide stencil kernel)
  if (col != 32 && col != 64 && col != 128) return false;
  // K = 128 into 32 channels needs 64 float2 accumulators next to a 64-pixel tile: 6 warps per SM; the tensor path
  // takes it
  if (col == 128 && k.Cout == 32) return false;
  p->nseg = k.nseg; p->K = col;
  *tp = col <= 64 ? 128 : 64;
  if (k.Wout % *tp != 0) return false;
  p->Hin = k.Hin; p->Win = k.Win; p->Wout = k.Wout; p->Hout = k.Hout;
  p->s1 = s1 ? 1 : 0; p->iuy = k.ay.iu; p->i0y = k.ay.i0; p->iux = k.ax.iu; p->i0x = k.ax.i0;
  p->tiles_per_row = k.Wout / *tp;
  const long long nt = (long long)k.N * k.Hout * p->tiles_per_row;
  if (nt < 4 || nt > (1ll << 31)) return false;
  p->ntiles = (uint32_t)nt;
  return true;
}

bool pf_fwd_applicable(const GConvK& k, const float* mask_y, const float* out) {
  PfParams p;
  int tp = 0;
  return aligned16(out) && (mask_y == nullptr || aligned16(mask_y)) && pf_build(k, &p, &tp);
}

template <int K4, int NOUT, int TP, int NS>
static int pf_launch(const PfParams& p, const float* bias, int act, float* out, float beta, const float* mask_y,
                     int mask_act, cudaStream_t st) {
  using Cfg = PfCfg<K4, NOUT, TP, NS>;
  constexpr size_t smem = Cfg::SMEM;
  constexpr unsigned per_sm = (unsigned)Cfg::MB;
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pf_fwd_kernel<K4, NOUT, TP, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const unsigned grid = p.ntiles < (unsigned)sm_count() * per_sm ? p.ntiles : (unsigned)sm_count() * per_sm;
  pf_fwd_kernel<K4, NOUT, TP, NS><<<grid, TP * NS, smem, st>>>(p, bias, act, out, beta, mask_y, mask_act);
  NLT_CUDA_LAUNCH_CHECK("pf_fwd_kernel");
  return NLT_OK;
}

// main-stream only (shares pwx_cw)
int launch_pf_fwd(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act, float* out,
                  cudaStream_t st) {
  PfParams p;
  int tp = 0;
  if (!pf_build(k, &p, &tp)) return set_err(NLT_ERR_INVALID, "pf_fwd not applicable");
  pf_pack_w_kernel<<<4, 256, 0, st>>>(p, k.w, k.wt, k.wc, k.wn, k.Cout, make_int4(k.ay.d0, k.ay.ds, k.ax.d0, k.ax.ds));
  NLT_CUDA_LAUNCH_CHECK("pf_pack_w_kernel");
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, pwx_cw_stage);
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbolAsync(pwx_cw, stage, (size_t)(p.K / 2) * k.Cout * sizeof(float2), 0, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "pwx weight table: %s", cudaGetErrorString(e));
  const int ns = opt(Opt::PF_NS);      // threads per pixel (default 1; 2 = the output split)
#define PF_GO(K4_, N_, TP_) \
  do { if (ns == 1) return pf_launch<K4_, N_, TP_, 1>(p, bias, act, out, beta, mask_y, mask_act, st); \
       return pf_launch<K4_, N_, TP_, 2>(p, bias, act, out, beta, mask_y, mask_act, st); } while (0)
  if (p.K == 32) { if (k.Cout == 16) PF_GO(8, 16, 128); PF_GO(8, 32, 128); }
  if (p.K == 64) { if (k.Cout == 16) PF_GO(16, 16, 128); PF_GO(16, 32, 128); }
  PF_GO(32, 16, 64);
#undef PF_GO
}

// up-convs 2x2 / stride 2 into 4 or 8 channels in their depth-to-space form (levels 11-12): the same outer products with
// the 16 gradient columns gathered from the 2x2 output block (one launch for 4 channels, one per output row for 8)
static bool pwx_wgrad_d2s_ok(const GConvK& k) {
  if (!k.d2s || k.d2s_s != 2 || k.M == 0 || (k.cout_true != 4 && k.cout_true != 8) || k.Cout != 4 * k.cout_true) return false;
  if (k.ay.nt != k.Hin || k.ax.nt != k.Win || k.Hout != 2 * k.Hin || k.Wout != 2 * k.Win || k.Win % PWX_T != 0) return false;
  int K = 0;
  for (int s = 0; s < k.nseg; ++s) {
    if (k.seg[s].sub != nullptr || k.seg[s].bcast) return false;
    K += k.seg[s].C;
  }
  return K > 16 && K <= PWX_KMAX - 8 && k.M >= 4 * PWX_T;
}

bool pwx_wgrad_applicable(const GConvK& k, const float* G) {
  if (!(pwx_shape_ok(k) || pwx_wgrad_d2s_ok(k)) || (G != nullptr && !aligned16(G))) return false;
  PwxParams p;
  return pwx_build(k, true, &p, nullptr, nullptr, nullptr) && pwx_wgrad_smem(p) <= PWX_WGRAD_SMEM_MAX;
}

static size_t pwx_wgrad_smem(const PwxParams& p);
static unsigned pwx_wgrad_grid(const PwxParams& p) {
  const unsigned per_sm = pwx_wgrad_smem(p) > PWX_SMEM_MAX ? 3u : (unsigned)PWX_CTAS_PER_SM;      // resident CTAs
  return p.ntiles < (unsigned)sm_count() * per_sm ? p.ntiles : (unsigned)sm_count() * per_sm;
}

size_t pwx_wgrad_ws_floats(const GConvK& k) {
  PwxParams p;
  int kd_pad = 0;
  if (!pwx_build(k, true, &p, &kd_pad, nullptr, nullptr)) return 0;
  return (size_t)pwx_wgrad_grid(p) * kd_pad * (k.d2s ? k.Cout : 16);
}

template <int NG>
static int pwx_wgrad_launch(const PwxParams& p, const float* G, float* ws, int kd_pad, int bias_row, cudaStream_t st,
                            int ld = 16, int coff = 0, int gmode = 0, int Win = 0, int gsub = 0) {
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 64 && !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pwx_wgrad_kernel<NG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PWX_WGRAD_SMEM_MAX);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set[dev] = true;
  }
  pwx_wgrad_kernel<NG><<<pwx_wgrad_grid(p), PWX_THREADS, pwx_wgrad_smem(p), st>>>(p, G, ws, kd_pad, bias_row, ld, coff, gmode,
                                                                                  Win, gsub);
  NLT_CUDA_LAUNCH_CHECK("pwx_wgrad_kernel");
  return NLT_OK;
}

int launch_pwx_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  PwxParams p;
  int kd_pad = 0, bias_row = 0, GS = 0;
  if (!pwx_build(k, true, &p, &kd_pad, &bias_row, &GS)) return set_err(NLT_ERR_INVALID, "pwx_wgrad not applicable");
  // rows of pad channels inside a k-group are never read by the reduce stage, but the workspace may hold NaN
  // bit patterns from an earlier use: the reduce stage only touches (c + e < C) rows, so nothing to clear
  w->g = k; w->GS = GS; w->KG = GS + 1; w->ld = k.d2s ? k.Cout : 16; w->nsplit = (int)pwx_wgrad_grid(p); w->pix_per_split = 0;
  *KD_pad = (size_t)kd_pad;
  const int passes = k.d2s ? k.Cout / 16 : 1;
  const int gmode = k.d2s ? (k.cout_true == 4 ? 1 : 2) : 0;
  for (int ps = 0; ps < passes; ++ps) {
    int rc;
    switch (p.K4 / 8) {
      case 1: rc = pwx_wgrad_launch<1>(p, G, ws, kd_pad, bias_row, st, w->ld, 16 * ps, gmode, k.Win, ps); break;
      case 2: rc = pwx_wgrad_launch<2>(p, G, ws, kd_pad, bias_row, st, w->ld, 16 * ps, gmode, k.Win, ps); break;
      case 3: rc = pwx_wgrad_launch<3>(p, G, ws, kd_pad, bias_row, st, w->ld, 16 * ps, gmode, k.Win, ps); break;
      default: rc = pwx_wgrad_launch<4>(p, G, ws, kd_pad, bias_row, st, w->ld, 16 * ps, gmode, k.Win, ps); break;
    }
    if (rc != NLT_OK) return rc;
  }
  return NLT_OK;
}

// =============================================================================================
// Input gradient of a 2x2 / stride-2 convolution into 16-channel sources ("depth-to-space" pointwise op):
//   every low-resolution gradient pixel dz[p, 0..K) (K = 16 or 32) produces the 2x2 block of 16-channel input
//   gradients above it:  dx[2y+dy, 2x+dx, c] = sum_k dz[y, x, k] * W[tap(dy,dx), c, k]   (64 outputs per pixel).
// This is the level-1 / level-2 step of the backward chain and, at 1024^2, the largest single launch group of the
// whole step.  It is a pure stream (128-256 MB in, 0.5-1 GB out + the read-modify-write operands), so:
//   * thread = gradient pixel: dz row straight from global memory (a warp reads one contiguous run), the 64 outputs
//     as 32 float2 accumulators, weights from CONSTANT memory (constant-bank FMA operands, no LSU traffic);
//   * a tile of 256 pixels of one lattice row owns two contiguous 32 KB runs of the output (rows 2y and 2y+1):
//     results are staged in shared memory and leave as fully coalesced 16-byte stores, with the old gradient
//     (beta = 1), the activation mask and the fused pointwise term (the final 1x1 conv's input gradient riding along,
//     nlt_gconv_fwd_fused) applied in that same coalesced pass.
// =============================================================================================
constexpr int PWD_THREADS = 256;
constexpr int PWD_KMAX = 64, PWD_NMAX = 128;                       // gradient channels, outputs per gradient pixel
__constant__ float2 pwd_cw[PWD_KMAX * PWD_NMAX / 2];               // [k][m] = (W[k][n' = 2m], W[k][2m + 1]), n' = tap*CS + c
__device__ float2 pwd_cw_stage[PWD_KMAX * PWD_NMAX / 2];

struct PwdParams {
  const float* dz;        // [M][K]
  int K;
  uint32_t M;             // lattice pixels = N * Hin * Win
  int Win;                // power of two; a tile is TP consecutive lattice pixels: part of a row or whole rows
  int lwin, lw2;          // log2(Win), log2(2 * min(Win, TP))
  uint32_t ntiles;
  float beta;
  const float* mask_y;
  int mask_act;
  float* out;             // [N*2Hin][2Win][CS]
  // fused pointwise term: out[opix, c] += sum_k ex_x[opix, k] * ex_w[k*wk + c*wn]
  const float* ex_x;
  int ex_K;
  const float* ex_w;
  long long ex_wk, ex_wn;
  // the layer's weights W[tap][k][c] = w[tap * wt + k * wc + c * wn] and the activation split (pwd2s_mma_kernel only)
  const float* w;
  long long wt, wc, wn;
  int rawhi;
};

__global__ void pwd_pack_w_kernel(const GConvK g, int K, int CS) {
  const int half = 2 * CS;                                         // pairs per k: 4*CS / 2
  const int total = K * half;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int kk = i / half, m = i - kk * half;
    const int np = 2 * m, tap = np / CS, c = np - tap * CS;         // (n', n' + 1) share the tap: c is even
    const float* w0 = g.w + (long long)tap * g.wt + (long long)kk * g.wc + (long long)c * g.wn;
    pwd_cw_stage[i] = make_float2(__ldg(w0), __ldg(w0 + g.wn));
  }
}

// weights of the fused pointwise term, [PW_EX_KMAX][CS] (zero beyond ex_K)
template <int CS>
__device__ __forceinline__ void pwd_load_exw(const PwdParams& p, float* exw) {
  for (int i = threadIdx.x; i < PW_EX_KMAX * CS; i += PWD_THREADS)
    exw[i] = (p.ex_x != nullptr && i < p.ex_K * CS)
                 ? __ldg(p.ex_w + (long long)(i / CS) * p.ex_wk + (long long)(i % CS) * p.ex_wn) : 0.f;
}

// ---- coalesced output runs of one staged tile (so: [TP][SROW], column n' = tap * CS + c): per lattice row of the
// tile, rows 2*row and 2*row + 1 of the output, 2*wtile pixels of CS channels each.  TP*CS float4 per tile, in
// batches of 4 per thread: every read-modify-write operand of a batch is requested before the first one is used ----
template <int TP, int CS, int SROW>
__device__ __forceinline__ void pwd_store_tile(const PwdParams& p, const float* so, const float* exw, uint32_t row0,
                                               uint32_t x0) {
  constexpr int C4 = CS / 4;
  constexpr int PER_THREAD = TP * CS / PWD_THREADS;
  const int tid = threadIdx.x;
  const int Wout = 2 * p.Win;
  const int wtile = p.Win < TP ? p.Win : TP;                       // lattice pixels per row inside a tile
#pragma unroll 1
  for (int b4 = 0; b4 < PER_THREAD / 4; ++b4) {
    float4 v[4], old[4], ym[4];
    float xe[4][PW_EX_KMAX];
    uint32_t o4[4];                                                // float4 index into out (pwd2s_applicable: < 2^32)
    int jq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int f = tid + (b4 * 4 + u) * PWD_THREADS;              // float4 index inside the tile's outputs
      const int j = f % C4;                                        // C4, 2 * wtile: powers of two
      int r = f / C4;
      const int ox = r & (2 * wtile - 1);
      r >>= p.lw2;
      const int dy = r & 1, lr = r >> 1;                           // output row parity, lattice row inside the tile
      const int px = lr * wtile + (ox >> 1), dx = ox & 1;
      jq[u] = j;
      o4[u] = ((2 * (row0 + lr) + dy) * (uint32_t)Wout + 2 * x0 + ox) * C4 + j;
      if (p.beta != 0.f) old[u] = reinterpret_cast<const float4*>(p.out)[o4[u]];
      if (p.mask_y != nullptr) ym[u] = __ldg(reinterpret_cast<const float4*>(p.mask_y) + o4[u]);
      if (p.ex_x != nullptr) {
#pragma unroll
        for (int k = 0; k < PW_EX_KMAX; ++k) xe[u][k] = k < p.ex_K ? __ldg(p.ex_x + (size_t)(o4[u] / C4) * p.ex_K + k) : 0.f;
      }
      v[u] = *reinterpret_cast<const float4*>(so + px * SROW + (dy * 2 + dx) * CS + j * 4);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (p.ex_x != nullptr) {
#pragma unroll
        for (int k = 0; k < PW_EX_KMAX; ++k) {
          const float* wk = exw + k * CS + jq[u] * 4;
          v[u].x = fmaf(xe[u][k], wk[0], v[u].x); v[u].y = fmaf(xe[u][k], wk[1], v[u].y);
          v[u].z = fmaf(xe[u][k], wk[2], v[u].z); v[u].w = fmaf(xe[u][k], wk[3], v[u].w);
        }
      }
      if (p.beta != 0.f) {
        v[u].x += p.beta * old[u].x; v[u].y += p.beta * old[u].y; v[u].z += p.beta * old[u].z; v[u].w += p.beta * old[u].w;
      }
      if (p.mask_y != nullptr) {
        v[u].x *= act_bwd_from_y(ym[u].x, p.mask_act); v[u].y *= act_bwd_from_y(ym[u].y, p.mask_act);
        v[u].z *= act_bwd_from_y(ym[u].z, p.mask_act); v[u].w *= act_bwd_from_y(ym[u].w, p.mask_act);
      }
      reinterpret_cast<float4*>(p.out)[o4[u]] = v[u];
    }
  }
}

// K gradient channels, CS channels of the source whose gradient is produced (16: thread = pixel, all four taps;
// 32: two threads per pixel, thread half h owns the taps of output row 2y + h -- a warp is uniform in h, so the
// constant-memory operands stay warp-uniform).
template <int K, int CS>
__global__ void __launch_bounds__(PWD_THREADS, 2)
pwd2s_kernel(const PwdParams p) {
  constexpr int TPP = CS / 16;                                     // threads per gradient pixel
  constexpr int TP = PWD_THREADS / TPP;                            // gradient pixels per tile
  constexpr int NP = 4 * CS;                                       // outputs per gradient pixel
  constexpr int SROW = NP + 4;                                     // floats per staged pixel
  extern __shared__ __align__(16) float so[];                      // [TP][SROW]
  __shared__ float exw[PW_EX_KMAX * CS];
  const int tid = threadIdx.x;
  const int half = tid / TP, lp = tid - half * TP;                 // tap-row half, pixel inside the tile
  pwd_load_exw<CS>(p, exw);
  __syncthreads();
  auto load_x = [&](uint32_t t, float4 (&xv)[K / 4]) {
    const float4* xr = reinterpret_cast<const float4*>(p.dz + ((size_t)t * TP + lp) * K);
#pragma unroll
    for (int q = 0; q < K / 4; ++q) xv[q] = __ldg(xr + q);
  };
  constexpr bool PREFETCH = K * CS <= 512;                         // (K, CS) = (32, 32) / (64, *): the extra registers spill
  float4 xcur[PREFETCH ? K / 4 : 1];
  if (PREFETCH && blockIdx.x < p.ntiles) load_x(blockIdx.x, reinterpret_cast<float4(&)[K / 4]>(xcur));
  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    const uint32_t start = t * TP;                                 // first lattice pixel (flat: (n*Hin + y)*Win + x)
    const uint32_t row0 = start >> p.lwin, x0 = start & ((uint32_t)p.Win - 1u);
    // ---- this thread's 64 outputs ----
    float2 acc[32];
#pragma unroll
    for (int m = 0; m < 32; ++m) acc[m] = make_float2(0.f, 0.f);
    const float4* xrow = reinterpret_cast<const float4*>(p.dz + ((size_t)t * TP + lp) * K);
    // the tap-row half is warp-uniform, but only a COMPILE-TIME table offset keeps the weights constant-bank operands;
    // with `half * 32` as a run-time offset the compiler emits per-thread constant loads
    auto mac = [&](auto hc) {
      constexpr int H = decltype(hc)::value;
#pragma unroll
      for (int q = 0; q < K / 4; ++q) {
        const float4 xq = PREFETCH ? xcur[q] : __ldg(xrow + q);
        const float xs[4] = {xq.x, xq.y, xq.z, xq.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 xx = make_float2(xs[e], xs[e]);
#pragma unroll
          for (int m = 0; m < 32; ++m) acc[m] = ffma2(xx, pwd_cw[(4 * q + e) * (NP / 2) + H * 32 + m], acc[m]);
        }
      }
    };
    if (TPP == 1 || half == 0) mac(std::integral_constant<int, 0>{});
    else mac(std::integral_constant<int, TPP - 1>{});
    if (PREFETCH && t + gridDim.x < p.ntiles)                      // next tile's gradient rows: in flight during the write phase
      load_x(t + gridDim.x, reinterpret_cast<float4(&)[K / 4]>(xcur));
    __syncthreads();                                               // the previous tile's staged values have been read
    float4* srow = reinterpret_cast<float4*>(so + lp * SROW + half * 64);
#pragma unroll
    for (int j = 0; j < 16; ++j) srow[j] = make_float4(acc[2 * j].x, acc[2 * j].y, acc[2 * j + 1].x, acc[2 * j + 1].y);
    __syncthreads();
    pwd_store_tile<TP, CS, SROW>(p, so, exw, row0, x0);
  }
}

static bool pwd_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

bool pwd2s_applicable(const GConvK& k, const float* bias, int act, const float* out, const float* mask_y,
                      const PwExtra* ex) {
  if (!k.d2s || k.d2s_s != 2 || k.nseg != 1 || (k.cout_true != 16 && k.cout_true != 32) || k.Cout != 4 * k.cout_true ||
      k.M == 0) return false;
  const Seg& sg = k.seg[0];
  const int K = sg.C;
  if (!sg.vec || sg.sub != nullptr || sg.bcast) return false;
  if (k.cout_true == 16 ? (K != 16 && K != 32) : (K != 32 && K != 64)) return false;
  if (bias != nullptr || act != 0) return false;
  const int TP = PWD_THREADS / (k.cout_true / 16);
  if (k.ax.nt != k.Win || k.ay.nt != k.Hin || !pwd_pow2(k.Win) || k.M % TP != 0) return false;
  if (k.Win < TP && (TP % k.Win != 0 || ((long long)k.N * k.Hin) % (TP / k.Win) != 0)) return false;
  if (k.Hout != 2 * k.Hin || k.Wout != 2 * k.Win) return false;
  if ((unsigned long long)k.M * k.cout_true >= (1ull << 32)) return false;      // float4 index of the output: 32 bits
  if (!aligned16(out) || (mask_y != nullptr && !aligned16(mask_y))) return false;
  if (ex != nullptr && (ex->K < 1 || ex->K > PW_EX_KMAX || ex->x == nullptr || ex->w == nullptr)) return false;
  return true;
}

// tile geometry of a launch with TP lattice pixels per tile (pwd2s_applicable checked that tiles cover whole rows or
// row parts)
static void pwd_tiling(PwdParams& p, int TP) {
  p.ntiles = p.M / TP;
  p.lwin = 0;
  while ((1 << p.lwin) < p.Win) ++p.lwin;
  const int w2 = 2 * (p.Win < TP ? p.Win : TP);
  p.lw2 = 0;
  while ((1 << p.lw2) < w2) ++p.lw2;
}

static PwdParams pwd_params(const GConvK& k, float beta, const float* mask_y, int mask_act, float* out, const PwExtra* ex) {
  PwdParams p;
  memset(&p, 0, sizeof(p));
  p.dz = k.seg[0].ptr; p.K = k.seg[0].C; p.M = k.M; p.Win = k.Win;
  p.beta = beta; p.mask_y = mask_y; p.mask_act = mask_act; p.out = out;
  if (ex != nullptr) { p.ex_x = ex->x; p.ex_K = ex->K; p.ex_w = ex->w; p.ex_wk = ex->wk; p.ex_wn = ex->wn; }
  p.w = k.w; p.wt = k.wt; p.wc = k.wc; p.wn = k.wn;
  return p;
}

template <int K, int CS>
static int pwd2s_launch(const PwdParams& p0, cudaStream_t st) {
  constexpr int TP = PWD_THREADS / (CS / 16);
  PwdParams p = p0;
  pwd_tiling(p, TP);
  const size_t smem = (size_t)TP * (4 * CS + 4) * sizeof(float);
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pwd2s_kernel<K, CS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const unsigned grid = p.ntiles < 2u * sm_count() ? p.ntiles : 2u * sm_count();   // 2 CTAs per SM
  pwd2s_kernel<K, CS><<<grid, PWD_THREADS, smem, st>>>(p);
  NLT_CUDA_LAUNCH_CHECK("pwd2s_kernel");
  return NLT_OK;
}

// NOTE (as for the forward above): one constant-memory weight table per device -- launches from different streams of
// one device must not overlap; the engine issues input gradients from its main stream only.
int launch_pwd2s(const GConvK& k, float beta, const float* mask_y, int mask_act, float* out, cudaStream_t st,
                 const PwExtra* ex) {
  const int K = k.seg[0].C, CS = k.cout_true;
  pwd_pack_w_kernel<<<8, 256, 0, st>>>(k, K, CS);
  NLT_CUDA_LAUNCH_CHECK("pwd_pack_w_kernel");
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, pwd_cw_stage);
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbolAsync(pwd_cw, stage, (size_t)K * 2 * CS * sizeof(float2), 0, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "pwd weight table: %s", cudaGetErrorString(e));
  const PwdParams p = pwd_params(k, beta, mask_y, mask_act, out, ex);
  if (CS == 16) return K == 16 ? pwd2s_launch<16, 16>(p, st) : pwd2s_launch<32, 16>(p, st);
  return K == 32 ? pwd2s_launch<32, 32>(p, st) : pwd2s_launch<64, 32>(p, st);
}

// =============================================================================================
// The same depth-to-space input gradient on the tensor cores: per tile, the [TP x K] gradient rows times the
// [K x 4*CS] weights as mma.sync m16n8k8 TF32 products with the 3xTF32 split of the wgmma kernels (activation hi
// truncated or rounded per tc_rawhi, weights hi / lo rounded; three products, small terms first), so that the
// product costs a few hundred tensor instructions per tile instead of the CUDA-core FMA stream of pwd2s_kernel.
//   * weights: read once per CTA from the layer's kernel through the descriptor strides, split, and kept in shared
//     memory in mma B-fragment order (one conflict-free LDS.128 per lane gives the hi and lo pair);
//   * persistent grid of one wave; the gradient rows of the next tile are copied by cp.async into the second of two
//     stages while this tile computes and stores;
//   * tile = TP = 2048 / CS lattice pixels, 8 warps: warp = 16 pixels x 64 output columns;
//   * the accumulators are staged in shared memory and leave through pwd_store_tile, the coalesced read-modify-write
//     pass of pwd2s_kernel (beta, activation mask, fused pointwise term).
// =============================================================================================
template <int K, int CS>
struct PwmCfg {
  static constexpr int TP = 128 * 16 / CS;                        // lattice pixels per tile
  static constexpr int MT = TP / 16;                              // m16 tiles per tile: warps per column group
  static constexpr int NT = 4 * CS / 8;                           // n8 tiles of the [K x 4*CS] product
  static constexpr int NTW = 8;                                   // n8 tiles per warp
  static constexpr int XROW = K + 4;                              // staged gradient row (floats): conflict-free A loads
  static constexpr int SROW = 4 * CS + 8;                         // staged output row (floats): conflict-free float2 stores
  static constexpr size_t W_FLOATS = (size_t)K * 4 * CS * 2;
  static constexpr size_t X_FLOATS = (size_t)TP * XROW;
  static constexpr size_t SMEM = (W_FLOATS + 2 * X_FLOATS + (size_t)TP * SROW) * sizeof(float);
  static_assert(MT * (NT / NTW) * 32 == PWD_THREADS, "one warp per 16 pixels x 64 columns");
};

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], float b0, float b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}

template <int K, int CS>
__global__ void __launch_bounds__(PWD_THREADS, 2)
pwd2s_mma_kernel(const PwdParams p) {
  using C = PwmCfg<K, CS>;
  extern __shared__ __align__(16) float smem[];
  float4* wf = reinterpret_cast<float4*>(smem);                   // [K/8][NT][lane]: (hi b0, hi b1, lo b0, lo b1)
  float* xs = smem + C::W_FLOATS;                                 // 2 x [TP][XROW]
  float* so = xs + 2 * C::X_FLOATS;                               // [TP][SROW]
  __shared__ float exw[PW_EX_KMAX * CS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, tq = lane & 3;                        // mma fragment row / column group of the lane

  // B fragment of (k-step ks, n8 tile nt) for lane l: b0 = W[8ks + l%4][8nt + l/4], b1 = the same at k + 4
  for (int i = tid; i < K / 8 * C::NT * 32; i += PWD_THREADS) {
    const int l = i & 31, nt = (i >> 5) % C::NT, ks = (i >> 5) / C::NT;
    const int n = 8 * nt + (l >> 2), k = 8 * ks + (l & 3);
    const int tap = n / CS, c = n - tap * CS;
    const float* w0 = p.w + tap * p.wt + k * p.wc + c * p.wn;
    const float v0 = __ldg(w0), v1 = __ldg(w0 + 4 * p.wc);
    const float h0 = tf32_rna(v0), h1 = tf32_rna(v1);
    wf[i] = make_float4(h0, h1, tf32_rna(v0 - h0), tf32_rna(v1 - h1));
  }
  pwd_load_exw<CS>(p, exw);

  auto stage = [&](uint32_t t, int buf) {                         // gradient rows of tile t: TP * K contiguous floats
    const float4* src = reinterpret_cast<const float4*>(p.dz + (size_t)t * C::TP * K);
    const uint32_t dst = pwx_smem_u32(xs + buf * C::X_FLOATS);
#pragma unroll
    for (int i = tid; i < C::TP * K / 4; i += PWD_THREADS) {
      const int px = i / (K / 4), q = i % (K / 4);
      cp_async16(dst + (px * C::XROW + 4 * q) * 4, src + i);
    }
  };
  if (blockIdx.x < p.ntiles) stage(blockIdx.x, 0);
  cp_async_commit();
  const int mt = warp % C::MT, ng = warp / C::MT;                 // pixel rows 16 mt.., columns 64 ng..
  int buf = 0;
  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x, buf ^= 1) {
    if (t + gridDim.x < p.ntiles) stage(t + gridDim.x, buf ^ 1);  // the other stage was last read before the staging barrier
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();                                              // tile t has landed; the previous tile's outputs are stored

    float acc[C::NTW][4];
#pragma unroll
    for (int j = 0; j < C::NTW; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    const float* xa = xs + buf * C::X_FLOATS + (16 * mt + gq) * C::XROW + tq;
#pragma unroll 1
    for (int ks = 0; ks < K / 8; ++ks) {                         // (unrolled, the B fragments of all k-steps are hoisted and spill)
      uint32_t ah[4], al[4];
      tf32_split(xa[8 * ks], p.rawhi, ah[0], al[0]);
      tf32_split(xa[8 * C::XROW + 8 * ks], p.rawhi, ah[1], al[1]);
      tf32_split(xa[8 * ks + 4], p.rawhi, ah[2], al[2]);
      tf32_split(xa[8 * C::XROW + 8 * ks + 4], p.rawhi, ah[3], al[3]);
#pragma unroll
      for (int j = 0; j < C::NTW; ++j) {
        const float4 b = wf[(ks * C::NT + ng * C::NTW + j) * 32 + lane];
        mma_tf32(acc[j], al, b.x, b.y);                           // small terms first
        mma_tf32(acc[j], ah, b.z, b.w);
        mma_tf32(acc[j], ah, b.x, b.y);
      }
    }
#pragma unroll
    for (int j = 0; j < C::NTW; ++j) {
      float* r0 = so + (16 * mt + gq) * C::SROW + 8 * (ng * C::NTW + j) + 2 * tq;
      *reinterpret_cast<float2*>(r0) = make_float2(acc[j][0], acc[j][1]);
      *reinterpret_cast<float2*>(r0 + 8 * C::SROW) = make_float2(acc[j][2], acc[j][3]);
    }
    __syncthreads();                                              // outputs staged; every read of stage buf is done
    const uint32_t start = t * C::TP;
    pwd_store_tile<C::TP, CS, C::SROW>(p, so, exw, start >> p.lwin, start & ((uint32_t)p.Win - 1u));
  }
}

template <int K, int CS>
static int pwd2s_mma_launch(const PwdParams& p0, cudaStream_t st) {
  using C = PwmCfg<K, CS>;
  PwdParams p = p0;
  pwd_tiling(p, C::TP);
  int dev = 0;
  cudaGetDevice(&dev);
  static int per_sm[64] = {0};                                    // resident CTAs per SM, per device
  int& n = per_sm[dev >= 0 && dev < 64 ? dev : 0];
  if (n == 0) {
    cudaError_t e = cudaFuncSetAttribute(pwd2s_mma_kernel<K, CS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, pwd2s_mma_kernel<K, CS>, PWD_THREADS, C::SMEM);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "pwd2s_mma_kernel attributes: %s", cudaGetErrorString(e));
    if (n < 1) return set_err(NLT_ERR_CUDA, "pwd2s_mma_kernel: no CTA fits on an SM");
  }
  const unsigned wave = (unsigned)sm_count() * (unsigned)n;
  const unsigned grid = p.ntiles < wave ? p.ntiles : wave;
  pwd2s_mma_kernel<K, CS><<<grid, PWD_THREADS, C::SMEM, st>>>(p);
  NLT_CUDA_LAUNCH_CHECK("pwd2s_mma_kernel");
  return NLT_OK;
}

int launch_pwd2s_mma(const GConvK& k, float beta, const float* mask_y, int mask_act, float* out, cudaStream_t st,
                     const PwExtra* ex) {
  const int K = k.seg[0].C, CS = k.cout_true;
  PwdParams p = pwd_params(k, beta, mask_y, mask_act, out, ex);
  p.rawhi = opt(Opt::TC_RAWHI);
  if (CS == 16) return K == 16 ? pwd2s_mma_launch<16, 16>(p, st) : pwd2s_mma_launch<32, 16>(p, st);
  return K == 32 ? pwd2s_mma_launch<32, 32>(p, st) : pwd2s_mma_launch<64, 32>(p, st);
}

// =============================================================================================
// Weight gradient of the 2x2 convolutions (stride 1 or 2) of the 16- / 32-channel levels:
//   dW[tap, c, n] = sum_p x[(s*y + dy, s*x + dx), c] * dz[(y, x), n]     K = 4 * sum_seg C <= 128, N = 16 or 32.
// Same arithmetic shape as pwx_wgrad_kernel (an outer product per pixel, FMA pairs with the gradient staged duplicated),
// with the pixel's K-vector gathered from a staged input patch: a tile is 64 output pixels of one output row, its
// input is two row segments per source (s*64 (+1 halo) pixels, contiguous in memory) copied by cp.async.  warp =
// pixel, lane = (channel group, output quad); for N = 32, K = 128 two warps split the K rows of a pixel.  One fp32
// partial per CTA in the k-group layout of WgradK (row = 4 * group + e, groups in (tap, source, channel quad) order).
// =============================================================================================
constexpr int PWS_TP = 64;            // output pixels per tile
constexpr int PWS_THREADS = 128;
constexpr int PWS_WARPS = 4;
constexpr int PWS_CTAS_PER_SM = 4;

struct PwsParams {
  const float* seg_ptr[NLT_MAX_SEG];
  int seg_C[NLT_MAX_SEG];
  int seg_soff[NLT_MAX_SEG];     // float offset of the source's patch inside the x stage
  int nseg, ctot;                // sum of channels
  int s;                         // stride (1 or 2)
  int pw;                        // staged pixels per row: s * TP + (s == 1)
  int N, Hin, Win, Hout, Wout;
  int tiles_per_row;
  uint32_t ntiles;
  int xfloats;                   // floats of the x stage
  int kd_pad, bias_row;
};

template <int NQ, int NG, int KSPLIT>     // output quads (N / 4), channel groups per lane, warps sharing a pixel's K rows
__global__ void __launch_bounds__(PWS_THREADS, PWS_CTAS_PER_SM)
pws_wgrad_kernel(const PwsParams p, const float* __restrict__ G, float* __restrict__ ws) {
  constexpr int NCG = 32 / NQ;                  // channel-group lanes
  constexpr int N = NQ * 4;
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                             // per source: [2 rows][pw pixels][C]
  float* gs = xs + p.xfloats;                   // [TP][2N]: dz duplicated (d, d)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cg = lane / NQ, ng = lane % NQ;
  const int khalf = warp % KSPLIT, pwarp = warp / KSPLIT;
  constexpr int PSTEP = PWS_WARPS / KSPLIT;     // warps that walk the tile's pixels

  // this lane's channel groups: g = (khalf * NG + j) * NCG + cg over (tap, source, channel quad)
  int goff[NG], gstr[NG];
#pragma unroll
  for (int j = 0; j < NG; ++j) {
    const int g = (khalf * NG + j) * NCG + cg;
    const int gpt = p.ctot >> 2;                // groups per tap
    const int tap = g / gpt;
    int r = g - tap * gpt, sidx = 0;
    while (sidx < p.nseg - 1 && r >= (p.seg_C[sidx] >> 2)) { r -= p.seg_C[sidx] >> 2; ++sidx; }
    const int C = p.seg_C[sidx];
    const int dy = tap >> 1, dx = tap & 1;
    goff[j] = p.seg_soff[sidx] + (dy * p.pw + dx) * C + r * 4;
    gstr[j] = p.s * C;
  }

  float2 acc[NG][2][4];
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < NG; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int n = 0; n < 4; ++n) acc[j][h][n] = make_float2(0.f, 0.f);

  const uint32_t xs_u = pwx_smem_u32(xs);
  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    const uint32_t orow = t / (uint32_t)p.tiles_per_row;              // flat output row n*Hout + y
    const int x0 = (int)(t - orow * (uint32_t)p.tiles_per_row) * PWS_TP;
    const int n = (int)(orow / (uint32_t)p.Hout), y = (int)(orow - (uint32_t)n * p.Hout);
    // ---- stage the input patch: per source two row segments; out-of-image parts (SAME padding) are zeroed ----
    for (int sidx = 0; sidx < p.nseg; ++sidx) {
      const int C = p.seg_C[sidx], c4 = C >> 2;
      for (int dy = 0; dy < 2; ++dy) {
        const int iy = p.s * y + dy;
        const int ix0 = p.s * x0;
        const int npx = min(p.pw, p.Win - ix0);                       // pixels of the run that exist
        float* dst = xs + p.seg_soff[sidx] + dy * p.pw * C;
        if (iy < p.Hin) {
          const float4* src = reinterpret_cast<const float4*>(p.seg_ptr[sidx] + (((size_t)n * p.Hin + iy) * p.Win + ix0) * C);
          const int n4 = npx * c4;
          for (int i = tid; i < n4; i += PWS_THREADS) cp_async16(xs_u + (uint32_t)((dst - xs) + i * 4) * 4, src + i);
          for (int i = npx * C + tid; i < p.pw * C; i += PWS_THREADS) dst[i] = 0.f;
        } else {
          for (int i = tid; i < p.pw * C; i += PWS_THREADS) dst[i] = 0.f;
        }
      }
    }
    cp_async_commit();
    {   // dz of the tile: TP * N floats, stored duplicated (d, d)
      const float4* src = reinterpret_cast<const float4*>(G + ((size_t)orow * p.Wout + x0) * N);
      constexpr int NQT = PWS_TP * NQ;                                  // float4 of the tile
#pragma unroll
      for (int i = 0; i < (NQT + PWS_THREADS - 1) / PWS_THREADS; ++i) {
        const int qi = tid + i * PWS_THREADS;
        if (qi < NQT) {
          const float4 r = __ldg(src + qi);
          float4* d = reinterpret_cast<float4*>(gs + (qi / NQ) * (2 * N) + (qi % NQ) * 8);
          d[0] = make_float4(r.x, r.x, r.y, r.y);
          d[1] = make_float4(r.z, r.z, r.w, r.w);
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();

#pragma unroll 2
    for (int i = 0; i < PWS_TP / PSTEP; ++i) {
      const int px = pwarp + PSTEP * i;
      const float4* gq = reinterpret_cast<const float4*>(gs + px * (2 * N) + ng * 8);
      const float4 g0 = gq[0], g1 = gq[1];
      const float2 gd[4] = {make_float2(g0.x, g0.y), make_float2(g0.z, g0.w), make_float2(g1.x, g1.y),
                            make_float2(g1.z, g1.w)};
      bs[0] += g0.x; bs[1] += g0.z; bs[2] += g1.x; bs[3] += g1.z;
#pragma unroll
      for (int j = 0; j < NG; ++j) {
        const float4 xv = *reinterpret_cast<const float4*>(xs + goff[j] + px * gstr[j]);
        const float2 xa = make_float2(xv.x, xv.y), xb = make_float2(xv.z, xv.w);
#pragma unroll
        for (int nn = 0; nn < 4; ++nn) {
          acc[j][0][nn] = ffma2(xa, gd[nn], acc[j][0][nn]);
          acc[j][1][nn] = ffma2(xb, gd[nn], acc[j][1][nn]);
        }
      }
    }
    __syncthreads();                                                   // everyone is done with this tile's stages
  }

  // ---- reduce the warps of each K half in fixed order, one partial per CTA ----
  constexpr int ROWS_H = NG * NCG * 4;                                 // weight rows of one K half
  float* red = smem;                                                   // [warp][ROWS_H][N]
#pragma unroll
  for (int j = 0; j < NG; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = (j * NCG + cg) * 4 + 2 * h;                      // row inside this warp's K half
      float* r0 = red + ((size_t)warp * ROWS_H + row) * N + ng * 4;
      *reinterpret_cast<float4*>(r0) = make_float4(acc[j][h][0].x, acc[j][h][1].x, acc[j][h][2].x, acc[j][h][3].x);
      *reinterpret_cast<float4*>(r0 + N) = make_float4(acc[j][h][0].y, acc[j][h][1].y, acc[j][h][2].y, acc[j][h][3].y);
    }
  float* redb = red + (size_t)PWS_WARPS * ROWS_H * N;                  // [warp][N] bias partials (K half 0 only)
  if (cg == 0 && khalf == 0) *reinterpret_cast<float4*>(redb + pwarp * N + ng * 4) = make_float4(bs[0], bs[1], bs[2], bs[3]);
  __syncthreads();
  float* dst = ws + (size_t)blockIdx.x * p.kd_pad * N;
  for (int i = tid; i < KSPLIT * ROWS_H * N; i += PWS_THREADS) {
    const int nn = i % N, r = i / N;                                   // r = global weight row = kh * ROWS_H + row
    const int kh = r / ROWS_H, row = r - kh * ROWS_H;
    float sum = 0.f;
#pragma unroll
    for (int pwv = 0; pwv < PSTEP; ++pwv) sum += red[((size_t)(pwv * KSPLIT + kh) * ROWS_H + row) * N + nn];
    dst[(size_t)r * N + nn] = sum;
  }
  if (tid < N) {
    float sum = 0.f;
#pragma unroll
    for (int pwv = 0; pwv < PSTEP; ++pwv) sum += redb[pwv * N + tid];
    dst[(size_t)p.bias_row * N + tid] = sum;
  }
}

struct PwsPlan {
  bool ok;
  int nq, ng, ksplit;
  PwsParams p;
  size_t smem;
  unsigned grid;
};

static PwsPlan pws_plan(const GConvK& k) {
  PwsPlan pl;
  memset(&pl, 0, sizeof(pl));
  if (k.d2s || k.M == 0) return pl;
  if (k.Cout != k.cout_true || (k.Cout != 16 && k.Cout != 32)) return pl;
  if (k.ay.nu != 2 || k.ax.nu != 2 || k.ay.iu != 1 || k.ax.iu != 1 || k.ay.i0 != 0 || k.ax.i0 != 0) return pl;
  if (k.ay.it != k.ax.it || (k.ay.it != 1 && k.ay.it != 2)) return pl;
  if (k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0 || k.ay.d0 != 0 || k.ax.d0 != 0 || k.ay.ds != 1 ||
      k.ax.ds != 1 || k.kw != 2) return pl;
  if (k.ay.nt != k.Hout || k.ax.nt != k.Wout || k.Wout % PWS_TP != 0) return pl;
  PwsParams& p = pl.p;
  p.s = k.ay.it;
  if (p.s == 2 && (k.Hin != 2 * k.Hout || k.Win != 2 * k.Wout)) return pl;
  if (p.s == 1 && (k.Hin != k.Hout || k.Win != k.Wout)) return pl;
  p.pw = p.s * PWS_TP + (p.s == 1 ? 1 : 0);
  int off = 0;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    if (!sg.vec || sg.sub != nullptr || sg.bcast) return pl;
    p.seg_ptr[s] = sg.ptr; p.seg_C[s] = sg.C; p.seg_soff[s] = off;
    off += 2 * p.pw * sg.C;
    p.ctot += sg.C;
  }
  p.nseg = k.nseg;
  const int K4 = p.ctot;                       // float4 groups: 4 taps * ctot / 4
  pl.nq = k.Cout / 4;
  const int ncg = 32 / pl.nq;
  if (K4 % ncg != 0) return pl;
  int groups = K4 / ncg;                       // per lane without K split
  pl.ksplit = 1;
  if (groups > 4) { if (groups % 2 != 0) return pl; pl.ksplit = 2; groups /= 2; }
  if (groups != 2 && groups != 4) return pl;
  pl.ng = groups;
  p.N = k.N; p.Hin = k.Hin; p.Win = k.Win; p.Hout = k.Hout; p.Wout = k.Wout;
  p.tiles_per_row = k.Wout / PWS_TP;
  const long long nt = (long long)k.N * k.Hout * p.tiles_per_row;
  if (nt < 4 || nt > (1ll << 31)) return pl;
  p.ntiles = (uint32_t)nt;
  p.xfloats = (off + 3) / 4 * 4;
  p.kd_pad = (K4 + 1) * 4;
  p.bias_row = K4 * 4;
  const size_t stage = ((size_t)p.xfloats + (size_t)PWS_TP * 2 * k.Cout) * sizeof(float);
  const size_t red = ((size_t)PWS_WARPS * (pl.ng * ncg * 4) * k.Cout + PWS_WARPS * k.Cout) * sizeof(float);
  pl.smem = stage > red ? stage : red;
  if (pl.smem > 56 * 1024) return pl;
  pl.grid = p.ntiles < (unsigned)sm_count() * PWS_CTAS_PER_SM ? p.ntiles : (unsigned)sm_count() * PWS_CTAS_PER_SM;
  pl.ok = true;
  return pl;
}

bool pws_wgrad_applicable(const GConvK& k, const float* G) {
  return (G == nullptr || aligned16(G)) && pws_plan(k).ok;
}

size_t pws_wgrad_ws_floats(const GConvK& k) {
  PwsPlan pl = pws_plan(k);
  return pl.ok ? (size_t)pl.grid * pl.p.kd_pad * k.Cout : 0;
}

template <int NQ, int NG, int KS>
static int pws_launch(const PwsPlan& pl, const float* G, float* ws, cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {false};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pws_wgrad_kernel<NQ, NG, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  pws_wgrad_kernel<NQ, NG, KS><<<pl.grid, PWS_THREADS, pl.smem, st>>>(pl.p, G, ws);
  NLT_CUDA_LAUNCH_CHECK("pws_wgrad_kernel");
  return NLT_OK;
}

int launch_pws_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  PwsPlan pl = pws_plan(k);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "pws_wgrad not applicable");
  w->g = k; w->GS = pl.p.ctot / 4; w->KG = pl.p.ctot + 1; w->ld = k.Cout; w->nsplit = (int)pl.grid; w->pix_per_split = 0;
  *KD_pad = (size_t)pl.p.kd_pad;
  if (pl.nq == 4) return pl.ng == 2 ? pws_launch<4, 2, 1>(pl, G, ws, st) : pws_launch<4, 4, 1>(pl, G, ws, st);
  if (pl.ksplit == 1) return pl.ng == 2 ? pws_launch<8, 2, 1>(pl, G, ws, st) : pws_launch<8, 4, 1>(pl, G, ws, st);
  return pl.ng == 2 ? pws_launch<8, 2, 2>(pl, G, ws, st) : pws_launch<8, 4, 2>(pl, G, ws, st);
}

}  // namespace nlt
