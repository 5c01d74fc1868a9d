// Lean kernels for the few-channel layers at (near) full resolution: levels 11-12 of the decoder and the second
// convs of the level-1 blocks (nlt/networks/convnet.py:50-59, 67-76 at depth0 = 16: 4 -> 4 and 8 -> 8 channels at
// 1024^2 / 512^2, 16 -> 16 at 512^2).  They move 30-130 bytes per pixel for 64-1024 FMAs: pure streams, for which the
// general small-stencil kernel (nlt_small.cu: any tap set, any pixel map, runtime segment lists, 64-bit pixel decode per
// thread) spends several hundred instructions of bookkeeping per pixel.
//
// Here a CTA owns a run of consecutive pixels of ONE lattice row: the image / row decode happens once per CTA, a
// thread's addresses are `row base + x * C`, tap rows that fall outside the image are skipped for the whole CTA, all
// channel loops are compile-time, weights come from constant memory as FMA operands.
#include "nlt_common.cuh"

namespace nlt {

constexpr int TINY_THREADS = 128;
constexpr int TINY_KMAX = 4 * 16;                  // taps * input channels
__constant__ float2 tiny_cw[TINY_KMAX * 8];        // [k][m] = (W[k][2m], W[k][2m + 1]), up to 16 outputs
__device__ float2 tiny_cw_stage[TINY_KMAX * 8];

// weight of (tap index in kernel order, input channel c, output n), pairs over n
__global__ void tiny_pack_w_kernel(const GConvK g, int cin, int cout) {
  const int ntaps = g.ay.nu * g.ax.nu;
  const int half = cout / 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ntaps * cin * half; i += gridDim.x * blockDim.x) {
    const int k = i / half, m = i - k * half;
    const int tapi = k / cin, c = k - tapi * cin;
    const int uy = tapi / g.ax.nu, ux = tapi - uy * g.ax.nu;
    const int tap = (g.ay.d0 + g.ay.ds * uy) * g.kw + (g.ax.d0 + g.ax.ds * ux);
    const float* w0 = g.w + (long long)tap * g.wt + (long long)c * g.wc + (long long)(2 * m) * g.wn;
    tiny_cw_stage[i] = make_float2(__ldg(w0), __ldg(w0 + g.wn));
  }
}

struct TinyParams {
  const float* in;
  float* out;
  const float* bias;
  const float* mask_y;
  int N, H, W;               // lattice = input = output size (stride-1 maps)
  int nty, ntx;              // taps
  int iuy, i0y, iux, i0x;    // input coordinate = lattice coordinate + tap * iu + i0
  int act, mask_act;
  float beta;
  int xtiles;                // CTAs per row
};

template <int CIN, int COUT, int MINB>
__global__ void __launch_bounds__(TINY_THREADS, MINB)
tiny_stencil_kernel(const TinyParams p) {
  const int row = blockIdx.x / p.xtiles;                       // n * H + y
  const int x = (blockIdx.x - row * p.xtiles) * TINY_THREADS + threadIdx.x;
  const int n = row / p.H, y = row - n * p.H;
  float2 acc[COUT / 2];
#pragma unroll
  for (int m = 0; m < COUT / 2; ++m)
    acc[m] = p.bias ? make_float2(__ldg(p.bias + 2 * m), __ldg(p.bias + 2 * m + 1)) : make_float2(0.f, 0.f);
  constexpr int G = CIN / 4;
  // all four taps of a pixel are in flight before the first FMA (CIN <= 8), or one tap row at a time (CIN = 16)
  constexpr int ROWS_PER_BATCH = (CIN <= 8) ? 2 : 1;
#pragma unroll
  for (int b = 0; b < 2 / ROWS_PER_BATCH; ++b) {
    float4 v[ROWS_PER_BATCH][2][G];
#pragma unroll
    for (int r = 0; r < ROWS_PER_BATCH; ++r) {
      const int uy = b * ROWS_PER_BATCH + r;
      const int iy = y + uy * p.iuy + p.i0y;
      const bool rowok = uy < p.nty && (unsigned)iy < (unsigned)p.H;      // SAME padding: CTA-uniform
      const float* rbase = p.in + ((size_t)n * p.H + (rowok ? iy : 0)) * p.W * CIN;
#pragma unroll
      for (int ux = 0; ux < 2; ++ux) {
        const int ix = x + ux * p.iux + p.i0x;
        const bool in = rowok && ux < p.ntx && (unsigned)ix < (unsigned)p.W;
#pragma unroll
        for (int q = 0; q < G; ++q)
          v[r][ux][q] = in ? ld4(rbase + (size_t)ix * CIN + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS_PER_BATCH; ++r)
#pragma unroll
      for (int ux = 0; ux < 2; ++ux) {
        const int kbase = ((b * ROWS_PER_BATCH + r) * p.ntx + ux) * CIN;     // rows / taps beyond nty / ntx hold zeros
        if ((b * ROWS_PER_BATCH + r) >= p.nty || ux >= p.ntx) continue;
#pragma unroll
        for (int q = 0; q < G; ++q) {
          const float xs[4] = {v[r][ux][q].x, v[r][ux][q].y, v[r][ux][q].z, v[r][ux][q].w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 xx = make_float2(xs[e], xs[e]);
            const float2* w = tiny_cw + (kbase + 4 * q + e) * (COUT / 2);
#pragma unroll
            for (int m = 0; m < COUT / 2; ++m) acc[m] = ffma2(xx, w[m], acc[m]);
          }
        }
      }
  }
  if (x >= p.W) return;
  const size_t ob = ((size_t)row * p.W + x) * COUT;
  float4 oldv[COUT / 4], yv[COUT / 4];
#pragma unroll
  for (int q = 0; q < COUT / 4; ++q) {
    if (p.beta != 0.f) oldv[q] = *reinterpret_cast<const float4*>(p.out + ob + 4 * q);
    if (p.mask_y != nullptr) yv[q] = ld4(p.mask_y + ob + 4 * q);
  }
#pragma unroll
  for (int q = 0; q < COUT / 4; ++q) {
    float o[4] = {act_fwd(acc[2 * q].x, p.act), act_fwd(acc[2 * q].y, p.act), act_fwd(acc[2 * q + 1].x, p.act),
                  act_fwd(acc[2 * q + 1].y, p.act)};
    if (p.beta != 0.f) { o[0] += p.beta * oldv[q].x; o[1] += p.beta * oldv[q].y; o[2] += p.beta * oldv[q].z; o[3] += p.beta * oldv[q].w; }
    if (p.mask_y != nullptr) {
      o[0] *= act_bwd_from_y(yv[q].x, p.mask_act); o[1] *= act_bwd_from_y(yv[q].y, p.mask_act);
      o[2] *= act_bwd_from_y(yv[q].z, p.mask_act); o[3] *= act_bwd_from_y(yv[q].w, p.mask_act);
    }
    *reinterpret_cast<float4*>(p.out + ob + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

bool tiny_stencil_applicable(const GConvK& k, const float* out, const float* mask_y) {
  if (k.d2s || k.M == 0 || k.nseg != 1) return false;
  const Seg& sg = k.seg[0];
  if (!sg.vec || sg.sub != nullptr || sg.bcast) return false;
  if (sg.C != k.Cout || k.Cout != k.cout_true || (k.Cout != 4 && k.Cout != 8 && k.Cout != 16)) return false;
  if (k.ay.nu < 1 || k.ax.nu < 1 || k.ay.nu > 2 || k.ax.nu > 2 || k.ay.nu * k.ax.nu * sg.C > TINY_KMAX) return false;
  if (k.ay.it != 1 || k.ax.it != 1 || k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0) return false;
  if (k.Hin != k.Hout || k.Win != k.Wout || k.ay.nt != k.Hout || k.ax.nt != k.Wout) return false;
  if (k.Wout < TINY_THREADS / 2) return false;
  return aligned16(out) && (mask_y == nullptr || aligned16(mask_y));
}

// NOTE: one constant-memory weight table per device (see nlt_pwx.cu): main-stream ops only.
int launch_tiny_stencil(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                        float* out, cudaStream_t st) {
  const int C = k.Cout;
  tiny_pack_w_kernel<<<2, 256, 0, st>>>(k, C, C);
  NLT_CUDA_LAUNCH_CHECK("tiny_pack_w_kernel");
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, tiny_cw_stage);
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbolAsync(tiny_cw, stage, (size_t)k.ay.nu * k.ax.nu * C * (C / 2) * sizeof(float2), 0,
                                cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "tiny weight table: %s", cudaGetErrorString(e));
  TinyParams p;
  memset(&p, 0, sizeof(p));
  p.in = k.seg[0].ptr; p.out = out; p.bias = bias; p.mask_y = mask_y;
  p.N = k.N; p.H = k.Hout; p.W = k.Wout;
  p.nty = k.ay.nu; p.ntx = k.ax.nu;
  p.iuy = k.ay.iu; p.i0y = k.ay.i0; p.iux = k.ax.iu; p.i0x = k.ax.i0;
  p.act = act; p.mask_act = mask_act; p.beta = beta;
  p.xtiles = (k.Wout + TINY_THREADS - 1) / TINY_THREADS;
  const unsigned grid = (unsigned)((size_t)k.N * k.Hout * p.xtiles);
  if (C == 4) tiny_stencil_kernel<4, 4, 12><<<grid, TINY_THREADS, 0, st>>>(p);
  else if (C == 8) tiny_stencil_kernel<8, 8, 8><<<grid, TINY_THREADS, 0, st>>>(p);
  else tiny_stencil_kernel<16, 16, 8><<<grid, TINY_THREADS, 0, st>>>(p);
  NLT_CUDA_LAUNCH_CHECK("tiny_stencil_kernel");
  return NLT_OK;
}

}  // namespace nlt
