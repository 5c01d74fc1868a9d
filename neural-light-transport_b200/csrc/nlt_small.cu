// Small-channel specialisations for the full-resolution edge of the network
// (the layers that own ~65 % of the HBM bytes: SURVEY.md 8a).
//
//  * pw_conv_kernel      : 1x1 / stride-1 convs and their input gradients with
//                          <= 64 input and <= 16 output channels (level-0 convs
//                          5->16 / 3->16, final conv 36->3 and its dgrad).  One
//                          thread = one pixel x one quad of output channels,
//                          weights broadcast from shared memory, no tile staging:
//                          pure streaming, HBM-bound.
//  * wgrad_small_kernel  : weight/bias gradients whose [K x N] result is small
//                          (N <= 16).  Each WARP owns a private pixel stream and
//                          keeps the whole dW tile in registers (k-groups across
//                          lanes); warps, then CTAs, are reduced in a fixed order
//                          (deterministic).  Replaces the tiled split-K kernel
//                          where that one wasted 90 % of its lanes.
#include "nlt_common.cuh"

namespace nlt {


// -----------------------------------------------------------------------------
// pointwise conv
// -----------------------------------------------------------------------------
constexpr int PW_KMAX = 64;
constexpr int PW_THREADS = 256;

bool pw_conv_applicable(const GConvK& k) {
  if (k.ay.nu != 1 || k.ax.nu != 1) return false;
  // identity pixel map: input coordinate == lattice coordinate (== output coordinate unless depth-to-space)
  const AxisMap* ax[2] = {&k.ay, &k.ax};
  for (int i = 0; i < 2; ++i) {
    const AxisMap& a = *ax[i];
    if (a.it != 1 || a.i0 != 0 || a.o0 != 0 || a.os != 1) return false;
  }
  if (k.ay.nt != k.Hin || k.ax.nt != k.Win) return false;
  if (!k.d2s && (k.Hout != k.Hin || k.Wout != k.Win)) return false;
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) ctot += k.seg[s].C;
  // GEMM columns: Cout (d2s: k*k*cout_true, a multiple of 4)
  return ctot <= PW_KMAX && k.Cout <= 64 && (k.Cout <= 16 || k.Cout % 4 == 0);
}

// One thread = one pixel x QT consecutive quads of GEMM columns (QT*4 outputs), R pixels in flight.
// QT = 4 means a thread owns 16 output channels of a pixel: every input value is loaded once per 64 FMAs
// and the thread stores 64 contiguous bytes (the QT = 1 form is issue-bound: ~14 overhead instructions per FMA).
// 4 CTAs per SM (64 registers, a few spilled words outside the k loop): the kernel is latency-bound and wants the
// occupancy more than the registers of the unconstrained allocation (90+).
//
// EX: a second, pointwise term on the OUTPUT lattice is added in the epilogue,
//   out[pix, c] += sum_k ex.x[pix, k] * ex.w[k * wk + c * wn]        (k < ex.K <= PW_EX_KMAX)
// which lets the input gradient of a 1x1 conv ride on the launch that writes the same tensor (no extra
// write + read-modify-write pass over it).
template <int NQ, int QT, int R, int EXM>
__global__ void __launch_bounds__(PW_THREADS, 4)
pw_conv_kernel(const GConvK g, const float* __restrict__ bias, const int act, const float beta,
               const float* __restrict__ mask_y, const int mask_act, float* __restrict__ out, const PwExtra ex) {
  static_assert(NQ % QT == 0, "quads per thread");
  constexpr int LPP = NQ / QT;            // lanes per pixel
  constexpr bool EX = EXM != 0;           // fused pointwise term; EXM: 1 same pixel, 2 lane-per-tap shuffle, 3 per quad
  static_assert(EXM != 2 || (LPP > 1 && LPP == QT), "shuffle mode: one lane per tap");
  __shared__ float4 Ws[PW_KMAX * NQ];     // [k][quad] : 4 consecutive GEMM columns
  __shared__ float4 Wx[EX ? PW_EX_KMAX * 16 : 1];   // [k][channel quad of the output pixel] (cout_true <= 64)
  const int tid = threadIdx.x;
  if (EX) {
    const int cq = g.cout_true >> 2;
    for (int idx = tid; idx < ex.K * cq; idx += PW_THREADS) {
      const int k = idx / cq, q = idx - k * cq;
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = __ldg(ex.w + (long long)k * ex.wk + (long long)(q * 4 + e) * ex.wn);
      Wx[idx] = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
  const int tap = (g.ay.d0) * g.kw + g.ax.d0;
  int K = 0;
  for (int s = 0; s < g.nseg; ++s) K += g.seg[s].C;
  for (int idx = tid; idx < K * NQ; idx += PW_THREADS) {
    const int k = idx / NQ, q = idx - k * NQ;
    int t = tap, nn0 = q * 4;
    if (g.d2s) { t = (int)fdiv((uint32_t)(q * 4), g.div_ct); nn0 = q * 4 - t * g.cout_true; }   // cout_true % 4 == 0: a quad stays in one tap
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      v[e] = q * 4 + e < g.Cout ? __ldg(g.w + (long long)t * g.wt + (long long)k * g.wc + (long long)(nn0 + e) * g.wn) : 0.f;
    Ws[idx] = make_float4(v[0], v[1], v[2], v[3]);
  }
  __syncthreads();

  constexpr int PPB = PW_THREADS / LPP;    // pixels per pass
  // quad j of this thread is QD(j) = qa + j * LPP: the LPP lanes of a pixel hold ADJACENT quads, so each
  // 16-byte load / store instruction of the epilogue covers LPP*16 contiguous bytes per pixel (whole
  // 32-byte sectors) instead of 16 bytes out of every QT*16
  const int qa = tid % LPP;
  const int lane_in_warp = tid & 31;
#define QD(j_) (qa + (j_) * LPP)
  const uint32_t pbase = (uint32_t)blockIdx.x * (PPB * R) + tid / LPP;
  const uint32_t hw = g.div_yx.d;

  uint32_t p[R];
  bool ok[R];
  float acc[R][QT][4];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    p[r] = pbase + r * PPB;
    ok[r] = p[r] < g.M;
  }
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int j = 0; j < QT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[r][j][e] = 0.f;
  if (bias != nullptr) {      // (input-gradient launches carry no bias: keep their prologue free of the loads)
#pragma unroll
    for (int j = 0; j < QT; ++j) {
      int cb = QD(j) * 4;
      if (g.d2s) cb -= (int)fdiv((uint32_t)cb, g.div_ct) * g.cout_true;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float b = QD(j) * 4 + e < g.Cout ? __ldg(bias + cb + e) : 0.f;
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r][j][e] = b;
      }
    }
  }

  // fused pointwise term: its K inputs per output pixel are fetched BEFORE the k loop, so that their latency
  // overlaps the main loads (fetched in the epilogue they add an exposed memory round trip to a
  // latency-bound kernel: measured +25 % per launch).  Modes (chosen by the host, pw_extra_mode):
  //   1 (not depth-to-space): all quads of the thread belong to output pixel p.
  //   2 (depth-to-space, one tap = 4*LPP channels, QT taps): quad j of every lane of the pixel's lane
  //     group belongs to tap j; lane a fetches tap a's pixel and the epilogue reads it by shuffle.
  //   3: anything else -- fetched per quad in the epilogue.
  constexpr int ex_mode = EXM == 3 ? 0 : EXM;
  float xs[EX ? R : 1][PW_EX_KMAX];
  if (EX && ex_mode != 0) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      size_t pix = p[r];
      if (ex_mode == 2) {
        int n, ty, tx;
        decode_pixel(g, p[r], n, ty, tx);
        const int dy = (int)fdiv((uint32_t)qa, g.div_s), dx = qa - dy * g.d2s_s;     // tap index == lane index in the group
        pix = ((uint32_t)n * g.Hout + ty * g.d2s_s + dy) * g.Wout + tx * g.d2s_s + dx;
      }
#pragma unroll
      for (int k2 = 0; k2 < PW_EX_KMAX; ++k2)
        xs[r][k2] = (ok[r] && k2 < ex.K) ? __ldg(ex.x + pix * ex.K + k2) : 0.f;
    }
  }
  int k = 0;
  for (int s = 0; s < g.nseg; ++s) {
    const Seg sg = g.seg[s];
    size_t po[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      uint32_t pp = p[r];
      if (sg.bcast) pp -= fdiv(pp, g.div_yx) * hw;   // batch-broadcast source: pixel index inside the image
      po[r] = (size_t)pp * sg.C;
    }
    if (sg.vec) {
      for (int c = 0; c < sg.C; c += 4) {
        float a[R][4];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok[r]) {
            v = ld4(sg.ptr + po[r] + c);
            if (sg.sub) { const float4 u = ld4(sg.sub + po[r] + c); v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w; }
          }
          a[r][0] = v.x; a[r][1] = v.y; a[r][2] = v.z; a[r][3] = v.w;
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
          for (int j = 0; j < QT; ++j) {
            const float4 w = Ws[(k + kk) * NQ + QD(j)];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              acc[r][j][0] = fmaf(a[r][kk], w.x, acc[r][j][0]); acc[r][j][1] = fmaf(a[r][kk], w.y, acc[r][j][1]);
              acc[r][j][2] = fmaf(a[r][kk], w.z, acc[r][j][2]); acc[r][j][3] = fmaf(a[r][kk], w.w, acc[r][j][3]);
            }
          }
        }
        k += 4;
      }
    } else {
      for (int c = 0; c < sg.C; ++c) {
        float a[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          a[r] = 0.f;
          if (ok[r]) {
            a[r] = __ldg(sg.ptr + po[r] + c);
            if (sg.sub) a[r] -= __ldg(sg.sub + po[r] + c);
          }
        }
#pragma unroll
        for (int j = 0; j < QT; ++j) {
          const float4 w = Ws[k * NQ + QD(j)];
#pragma unroll
          for (int r = 0; r < R; ++r) {
            acc[r][j][0] = fmaf(a[r], w.x, acc[r][j][0]); acc[r][j][1] = fmaf(a[r], w.y, acc[r][j][1]);
            acc[r][j][2] = fmaf(a[r], w.z, acc[r][j][2]); acc[r][j][3] = fmaf(a[r], w.w, acc[r][j][3]);
          }
        }
        ++k;
      }
    }
  }

  // the fused instantiations are only launched on the float4 output path (pw_extra_applicable)
  const bool vec_out = EX || ((g.cout_true % 4 == 0) && aligned16(out) && (mask_y == nullptr || aligned16(mask_y)));
  const bool rmw = (beta != 0.f) || (mask_y != nullptr);
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (!ok[r]) continue;
    // destination of quad QD(j): consecutive quads are consecutive channels of one output pixel
    size_t ob[QT];
    uint32_t opx[EX ? QT : 1];     // output pixel / channel quad of each column quad (fused pointwise term)
    int ocq[EX ? QT : 1];
    int n = 0, ty = 0, tx = 0;
    if (g.d2s) decode_pixel(g, p[r], n, ty, tx);
#pragma unroll
    for (int j = 0; j < QT; ++j) {
      const int col = QD(j) * 4;
      if (g.d2s) {
        const int t = (int)fdiv((uint32_t)col, g.div_ct), cb = col - t * g.cout_true;
        const int dy = (int)fdiv((uint32_t)t, g.div_s), dx = t - dy * g.d2s_s;
        // 32-bit pixel index (build_phases checks N*H*W < 2^31), one widening multiply for the offset
        const uint32_t pix = ((uint32_t)n * g.Hout + ty * g.d2s_s + dy) * g.Wout + tx * g.d2s_s + dx;
        ob[j] = (size_t)pix * (uint32_t)g.cout_true + cb;
        if (EX) { opx[j] = pix; ocq[j] = cb >> 2; }
      } else {
        ob[j] = (size_t)p[r] * g.Cout + col;
        if (EX) { opx[j] = p[r]; ocq[j] = col >> 2; }
      }
    }
    // read-modify-write operands are fetched EB quads at a time before the first store of the group
    // (all QT at once costs 8 more registers per quad and a whole CTA per SM of occupancy)
    constexpr int EB = QT >= 2 ? 2 : 1;
#pragma unroll
    for (int j0 = 0; j0 < QT; j0 += EB) {
      float4 oldv[EB], yv[EB];
#pragma unroll
      for (int jj = 0; jj < EB; ++jj) {
        const int j = j0 + jj;
        oldv[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
        yv[jj] = make_float4(1.f, 1.f, 1.f, 1.f);
        if (rmw && vec_out && QD(j) * 4 < g.Cout) {
          if (beta != 0.f) oldv[jj] = *reinterpret_cast<const float4*>(out + ob[j]);
          if (mask_y != nullptr) yv[jj] = ld4(mask_y + ob[j]);
        }
      }
#pragma unroll
      for (int jj = 0; jj < EB; ++jj) {
        const int j = j0 + jj;
        if (QD(j) * 4 >= g.Cout) continue;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = act_fwd(acc[r][j][e], act);
        if (EX) {     // host guarantees the float4 output path (cout_true % 4 == 0)
          if (ex_mode != 0) {
#pragma unroll
            for (int k2 = 0; k2 < PW_EX_KMAX; ++k2) {
              float a2 = xs[r][k2];
              if (LPP > 1 && ex_mode == 2)       // tap j's pixel was fetched by lane j of this pixel's lane group
                a2 = __shfl_sync(((1u << LPP) - 1u) << (lane_in_warp & ~(LPP - 1)), a2, j, LPP);
              if (k2 < ex.K) {
                const float4 wv = Wx[k2 * (g.cout_true >> 2) + ocq[j]];
                v[0] = fmaf(a2, wv.x, v[0]); v[1] = fmaf(a2, wv.y, v[1]);
                v[2] = fmaf(a2, wv.z, v[2]); v[3] = fmaf(a2, wv.w, v[3]);
              }
            }
          } else {
            const float* xp = ex.x + (size_t)opx[j] * ex.K;
            for (int k2 = 0; k2 < ex.K; ++k2) {
              const float a2 = __ldg(xp + k2);
              const float4 wv = Wx[k2 * (g.cout_true >> 2) + ocq[j]];
              v[0] = fmaf(a2, wv.x, v[0]); v[1] = fmaf(a2, wv.y, v[1]);
              v[2] = fmaf(a2, wv.z, v[2]); v[3] = fmaf(a2, wv.w, v[3]);
            }
          }
        }
        if (vec_out) {
          const float4 o = oldv[jj], y = yv[jj];
          v[0] += beta * o.x; v[1] += beta * o.y; v[2] += beta * o.z; v[3] += beta * o.w;
          if (mask_y != nullptr) {
            v[0] *= act_bwd_from_y(y.x, mask_act); v[1] *= act_bwd_from_y(y.y, mask_act);
            v[2] *= act_bwd_from_y(y.z, mask_act); v[3] *= act_bwd_from_y(y.w, mask_act);
          }
          *reinterpret_cast<float4*>(out + ob[j]) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (QD(j) * 4 + e >= g.Cout) continue;
            float t = v[e];
            if (beta != 0.f) t += beta * out[ob[j] + e];
            if (mask_y != nullptr) t *= act_bwd_from_y(__ldg(mask_y + ob[j] + e), mask_act);
            out[ob[j] + e] = t;
          }
        }
      }
    }
  }
}

#undef QD

// mode of the fused pointwise term for this op (see pw_conv_kernel)
static int pw_extra_mode(const GConvK& k, int lpp, int qt) {
  if (!k.d2s) return 1;
  if (lpp > 1 && lpp == qt && k.cout_true == 4 * lpp && k.d2s_s * k.d2s_s == qt) return 2;
  return 3;
}

template <int NQ, int QT, int R>
static void pw_launch(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                      float* out, const PwExtra* ex, cudaStream_t st) {
  constexpr int LPP = NQ / QT;
  constexpr int PPB = PW_THREADS / LPP * R;
  const unsigned grid = (k.M + PPB - 1) / PPB;
#define NLT_PW(M_, EX_) pw_conv_kernel<NQ, QT, R, M_><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out, EX_)
  if (ex == nullptr) { NLT_PW(0, PwExtra{}); return; }
  const int mode = pw_extra_mode(k, LPP, QT);
  if (mode == 1) NLT_PW(1, *ex);
  else if (mode == 2) { if constexpr (LPP > 1 && LPP == QT) NLT_PW(2, *ex); }
  else NLT_PW(3, *ex);
#undef NLT_PW
}

bool pw_extra_applicable(const GConvK& k, const PwExtra& ex, const float* out, const float* mask_y) {
  return pw_conv_applicable(k) && ex.K >= 1 && ex.K <= PW_EX_KMAX && k.cout_true % 4 == 0 && k.cout_true <= 64 &&
         aligned16(out) && (mask_y == nullptr || aligned16(mask_y));
}

int launch_pw_conv(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                   float* out, cudaStream_t st, const PwExtra* ex) {
  const int nq = (k.Cout + 3) / 4;
  if (nq <= 1) pw_launch<1, 1, 4>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  else if (nq == 2) pw_launch<2, 2, 4>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  else if (nq <= 4) pw_launch<4, 4, 2>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  else if (nq <= 8) pw_launch<8, 4, 2>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  // fused term: one pixel per thread -- at 64 registers the two-pixel form spills ~130 bytes per thread and
  // the local-memory traffic exceeded the useful traffic
  else if (ex != nullptr) pw_launch<16, 4, 1>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  else pw_launch<16, 4, 2>(k, bias, act, beta, mask_y, mask_act, out, ex, st);
  NLT_CUDA_LAUNCH_CHECK("pw_conv_kernel");
  return NLT_OK;
}

// ---- general small direct convolution (taps, strided / phase maps) -----------------
bool dconv_small_applicable(const GConvK& k) {
  // small direct convolution: every (tap, source channel) weight row fits the smem table
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) ctot += k.seg[s].C;
  const int ktot = k.ay.nu * k.ax.nu * ctot;
  if (ktot < 1 || ktot > PW_KMAX) return false;
  // measured against the tiled kernel: wins for the 4..16-channel stencils (K <= 32), and up to K = 64
  // when there are at most 8 output channels
  return (k.Cout <= 16 && ktot <= 32) || (k.Cout <= 8 && ktot <= 64);
}

// One thread = one lattice pixel x one quad of GEMM columns; R pixels per thread in flight; the weight
// table [tap][concat channel][quad] is broadcast from shared memory.  Handles any (small) tap set and
// pixel map of GConvK, so it also covers the 2x2/stride-1 stencils of the 4..16-channel full-resolution
// layers and the phase-decomposed / depth-to-space transposed convs.
template <int NQ, int R>
__global__ void __launch_bounds__(PW_THREADS, 3)
dconv_small_kernel(const GConvK g, const float* __restrict__ bias, const int act, const float beta,
               const float* __restrict__ mask_y, const int mask_act, float* __restrict__ out) {
  __shared__ float4 Ws[PW_KMAX * NQ];   // [k][quad] : 4 consecutive GEMM columns
  const int tid = threadIdx.x;
  int ctot = 0;
  for (int s = 0; s < g.nseg; ++s) ctot += g.seg[s].C;
  const int ntaps = g.ay.nu * g.ax.nu;
  for (int idx = tid; idx < ntaps * ctot * NQ; idx += PW_THREADS) {
    const int k = idx / NQ, q = idx - k * NQ;
    const int tapi = k / ctot, c = k - tapi * ctot;
    const int uy = tapi / g.ax.nu, ux = tapi - uy * g.ax.nu;
    const int tap = (g.ay.d0 + g.ay.ds * uy) * g.kw + (g.ax.d0 + g.ax.ds * ux);
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = q * 4 + e;
      int t = tap, nn = n;
      if (g.d2s) { t = n / g.cout_true; nn = n - t * g.cout_true; }
      v[e] = n < g.Cout ? __ldg(g.w + (long long)t * g.wt + (long long)c * g.wc + (long long)nn * g.wn) : 0.f;
    }
    Ws[idx] = make_float4(v[0], v[1], v[2], v[3]);
  }
  __syncthreads();

  constexpr int PPB = PW_THREADS / NQ;     // pixels per pass
  const int q = tid % NQ;
  const uint32_t pbase = (uint32_t)blockIdx.x * (PPB * R) + tid / NQ;
  // destination channel quad / tap of this thread's GEMM columns
  int qtap = 0, qcb = q * 4;
  if (g.d2s) { qtap = (q * 4) / g.cout_true; qcb = q * 4 - qtap * g.cout_true; }
  const int qdy = g.d2s ? qtap / g.d2s_s : 0, qdx = g.d2s ? qtap - qdy * g.d2s_s : 0;
  float b4[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) b4[e] = (bias != nullptr && q * 4 + e < g.Cout) ? __ldg(bias + qcb + e) : 0.f;

  int pn[R], pty[R], ptx[R];
  bool ok[R];
  float acc[R][4];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const uint32_t pp = pbase + r * PPB;
    ok[r] = pp < g.M;
    pn[r] = 0; pty[r] = 0; ptx[r] = 0;
    if (ok[r]) decode_pixel(g, pp, pn[r], pty[r], ptx[r]);
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[r][e] = b4[e];
  }
  auto out_off = [&](int r) -> size_t {
    int oy, ox;
    if (g.d2s) { oy = pty[r] * g.d2s_s + qdy; ox = ptx[r] * g.d2s_s + qdx; }
    else { oy = g.ay.o0 + g.ay.os * pty[r]; ox = g.ax.o0 + g.ax.os * ptx[r]; }
    return (((size_t)pn[r] * g.Hout + oy) * g.Wout + ox) * g.cout_true + qcb;
  };

  int k = 0;
  for (int uy = 0; uy < g.ay.nu; ++uy)
    for (int ux = 0; ux < g.ax.nu; ++ux) {
      size_t pin[R];       // input pixel index inside an image, and with the batch offset
      bool in[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int iy = pty[r] * g.ay.it + uy * g.ay.iu + g.ay.i0;
        const int ix = ptx[r] * g.ax.it + ux * g.ax.iu + g.ax.i0;
        in[r] = ok[r] && (unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win;
        pin[r] = (size_t)iy * g.Win + ix;
      }
      for (int s = 0; s < g.nseg; ++s) {
        const Seg sg = g.seg[s];
        size_t po[R];
#pragma unroll
        for (int r = 0; r < R; ++r)
          po[r] = (pin[r] + (sg.bcast ? 0 : (size_t)pn[r] * g.Hin * g.Win)) * sg.C;
        if (sg.vec) {
          for (int c = 0; c < sg.C; c += 4) {
            float4 a[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              a[r] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (in[r]) {
                a[r] = ld4(sg.ptr + po[r] + c);
                if (sg.sub) { const float4 u = ld4(sg.sub + po[r] + c); a[r].x -= u.x; a[r].y -= u.y; a[r].z -= u.z; a[r].w -= u.w; }
              }
            }
            const float4 w0 = Ws[(k + 0) * NQ + q], w1 = Ws[(k + 1) * NQ + q], w2 = Ws[(k + 2) * NQ + q],
                         w3 = Ws[(k + 3) * NQ + q];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              acc[r][0] = fmaf(a[r].x, w0.x, acc[r][0]); acc[r][1] = fmaf(a[r].x, w0.y, acc[r][1]);
              acc[r][2] = fmaf(a[r].x, w0.z, acc[r][2]); acc[r][3] = fmaf(a[r].x, w0.w, acc[r][3]);
              acc[r][0] = fmaf(a[r].y, w1.x, acc[r][0]); acc[r][1] = fmaf(a[r].y, w1.y, acc[r][1]);
              acc[r][2] = fmaf(a[r].y, w1.z, acc[r][2]); acc[r][3] = fmaf(a[r].y, w1.w, acc[r][3]);
              acc[r][0] = fmaf(a[r].z, w2.x, acc[r][0]); acc[r][1] = fmaf(a[r].z, w2.y, acc[r][1]);
              acc[r][2] = fmaf(a[r].z, w2.z, acc[r][2]); acc[r][3] = fmaf(a[r].z, w2.w, acc[r][3]);
              acc[r][0] = fmaf(a[r].w, w3.x, acc[r][0]); acc[r][1] = fmaf(a[r].w, w3.y, acc[r][1]);
              acc[r][2] = fmaf(a[r].w, w3.z, acc[r][2]); acc[r][3] = fmaf(a[r].w, w3.w, acc[r][3]);
            }
            k += 4;
          }
        } else {
          for (int c = 0; c < sg.C; ++c) {
            float a[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              a[r] = 0.f;
              if (in[r]) {
                a[r] = __ldg(sg.ptr + po[r] + c);
                if (sg.sub) a[r] -= __ldg(sg.sub + po[r] + c);
              }
            }
            const float4 w0 = Ws[k * NQ + q];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              acc[r][0] = fmaf(a[r], w0.x, acc[r][0]); acc[r][1] = fmaf(a[r], w0.y, acc[r][1]);
              acc[r][2] = fmaf(a[r], w0.z, acc[r][2]); acc[r][3] = fmaf(a[r], w0.w, acc[r][3]);
            }
            ++k;
          }
        }
      }
    }

  const bool vec_out = (g.cout_true % 4 == 0) && aligned16(out) && (mask_y == nullptr || aligned16(mask_y));
  float4 oldv[R], yv[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {   // batch the read-modify-write operands before the first store
    oldv[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    yv[r] = make_float4(1.f, 1.f, 1.f, 1.f);
    if (ok[r] && q * 4 < g.Cout && vec_out) {
      const size_t ob = out_off(r);
      if (beta != 0.f) oldv[r] = *reinterpret_cast<const float4*>(out + ob);
      if (mask_y != nullptr) yv[r] = ld4(mask_y + ob);
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (!ok[r] || q * 4 >= g.Cout) continue;
    const size_t ob = out_off(r);
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = act_fwd(acc[r][e], act);
    if (vec_out) {
      const float4 o = oldv[r], y = yv[r];
      v[0] += beta * o.x; v[1] += beta * o.y; v[2] += beta * o.z; v[3] += beta * o.w;
      if (mask_y != nullptr) {
        v[0] *= act_bwd_from_y(y.x, mask_act); v[1] *= act_bwd_from_y(y.y, mask_act);
        v[2] *= act_bwd_from_y(y.z, mask_act); v[3] *= act_bwd_from_y(y.w, mask_act);
      }
      *reinterpret_cast<float4*>(out + ob) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (q * 4 + e >= g.Cout) continue;
        float t = v[e];
        if (beta != 0.f) t += beta * out[ob + e];
        if (mask_y != nullptr) t *= act_bwd_from_y(__ldg(mask_y + ob + e), mask_act);
        out[ob + e] = t;
      }
    }
  }
}

// -----------------------------------------------------------------------------
// Wide form of the small direct convolution: one thread = one lattice pixel x ALL 16 output channels (4
// quads), R pixels per thread.  For the 16 -> 16 channel stencils (K = taps * C = 64) the tiled implicit-GEMM
// kernel spends most of its instructions on address generation; here every
// input float4 is loaded once per 64 FMAs and every weight LDS.128 feeds 4*R FMAs.  Vector sources only, no
// depth-to-space (those go to the pointwise kernel).
// -----------------------------------------------------------------------------
constexpr int DW_KMAX = 128;   // taps * channels of the widest routed stencil (32 -> 32 channels, 2x2)

// CW = true: the weight table [k][quad] lives in CONSTANT memory (filled per launch by dconv_cw_pack_kernel + a
// device-to-device symbol copy).  Every lane needs the same weight at the same time, so it is a constant-bank operand
// of the FMA: the 128 broadcast LDS.128 per pixel of the shared-memory form are not issued.
// One table per device: launches from different streams must not overlap (the engine issues forward convs and input
// gradients from its main stream only; weight gradients, on the side stream, never use this kernel).
__constant__ float4 dw_cw[DW_KMAX * 8];
__device__ float4 dw_cw_stage[DW_KMAX * 8];

__global__ void dconv_cw_pack_kernel(const GConvK g, int qt) {
  int ctot = 0;
  for (int s = 0; s < g.nseg; ++s) ctot += g.seg[s].C;
  const int ntaps = g.ay.nu * g.ax.nu;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < ntaps * ctot * qt; idx += gridDim.x * blockDim.x) {
    const int k = idx / qt, q = idx - k * qt;
    const int tapi = k / ctot, c = k - tapi * ctot;
    const int uy = tapi / g.ax.nu, ux = tapi - uy * g.ax.nu;
    const int tap = (g.ay.d0 + g.ay.ds * uy) * g.kw + (g.ax.d0 + g.ax.ds * ux);
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = q * 4 + e;
      v[e] = n < g.Cout ? __ldg(g.w + (long long)tap * g.wt + (long long)c * g.wc + (long long)n * g.wn) : 0.f;
    }
    dw_cw_stage[idx] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

template <int DW_QT, int R, int MINB, bool CW = false>
__global__ void __launch_bounds__(PW_THREADS, MINB)
dconv_wide_kernel(const GConvK g, const float* __restrict__ bias, const int act, const float beta,
                  const float* __restrict__ mask_y, const int mask_act, float* __restrict__ out) {
  __shared__ float4 Ws[CW ? 1 : (DW_QT == 4 ? PW_KMAX : DW_KMAX) * DW_QT];   // [k][quad]
  const int tid = threadIdx.x;
  int ctot = 0;
  for (int s = 0; s < g.nseg; ++s) ctot += g.seg[s].C;
  const int ntaps = g.ay.nu * g.ax.nu;
  if (!CW) {
    for (int idx = tid; idx < ntaps * ctot * DW_QT; idx += PW_THREADS) {
      const int k = idx / DW_QT, q = idx - k * DW_QT;
      const int tapi = k / ctot, c = k - tapi * ctot;
      const int uy = tapi / g.ax.nu, ux = tapi - uy * g.ax.nu;
      const int tap = (g.ay.d0 + g.ay.ds * uy) * g.kw + (g.ax.d0 + g.ax.ds * ux);
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = q * 4 + e;
        v[e] = n < g.Cout ? __ldg(g.w + (long long)tap * g.wt + (long long)c * g.wc + (long long)n * g.wn) : 0.f;
      }
      Ws[idx] = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
  }

  const uint32_t pbase = (uint32_t)blockIdx.x * (PW_THREADS * R) + tid;
  int pn[R], pty[R], ptx[R];
  bool ok[R];
  float acc[R][DW_QT][4];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const uint32_t pp = pbase + r * PW_THREADS;
    ok[r] = pp < g.M;
    pn[r] = 0; pty[r] = 0; ptx[r] = 0;
    if (ok[r]) decode_pixel(g, pp, pn[r], pty[r], ptx[r]);
#pragma unroll
    for (int j = 0; j < DW_QT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[r][j][e] = 0.f;
  }
  if (bias != nullptr) {
#pragma unroll
    for (int j = 0; j < DW_QT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float b = j * 4 + e < g.Cout ? __ldg(bias + j * 4 + e) : 0.f;
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r][j][e] = b;
      }
  }

  int k = 0;
  for (int uy = 0; uy < g.ay.nu; ++uy)
    for (int ux = 0; ux < g.ax.nu; ++ux) {
      uint32_t pin[R];     // input pixel index (batch included; build_phases checks N*H*W < 2^31)
      bool in[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int iy = pty[r] * g.ay.it + uy * g.ay.iu + g.ay.i0;
        const int ix = ptx[r] * g.ax.it + ux * g.ax.iu + g.ax.i0;
        in[r] = ok[r] && (unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win;
        pin[r] = ((uint32_t)pn[r] * g.Hin + iy) * g.Win + ix;
      }
      for (int s = 0; s < g.nseg; ++s) {
        const Seg sg = g.seg[s];
        const float* pa[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          uint32_t pix = pin[r];
          if (sg.bcast) pix -= (uint32_t)pn[r] * g.Hin * g.Win;
          pa[r] = sg.ptr + (size_t)pix * sg.C;
        }
        for (int c = 0; c < sg.C; c += 4) {
          float a[R][4];
#pragma unroll
          for (int r = 0; r < R; ++r) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in[r]) v = ld4(pa[r] + c);
            a[r][0] = v.x; a[r][1] = v.y; a[r][2] = v.z; a[r][3] = v.w;
          }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int j = 0; j < DW_QT; ++j) {
              if constexpr (CW) {
                const float4 w = dw_cw[(k + kk) * DW_QT + j];
#pragma unroll
                for (int r = 0; r < R; ++r) {
                  const float2 aa = make_float2(a[r][kk], a[r][kk]);
                  const float2 lo = ffma2(aa, make_float2(w.x, w.y), make_float2(acc[r][j][0], acc[r][j][1]));
                  const float2 hi = ffma2(aa, make_float2(w.z, w.w), make_float2(acc[r][j][2], acc[r][j][3]));
                  acc[r][j][0] = lo.x; acc[r][j][1] = lo.y; acc[r][j][2] = hi.x; acc[r][j][3] = hi.y;
                }
              } else {
                const float4 w = Ws[(k + kk) * DW_QT + j];
#pragma unroll
                for (int r = 0; r < R; ++r) {
                  acc[r][j][0] = fmaf(a[r][kk], w.x, acc[r][j][0]); acc[r][j][1] = fmaf(a[r][kk], w.y, acc[r][j][1]);
                  acc[r][j][2] = fmaf(a[r][kk], w.z, acc[r][j][2]); acc[r][j][3] = fmaf(a[r][kk], w.w, acc[r][j][3]);
                }
              }
            }
          }
          k += 4;
        }
      }
    }

  // epilogue: Cout % 4 == 0 and 16-byte aligned out / mask (checked by the host): float4 path only
  const int nqo = g.Cout >> 2;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (!ok[r]) continue;
    const int oy = g.ay.o0 + g.ay.os * pty[r], ox = g.ax.o0 + g.ax.os * ptx[r];
    const size_t ob = (size_t)(((uint32_t)pn[r] * g.Hout + oy) * g.Wout + ox) * (uint32_t)g.Cout;
    constexpr int EB = 2;
#pragma unroll
    for (int j0 = 0; j0 < DW_QT; j0 += EB) {
      float4 oldv[EB], yv[EB];
#pragma unroll
      for (int jj = 0; jj < EB; ++jj) {
        oldv[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
        yv[jj] = make_float4(1.f, 1.f, 1.f, 1.f);
        if (j0 + jj < nqo) {
          if (beta != 0.f) oldv[jj] = *reinterpret_cast<const float4*>(out + ob + (j0 + jj) * 4);
          if (mask_y != nullptr) yv[jj] = ld4(mask_y + ob + (j0 + jj) * 4);
        }
      }
#pragma unroll
      for (int jj = 0; jj < EB; ++jj) {
        const int j = j0 + jj;
        if (j >= nqo) continue;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = act_fwd(acc[r][j][e], act);
        const float4 o = oldv[jj], y = yv[jj];
        v[0] += beta * o.x; v[1] += beta * o.y; v[2] += beta * o.z; v[3] += beta * o.w;
        if (mask_y != nullptr) {
          v[0] *= act_bwd_from_y(y.x, mask_act); v[1] *= act_bwd_from_y(y.y, mask_act);
          v[2] *= act_bwd_from_y(y.z, mask_act); v[3] *= act_bwd_from_y(y.w, mask_act);
        }
        *reinterpret_cast<float4*>(out + ob + j * 4) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  }
}

static bool dconv_wide_common(const GConvK& k, const float* out, const float* mask_y, int cout, int kmax, bool multi_seg) {
  if (k.d2s || k.M == 0) return false;
  if (k.Cout != cout || k.cout_true != k.Cout) return false;
  // the hardware-validated route (16 outputs) takes ONE non-broadcast float4 source; the experimental routes also
  // take virtual concats (the kernel is written for any segment list)
  if (!multi_seg && k.nseg != 1) return false;
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) {
    if (!k.seg[s].vec || k.seg[s].sub != nullptr || k.seg[s].bcast) return false;
    ctot += k.seg[s].C;
  }
  const int ktot = k.ay.nu * k.ax.nu * ctot;
  if (ktot < 1 || ktot > kmax) return false;
  return aligned16(out) && (mask_y == nullptr || aligned16(mask_y));
}

bool dconv_wide_applicable(const GConvK& k, const float* out, const float* mask_y) {
  return dconv_wide_common(k, out, mask_y, 16, PW_KMAX, false) || dconv_wide_common(k, out, mask_y, 32, DW_KMAX, true) ||
         dconv_wide_common(k, out, mask_y, 8, DW_KMAX, true);
}

static int dconv_cw_fill(const GConvK& k, int qt, cudaStream_t st) {
  dconv_cw_pack_kernel<<<8, 256, 0, st>>>(k, qt);
  NLT_CUDA_LAUNCH_CHECK("dconv_cw_pack_kernel");
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) ctot += k.seg[s].C;
  const size_t n = (size_t)k.ay.nu * k.ax.nu * ctot * qt;
  void* stage = nullptr;
  cudaError_t e = cudaGetSymbolAddress(&stage, dw_cw_stage);
  if (e == cudaSuccess) e = cudaMemcpyToSymbolAsync(dw_cw, stage, n * sizeof(float4), 0, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "dconv weight table: %s", cudaGetErrorString(e));
  return NLT_OK;
}

int launch_dconv_wide(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                      float* out, cudaStream_t st) {
  // option "dconv_cw": the weights of the 16- / 8-output forms from a constant-memory table
  if (opt(Opt::DCONV_CW) == 1 && (k.Cout == 16 || k.Cout == 8)) {
    int rc = dconv_cw_fill(k, k.Cout / 4, st);
    if (rc != NLT_OK) return rc;
    if (k.Cout == 16) {
      constexpr int R = 2;
      const unsigned grid = (k.M + PW_THREADS * R - 1) / (PW_THREADS * R);
      dconv_wide_kernel<4, R, 3, true><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
    } else {
      const unsigned grid = (k.M + PW_THREADS * 4 - 1) / (PW_THREADS * 4);
      dconv_wide_kernel<2, 4, 3, true><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
    }
    NLT_CUDA_LAUNCH_CHECK("dconv_wide_kernel");
    return NLT_OK;
  }
  if (k.Cout == 16) {
    constexpr int R = 2;
    const unsigned grid = (k.M + PW_THREADS * R - 1) / (PW_THREADS * R);
    dconv_wide_kernel<4, R, 3><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
  } else if (k.Cout == 8) {                  // experimental: pixel x 8 outputs, four pixels per thread
    const unsigned grid = (k.M + PW_THREADS * 4 - 1) / (PW_THREADS * 4);
    dconv_wide_kernel<2, 4, 3><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
  } else if (opt(Opt::DCONV_WIDE32) == 2) {      // two pixels per thread: 8 FMAs per weight LDS.128, ~2 CTAs per SM
    const unsigned grid = (k.M + PW_THREADS * 2 - 1) / (PW_THREADS * 2);
    dconv_wide_kernel<8, 2, 2><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
  } else {                                   // one pixel per thread: 4 FMAs per weight LDS.128, 3 CTAs per SM
    const unsigned grid = (k.M + PW_THREADS - 1) / PW_THREADS;
    dconv_wide_kernel<8, 1, 3><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
  }
  NLT_CUDA_LAUNCH_CHECK("dconv_wide_kernel");
  return NLT_OK;
}

template <int NQ, int R>
static void dconv_launch(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                      float* out, cudaStream_t st) {
  constexpr int PPB = PW_THREADS / NQ * R;
  const unsigned grid = (k.M + PPB - 1) / PPB;
  dconv_small_kernel<NQ, R><<<grid, PW_THREADS, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
}

int launch_dconv_small(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                   float* out, cudaStream_t st) {
  const int nq = (k.Cout + 3) / 4;
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) ctot += k.seg[s].C;
  (void)ctot;
  if (nq <= 1) dconv_launch<1, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
  else if (nq == 2) dconv_launch<2, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
  else if (nq <= 4) dconv_launch<4, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
  else if (nq <= 8) dconv_launch<8, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
  else dconv_launch<16, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
  NLT_CUDA_LAUNCH_CHECK("dconv_small_kernel");
  return NLT_OK;
}

// -----------------------------------------------------------------------------
// warp-stream wgrad for small result tiles
// -----------------------------------------------------------------------------
constexpr int WS_WARPS = 4;
constexpr int WS_THREADS = WS_WARPS * 32;

struct WsPlan {
  int nq, p, kq, GS, KG, nsplit;
  uint32_t pps;
  size_t KD_pad;
  int ld;
};

static bool ws_plan(const GConvK& k, WsPlan& pl) {
  // depth-to-space form (transposed op with k == stride): ONE pass over the input lattice with
  // N' = k*k*Cout gradient columns, instead of k*k phases that each re-read the whole input
  if (k.Cout > 32 || k.M == 0 || (!k.d2s && k.Cout > 16)) return false;
  pl.nq = k.Cout <= 4 ? 1 : k.Cout <= 8 ? 2 : k.Cout <= 16 ? 4 : 8;
  pl.kq = 32 / pl.nq;
  pl.GS = 0;
  for (int s = 0; s < k.nseg; ++s) pl.GS += (k.seg[s].C + 3) / 4;
  pl.KG = k.ay.nu * k.ax.nu * pl.GS + 1;
  const int real = pl.KG - 1;
  int p = (real + pl.kq - 1) / pl.kq;
  if (p < 1) p = 1;
  // instantiated: NQ=8: P in {1,2,4,5}; NQ=4: P in {1,2,4,5}; NQ=2: {1,2}; NQ=1: {1,2}
  if (pl.nq >= 4) { if (p == 3) p = 4; if (p > 5) return false; }
  else if (p > 2) return false;
  pl.p = p;
  pl.ld = pl.nq * 4;
  pl.KD_pad = (size_t)(p * pl.kq + 1) * 4;
  long long want = (long long)sm_count() * (p <= 2 ? 8 : 4);
  const long long max_split = ((long long)k.M + 255) / 256;
  if (want > max_split) want = max_split;
  if (want < 1) want = 1;
  pl.pps = (uint32_t)(((long long)k.M + want - 1) / want);
  pl.nsplit = (int)((k.M + pl.pps - 1) / pl.pps);
  return true;
}

bool wgrad_small_applicable(const GConvK& k) {
  WsPlan pl;
  return ws_plan(k, pl);
}

size_t wgrad_small_ws_floats(const GConvK& k) {
  WsPlan pl;
  if (!ws_plan(k, pl)) return 0;
  return (size_t)pl.nsplit * pl.KD_pad * pl.ld;
}

template <int NQ, int P, int U>
__global__ void __launch_bounds__(WS_THREADS)
wgrad_small_kernel(const WgradK w, const float* __restrict__ G, float* __restrict__ ws) {
  constexpr int KQ = 32 / NQ;
  constexpr int ROWS = (P * KQ + 1) * 4;       // tile rows incl. the bias group
  constexpr int LD = NQ * 4;
  __shared__ float tile[ROWS * LD];

  const GConvK& g = w.g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kq = lane / NQ, nq = lane % NQ;

  // this lane's k-groups (fixed): kg_j = kq + j*KQ
  const float* jptr[P];
  const float* jsub[P];
  int jC[P], jc[P], jdy[P], jdx[P], jflag[P];   // flag: 0 dead, 1 vec, 2 scalar, |4 bcast
#pragma unroll
  for (int j = 0; j < P; ++j) {
    int uy, ux, s, c;
    decode_kgroup(w, kq + j * KQ, uy, ux, s, c);
    jptr[j] = nullptr; jsub[j] = nullptr; jC[j] = 0; jc[j] = 0; jdy[j] = 0; jdx[j] = 0; jflag[j] = 0;
    if (s >= 0) {
      const Seg sg = g.seg[s];
      jptr[j] = sg.ptr; jsub[j] = sg.sub; jC[j] = sg.C; jc[j] = c;
      jdy[j] = uy * g.ay.iu + g.ay.i0; jdx[j] = ux * g.ax.iu + g.ax.i0;
      jflag[j] = (sg.vec ? 1 : 2) | (sg.bcast ? 4 : 0);
    }
  }
  const bool g_vec = (g.cout_true % 4 == 0) && aligned16(G);

  float acc[P][4][4];
  float gsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < P; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
      for (int f = 0; f < 4; ++f) acc[j][e][f] = 0.f;

  const uint32_t p_begin = blockIdx.x * w.pix_per_split;
  const uint32_t p_end = min(g.M, p_begin + w.pix_per_split);

  auto load_pixel = [&](uint32_t m, float4 (&a)[P], float4& gv) {
    gv = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < P; ++j) a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m >= p_end) return;
    int n, ty, tx;
    decode_pixel(g, m, n, ty, tx);
    int oy = g.ay.o0 + g.ay.os * ty, ox = g.ax.o0 + g.ax.os * tx, cb = nq * 4;
    if (g.d2s) {      // gradient column quad -> (tap, channel quad) of the up-sampled output pixel
      const int tap = (nq * 4) / g.cout_true;
      cb = nq * 4 - tap * g.cout_true;
      const int dy = tap / g.d2s_s;
      oy = ty * g.d2s_s + dy; ox = tx * g.d2s_s + (tap - dy * g.d2s_s);
    }
    const size_t goff = (((size_t)n * g.Hout + oy) * g.Wout + ox) * g.cout_true + cb;
    if (nq * 4 < g.Cout) {
      if (g_vec) {
        gv = ld4(G + goff);
      } else {
        float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (nq * 4 + e < g.Cout) t[e] = __ldg(G + goff + e);
        gv = make_float4(t[0], t[1], t[2], t[3]);
      }
    }
    const int by = ty * g.ay.it, bx = tx * g.ax.it;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      if (jflag[j] == 0) continue;
      const int iy = by + jdy[j], ix = bx + jdx[j];
      if ((unsigned)iy >= (unsigned)g.Hin || (unsigned)ix >= (unsigned)g.Win) continue;
      const size_t off = (((size_t)((jflag[j] & 4) ? 0 : n) * g.Hin + iy) * g.Win + ix) * jC[j] + jc[j];
      if (jflag[j] & 1) {
        float4 v = ld4(jptr[j] + off);
        if (jsub[j]) { const float4 u = ld4(jsub[j] + off); v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w; }
        a[j] = v;
      } else {
        float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (jc[j] + e < jC[j]) {
            t[e] = __ldg(jptr[j] + off + e);
            if (jsub[j]) t[e] -= __ldg(jsub[j] + off + e);
          }
        a[j] = make_float4(t[0], t[1], t[2], t[3]);
      }
    }
  };
  auto fma_pixel = [&](const float4 (&a)[P], const float4& gv) {
    const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
    for (int f = 0; f < 4; ++f) gsum[f] += gg[f];
#pragma unroll
    for (int j = 0; j < P; ++j) {
      const float aa[4] = {a[j].x, a[j].y, a[j].z, a[j].w};
#pragma unroll
      for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int f = 0; f < 4; ++f) acc[j][e][f] = fmaf(aa[e], gg[f], acc[j][e][f]);
    }
  };

  // U pixels in flight per warp iteration (adjacent warps take adjacent pixels): the
  // kernel is a pure stream, so memory-level parallelism is what sets its speed
  for (uint32_t m = p_begin + warp; m < p_end; m += U * WS_WARPS) {
    float4 a[U][P], gv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) load_pixel(m + u * WS_WARPS, a[u], gv[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) fma_pixel(a[u], gv[u]);
  }

  // ---- fixed-order reduction over the CTA's warps, then one partial per CTA ----
  for (int i = tid; i < ROWS * LD; i += WS_THREADS) tile[i] = 0.f;
  __syncthreads();
  const int bias_row = (w.KG - 1) * 4;
  for (int wi = 0; wi < WS_WARPS; ++wi) {
    if (warp == wi) {
#pragma unroll
      for (int j = 0; j < P; ++j) {
        if (jflag[j] == 0) continue;
        const int kg = kq + j * KQ;
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
          for (int f = 0; f < 4; ++f) tile[(kg * 4 + e) * LD + nq * 4 + f] += acc[j][e][f];
      }
      if (kq == 0) {
#pragma unroll
        for (int f = 0; f < 4; ++f) tile[bias_row * LD + nq * 4 + f] += gsum[f];
      }
    }
    __syncthreads();
  }
  float* dst = ws + (size_t)blockIdx.x * ROWS * LD;
  for (int i = tid; i < ROWS * LD; i += WS_THREADS) dst[i] = tile[i];
}

// -----------------------------------------------------------------------------
// Row-run form of the warp-stream wgrad.  wgrad_small_kernel<4,2,4> issues ~170 warp instructions per
// pixel for 36 FMAs -- the flat pixel index is decoded and every source address rebuilt from scratch for
// every pixel.  Here a warp owns a run of WR_CHUNK consecutive lattice pixels of one row: (n, ty) and all
// base pointers are set up once per run and the pixel loop only adds constant strides.  Requires float4
// access everywhere (all segments vec, no subtracted source, gradient channels % 4 == 0); same workspace layout and the same
// fixed-order reduction as wgrad_small_kernel, so the two are interchangeable.
// -----------------------------------------------------------------------------
constexpr int WR_CHUNK = 64;

template <int NQ, int P, int U, int MINB>
__global__ void __launch_bounds__(WS_THREADS, MINB)
wgrad_rows_kernel(const WgradK w, const float* __restrict__ G, float* __restrict__ ws, const uint32_t cpr,
                  const uint32_t nchunks) {
  constexpr int KQ = 32 / NQ;
  constexpr int ROWS = (P * KQ + 1) * 4;
  constexpr int LD = NQ * 4;
  __shared__ float tile[ROWS * LD];

  const GConvK& g = w.g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kq = lane / NQ, nq = lane % NQ;

  const float* jptr[P];
  int jstr[P], jdy[P], jdx[P], jimg[P];   // pixel stride (floats), tap offsets, image stride (0: broadcast)
  bool jlive[P];
#pragma unroll
  for (int j = 0; j < P; ++j) {
    int uy, ux, s, c;
    decode_kgroup(w, kq + j * KQ, uy, ux, s, c);
    jptr[j] = nullptr; jstr[j] = 0; jdy[j] = 0; jdx[j] = 0; jimg[j] = 0; jlive[j] = false;
    if (s >= 0) {
      const Seg sg = g.seg[s];
      jptr[j] = sg.ptr + c;
      jstr[j] = sg.C;
      jdy[j] = uy * g.ay.iu + g.ay.i0; jdx[j] = ux * g.ax.iu + g.ax.i0;
      jimg[j] = sg.bcast ? 0 : 1;
      jlive[j] = true;
    }
  }
  // gradient column quad of this lane -> fixed (dy, dx, channel) inside the output pixel block
  int g_dy = 0, g_dx = 0, g_cb = nq * 4, g_sy = g.ay.os, g_sx = g.ax.os, g_y0 = g.ay.o0, g_x0 = g.ax.o0;
  if (g.d2s) {
    const int tap = (nq * 4) / g.cout_true;
    g_cb = nq * 4 - tap * g.cout_true;
    g_dy = tap / g.d2s_s; g_dx = tap - g_dy * g.d2s_s;
    g_sy = g.d2s_s; g_sx = g.d2s_s; g_y0 = 0; g_x0 = 0;
  }
  const bool g_live = nq * 4 < g.Cout;
  const int g_str = g_sx * g.cout_true;

  float acc[P][4][4];
  float gsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < P; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
      for (int f = 0; f < 4; ++f) acc[j][e][f] = 0.f;

  const int ntx = g.ax.nt, nty = g.ay.nt;
  for (uint32_t ch = blockIdx.x * WS_WARPS + warp; ch < nchunks; ch += gridDim.x * WS_WARPS) {
    const uint32_t row = ch / cpr;
    const int x0 = (int)(ch - row * cpr) * WR_CHUNK;
    const int xend = min(ntx, x0 + WR_CHUNK);
    const int n = (int)(row / (uint32_t)nty), ty = (int)(row - (uint32_t)n * nty);

    const float* gp = G + (((size_t)n * g.Hout + (g_y0 + g_sy * ty + g_dy)) * g.Wout + (g_x0 + g_dx)) * g.cout_true + g_cb;
    const float* pa[P];
    bool oky[P];
#pragma unroll
    for (int j = 0; j < P; ++j) {
      const int iy = ty * g.ay.it + jdy[j];
      oky[j] = jlive[j] && (unsigned)iy < (unsigned)g.Hin;
      const long long off = (((long long)(jimg[j] ? n : 0) * g.Hin + iy) * g.Win + jdx[j]) * jstr[j];
      pa[j] = jptr[j] + off;
    }

    for (int x = x0; x < xend; x += U) {
      float4 a[U][P], gv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int xx = x + u;
        const bool in = xx < xend;
        gv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in && g_live) gv[u] = ld4(gp + (long long)xx * g_str);
#pragma unroll
        for (int j = 0; j < P; ++j) {
          const int ix = xx * g.ax.it;
          const bool ok = in && oky[j] && (unsigned)(ix + jdx[j]) < (unsigned)g.Win;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok) v = ld4(pa[j] + (long long)ix * jstr[j]);
          a[u][j] = v;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float gg[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
#pragma unroll
        for (int f = 0; f < 4; ++f) gsum[f] += gg[f];
#pragma unroll
        for (int j = 0; j < P; ++j) {
          const float aa[4] = {a[u][j].x, a[u][j].y, a[u][j].z, a[u][j].w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int f = 0; f < 4; ++f) acc[j][e][f] = fmaf(aa[e], gg[f], acc[j][e][f]);
        }
      }
    }
  }

  for (int i = tid; i < ROWS * LD; i += WS_THREADS) tile[i] = 0.f;
  __syncthreads();
  const int bias_row = (w.KG - 1) * 4;
  for (int wi = 0; wi < WS_WARPS; ++wi) {
    if (warp == wi) {
#pragma unroll
      for (int j = 0; j < P; ++j) {
        if (!jlive[j]) continue;
        const int kg = kq + j * KQ;
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
          for (int f = 0; f < 4; ++f) tile[(kg * 4 + e) * LD + nq * 4 + f] += acc[j][e][f];
      }
      if (kq == 0) {
#pragma unroll
        for (int f = 0; f < 4; ++f) tile[bias_row * LD + nq * 4 + f] += gsum[f];
      }
    }
    __syncthreads();
  }
  float* dst = ws + (size_t)blockIdx.x * ROWS * LD;
  for (int i = tid; i < ROWS * LD; i += WS_THREADS) dst[i] = tile[i];
}

static bool wgrad_rows_ok(const GConvK& k, const float* G) {
  if (k.cout_true % 4 != 0 || k.Cout % 4 != 0 || !aligned16(G)) return false;
  for (int s = 0; s < k.nseg; ++s)
    if (!k.seg[s].vec || k.seg[s].sub != nullptr) return false;
  return true;
}

// -----------------------------------------------------------------------------
// thread-per-pixel wgrad for tiny results (K*N <= ~128: level-0 convs, final
// conv, the 4->4 full-resolution deconv).  Every THREAD owns a pixel stream and
// the complete dW tile in registers, so per pixel it costs only the loads and
// the K*N FMAs (no per-pixel work replicated across a warp); warp shuffles,
// then a fixed-order smem pass, reduce the tile (deterministic).
// -----------------------------------------------------------------------------
constexpr int TPP_MAX_LOADS = 12;
constexpr int TPP_THREADS = 128;

struct TppLoad {
  const float* ptr;
  const float* sub;
  int C, c, dy, dx, row, bcast;
};
struct TppK {
  GConvK g;
  TppLoad ld[TPP_MAX_LOADS];
  int nl;          // loads per pixel
  int rows;        // workspace rows (KG * 4 incl. the bias group)
  int ldw;         // workspace row stride (padded Cout)
  int bias_row;
};

template <int NL, int VEC, int N>
__global__ void __launch_bounds__(TPP_THREADS)
wgrad_tpp_kernel(const TppK t, const float* __restrict__ G, float* __restrict__ ws) {
  constexpr int R = NL * VEC;
  constexpr int NW = TPP_THREADS / 32;
  __shared__ float red[NW][R * N + N];
  const GConvK& g = t.g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float acc[R][N];
  float gsum[N];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int n = 0; n < N; ++n) acc[r][n] = 0.f;
#pragma unroll
  for (int n = 0; n < N; ++n) gsum[n] = 0.f;
  const bool g_vec = (N % 4 == 0) && (g.Cout == N) && aligned16(G);
  // K-split: blockIdx.y owns loads [l0, l0 + NL) of the pixel (its own rows of the result); every y
  // re-reads the (narrow) gradient, y == 0 also produces the bias sums
  const int l0 = blockIdx.y * NL;

  for (uint32_t m = blockIdx.x * TPP_THREADS + tid; m < g.M; m += gridDim.x * TPP_THREADS) {
    int n, ty, tx;
    decode_pixel(g, m, n, ty, tx);
    const int oy = g.ay.o0 + g.ay.os * ty, ox = g.ax.o0 + g.ax.os * tx;
    const size_t goff = (((size_t)n * g.Hout + oy) * g.Wout + ox) * g.Cout;
    float gv[N];
    if (g_vec) {
#pragma unroll
      for (int q = 0; q < N / 4; ++q) {
        const float4 v = ld4(G + goff + q * 4);
        gv[q * 4 + 0] = v.x; gv[q * 4 + 1] = v.y; gv[q * 4 + 2] = v.z; gv[q * 4 + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int e = 0; e < N; ++e) gv[e] = e < g.Cout ? __ldg(G + goff + e) : 0.f;
    }
    float a[R];
    const int by = ty * g.ay.it, bx = tx * g.ax.it;
#pragma unroll
    for (int l = 0; l < NL; ++l) {
      const TppLoad L = t.ld[l0 + l];
      const int iy = by + L.dy, ix = bx + L.dx;
#pragma unroll
      for (int e = 0; e < VEC; ++e) a[l * VEC + e] = 0.f;
      if ((unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win) {
        const size_t off = (((size_t)(L.bcast ? 0 : n) * g.Hin + iy) * g.Win + ix) * L.C + L.c;
        if (VEC == 4) {
          float4 v = ld4(L.ptr + off);
          if (L.sub) { const float4 u = ld4(L.sub + off); v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w; }
          a[l * VEC + 0] = v.x; a[l * VEC + (VEC > 1 ? 1 : 0)] = VEC > 1 ? v.y : v.x;
          a[l * VEC + (VEC > 2 ? 2 : 0)] = VEC > 2 ? v.z : v.x; a[l * VEC + (VEC > 3 ? 3 : 0)] = VEC > 3 ? v.w : v.x;
        } else {
          float v = __ldg(L.ptr + off);
          if (L.sub) v -= __ldg(L.sub + off);
          a[l * VEC] = v;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < N; ++e) gsum[e] += gv[e];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int e = 0; e < N; ++e) acc[r][e] = fmaf(a[r], gv[e], acc[r][e]);
  }

  // warp reduction (fixed butterfly order), then warps in fixed order
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int e = 0; e < N; ++e) {
      float v = acc[r][e];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][r * N + e] = v;
    }
#pragma unroll
  for (int e = 0; e < N; ++e) {
    float v = gsum[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][R * N + e] = v;
  }
  __syncthreads();
  float* dst = ws + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * t.rows * t.ldw;
  for (int i = tid; i < t.rows * t.ldw; i += TPP_THREADS) dst[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < R * N + (blockIdx.y == 0 ? N : 0); i += TPP_THREADS) {
    float v = 0.f;
#pragma unroll
    for (int wi = 0; wi < NW; ++wi) v += red[wi][i];
    int row, col;
    if (i < R * N) {
      const int r = i / N;
      col = i - r * N;
      row = t.ld[l0 + r / VEC].row + (r % VEC);
    } else {
      row = t.bias_row; col = i - R * N;
    }
    if (col < t.ldw) dst[(size_t)row * t.ldw + col] = v;
  }
}

struct TppPlan {
  bool ok;
  int nl, vec, n;
  int ksplit;      // blockIdx.y extent: the nl loads are split into ksplit groups of nl / ksplit
  int GS, KG, nsplit;
  TppK k;
};

static TppPlan tpp_plan(const GConvK& k) {
  TppPlan pl;
  pl.ok = false;
  if (k.d2s || k.M == 0 || k.Cout > 16) return pl;
  bool all_vec = true, none_vec = true;
  for (int s = 0; s < k.nseg; ++s) { if (k.seg[s].vec) none_vec = false; else all_vec = false; }
  if (!all_vec && !none_vec) return pl;
  pl.vec = all_vec ? 4 : 1;
  pl.n = k.Cout <= 3 ? 3 : k.Cout <= 4 ? 4 : k.Cout == 16 ? 16 : 0;
  if (pl.n == 0) return pl;
  pl.GS = 0;
  for (int s = 0; s < k.nseg; ++s) pl.GS += (k.seg[s].C + 3) / 4;
  const int taps = k.ay.nu * k.ax.nu;
  pl.KG = taps * pl.GS + 1;
  memset(&pl.k, 0, sizeof(pl.k));
  pl.k.g = k;
  int nl = 0;
  for (int uy = 0; uy < k.ay.nu; ++uy)
    for (int ux = 0; ux < k.ax.nu; ++ux) {
      int gs = 0;
      for (int s = 0; s < k.nseg; ++s) {
        const Seg& sg = k.seg[s];
        const int step = pl.vec;
        for (int c = 0; c < sg.C; c += step) {
          if (nl >= TPP_MAX_LOADS) return pl;
          TppLoad& L = pl.k.ld[nl++];
          L.ptr = sg.ptr; L.sub = sg.sub; L.C = sg.C; L.c = c; L.bcast = sg.bcast;
          L.dy = uy * k.ay.iu + k.ay.i0; L.dx = ux * k.ax.iu + k.ax.i0;
          L.row = ((uy * k.ax.nu + ux) * pl.GS + gs + c / 4) * 4 + (c % 4);
        }
        gs += (sg.C + 3) / 4;
      }
    }
  pl.nl = nl;
  if (nl * pl.vec * pl.n > 128) return pl;
  // instantiated (NL, VEC, N): scalar sources into 16 channels (level-0 convs) and
  // vector sources into <= 4 channels (final conv, 4->4 deconv)
  const bool inst = (pl.vec == 1 && pl.n == 16 && nl >= 1 && nl <= 8) ||
                    (pl.vec == 4 && pl.n == 3 && (nl == 9 || nl <= 4)) ||
                    (pl.vec == 4 && pl.n == 4 && nl >= 1 && nl <= 4);
  if (!inst) return pl;
  pl.k.nl = nl;
  pl.k.rows = pl.KG * 4;
  pl.k.ldw = (k.Cout + 3) / 4 * 4;
  pl.k.bias_row = (pl.KG - 1) * 4;
  long long want = (long long)sm_count() * 6;
  const long long max_split = ((long long)k.M + TPP_THREADS * 4 - 1) / (TPP_THREADS * 4);
  if (want > max_split) want = max_split;
  if (want < 1) want = 1;
  pl.nsplit = (int)want;
  // the 9-load tile (final conv: 36 channels -> 3) needs ~190 registers = 8 warps per SM; three blocks of 3
  // loads each run at 4x the occupancy and re-read only the 3-channel gradient
  pl.ksplit = (pl.vec == 4 && pl.n == 3 && nl == 9) ? 3 : 1;
  pl.ok = true;
  return pl;
}

bool wgrad_tpp_applicable(const GConvK& k) { return tpp_plan(k).ok; }

size_t wgrad_tpp_ws_floats(const GConvK& k) {
  TppPlan pl = tpp_plan(k);
  return pl.ok ? (size_t)pl.nsplit * pl.ksplit * pl.k.rows * pl.k.ldw : 0;
}

int launch_wgrad_tpp(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  TppPlan pl = tpp_plan(k);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "wgrad_tpp not applicable");
  w->g = k; w->GS = pl.GS; w->KG = pl.KG; w->ld = pl.k.ldw; w->nsplit = pl.nsplit * pl.ksplit; w->pix_per_split = 0;
  *KD_pad = (size_t)pl.k.rows;
  const dim3 grid(pl.nsplit, pl.ksplit);
#define NLT_TPP(NL_, V_, N_) wgrad_tpp_kernel<NL_, V_, N_><<<grid, TPP_THREADS, 0, st>>>(pl.k, G, ws)
  if (pl.vec == 1) {
    switch (pl.nl) {
      case 1: NLT_TPP(1, 1, 16); break; case 2: NLT_TPP(2, 1, 16); break; case 3: NLT_TPP(3, 1, 16); break;
      case 4: NLT_TPP(4, 1, 16); break; case 5: NLT_TPP(5, 1, 16); break; case 6: NLT_TPP(6, 1, 16); break;
      case 7: NLT_TPP(7, 1, 16); break; default: NLT_TPP(8, 1, 16); break;
    }
  } else if (pl.n == 3) {
    switch (pl.nl / pl.ksplit) {
      case 1: NLT_TPP(1, 4, 3); break; case 2: NLT_TPP(2, 4, 3); break; case 3: NLT_TPP(3, 4, 3); break;
      case 4: NLT_TPP(4, 4, 3); break; default: NLT_TPP(9, 4, 3); break;
    }
  } else {
    switch (pl.nl) {
      case 1: NLT_TPP(1, 4, 4); break; case 2: NLT_TPP(2, 4, 4); break; case 3: NLT_TPP(3, 4, 4); break;
      default: NLT_TPP(4, 4, 4); break;
    }
  }
#undef NLT_TPP
  NLT_CUDA_LAUNCH_CHECK("wgrad_tpp_kernel");
  return NLT_OK;
}

int launch_wgrad_small(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  WsPlan pl;
  if (!ws_plan(k, pl)) return set_err(NLT_ERR_INVALID, "wgrad_small not applicable");
  w->g = k; w->GS = pl.GS; w->KG = pl.KG; w->ld = pl.ld; w->nsplit = pl.nsplit; w->pix_per_split = pl.pps;
  *KD_pad = pl.KD_pad;
  const unsigned grid = pl.nsplit;
  const bool rows = opt(Opt::WGRAD_ROWS) == 1 && wgrad_rows_ok(k, G);   // option "wgrad_rows"; 0: flat-pixel form
  const uint32_t cpr = ((uint32_t)k.ax.nt + WR_CHUNK - 1) / WR_CHUNK;
  const uint32_t nchunks = (uint32_t)k.N * (uint32_t)k.ay.nt * cpr;
  // P <= 2 wants occupancy (128 registers, 4 CTAs per SM), the wide
  // P >= 4 tiles want more pixels in flight instead (they spill below ~220 registers)
#define NLT_WS(NQ_, P_)                                                                                        \
  do {                                                                                                         \
    constexpr int U0 = (P_ == 1 ? 8 : P_ == 2 ? 4 : 2);                                                        \
    if (rows)                                                                                                  \
      wgrad_rows_kernel<NQ_, P_, (P_ <= 2 ? U0 : 2 * U0), (P_ <= 2 ? 4 : 1)>                                   \
          <<<grid, WS_THREADS, 0, st>>>(*w, G, ws, cpr, nchunks);                                              \
    else                                                                                                       \
      wgrad_small_kernel<NQ_, P_, U0><<<grid, WS_THREADS, 0, st>>>(*w, G, ws);                                 \
  } while (0)
  if (pl.nq == 8) {
    if (pl.p == 1) NLT_WS(8, 1); else if (pl.p == 2) NLT_WS(8, 2); else if (pl.p == 4) NLT_WS(8, 4); else NLT_WS(8, 5);
  } else if (pl.nq == 4) {
    if (pl.p == 1) NLT_WS(4, 1); else if (pl.p == 2) NLT_WS(4, 2); else if (pl.p == 4) NLT_WS(4, 4); else NLT_WS(4, 5);
  } else if (pl.nq == 2) {
    if (pl.p == 1) NLT_WS(2, 1); else NLT_WS(2, 2);
  } else {
    if (pl.p == 1) NLT_WS(1, 1); else NLT_WS(1, 2);
  }
#undef NLT_WS
  NLT_CUDA_LAUNCH_CHECK("wgrad_small_kernel");
  return NLT_OK;
}

}  // namespace nlt
