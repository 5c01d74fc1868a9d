// Generalised convolution (SIMT fp32 path) for the NLT UV-space network.
//
// One kernel family covers Conv2D 'same', Conv2DTranspose 'same'
// (reference: nlt/networks/elements.py:26-39) and both of their input
// gradients, over a virtual channel-concat of up to 4 NHWC sources (the
// tf.concat / tf.reduce_mean glue of nlt/models/nlt.py:161-190 is never
// materialised).  Bias, activation, gradient accumulation (beta) and the
// activation-derivative mask are fused into the epilogue.
//
// Bound: for Cout <= 16 these layers are HBM-bound (AI ~ 4-7 FLOP/B); for
// larger Cout this fp32-FFMA path is FMA-bound and the wgmma path
// (nlt_tc.cu) takes over where the shape allows.
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include "nlt_common.cuh"

namespace nlt {

thread_local char g_err[512] = "";
unsigned long long g_launches = 0;

int set_err(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  static int n[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (n[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}

int build_phases(const nlt_gconv_desc* d, GConvK* out, int* nphase, bool allow_d2s) {
  NLT_CHECK_ARG(d != nullptr, "null descriptor");
  NLT_CHECK_ARG(d->N > 0 && d->Hin > 0 && d->Win > 0 && d->Hout > 0 && d->Wout > 0,
                "bad geometry N=%d in=%dx%d out=%dx%d", d->N, d->Hin, d->Win, d->Hout, d->Wout);
  NLT_CHECK_ARG(d->kh > 0 && d->kw > 0 && d->stride > 0 && d->kh <= 16 && d->kw <= 16 && d->stride <= 4,
                "bad kernel %dx%d stride %d", d->kh, d->kw, d->stride);
  NLT_CHECK_ARG(d->pad_t >= 0 && d->pad_l >= 0, "negative padding");
  NLT_CHECK_ARG(d->nseg >= 1 && d->nseg <= NLT_MAX_SEG, "nseg=%d out of range", d->nseg);
  NLT_CHECK_ARG(d->Cout > 0 && d->w != nullptr, "bad Cout/weights");
  NLT_CHECK_ARG((long long)d->N * d->Hout * d->Wout < (1ll << 31) &&
                (long long)d->N * d->Hin * d->Win < (1ll << 31), "too many pixels for 32-bit pixel index");
  GConvK base;
  memset(&base, 0, sizeof(base));
  base.N = d->N; base.Hin = d->Hin; base.Win = d->Win; base.Hout = d->Hout; base.Wout = d->Wout;
  base.kw = d->kw; base.nseg = d->nseg; base.Cout = d->Cout; base.w = d->w;
  base.wt = d->w_tap_stride; base.wc = d->w_c_stride; base.wn = d->w_n_stride;
  int coff = 0;
  for (int s = 0; s < d->nseg; ++s) {
    NLT_CHECK_ARG(d->seg_ptr[s] != nullptr && d->seg_C[s] > 0, "segment %d null/empty", s);
    Seg& sg = base.seg[s];
    sg.ptr = d->seg_ptr[s]; sg.sub = d->seg_sub[s]; sg.C = d->seg_C[s]; sg.coff = coff;
    sg.bcast = d->seg_bcast[s] ? 1 : 0;
    sg.vec = (sg.C % 4 == 0) && aligned16(sg.ptr) && (sg.sub == nullptr || aligned16(sg.sub));
    coff += sg.C;
  }
  const int s = d->stride;
  int np = 0;
  base.cout_true = d->Cout;
  const bool d2s = allow_d2s && d->transposed && s > 1 && d->kh == s && d->kw == s && d->pad_t == 0 &&
                   d->pad_l == 0 && d->Hout == d->Hin * s && d->Wout == d->Win * s && d->Cout % 4 == 0;
  if (d2s) {
    GConvK k = base;
    k.d2s = 1; k.d2s_s = s; k.Cout = s * s * d->Cout;
    k.ay = AxisMap{0, 1, d->Hin, 1, 0, 0, 0, 0, 1, d->Hin};
    k.ax = AxisMap{0, 1, d->Win, 1, 0, 0, 0, 0, 1, d->Win};
    out[np++] = k;
  } else if (!d->transposed) {
    GConvK k = base;
    k.ay = AxisMap{0, 1, d->Hout, s, 1, -d->pad_t, 0, 1, d->kh, d->Hin};
    k.ax = AxisMap{0, 1, d->Wout, s, 1, -d->pad_l, 0, 1, d->kw, d->Win};
    out[np++] = k;
  } else {
    for (int py = 0; py < s; ++py) {
      for (int px = 0; px < s; ++px) {
        if (py >= d->Hout || px >= d->Wout) continue;
        GConvK k = base;
        const int dy0 = (py + d->pad_t) % s, dx0 = (px + d->pad_l) % s;
        const int nuy = dy0 < d->kh ? (d->kh - dy0 + s - 1) / s : 0;
        const int nux = dx0 < d->kw ? (d->kw - dx0 + s - 1) / s : 0;
        k.ay = AxisMap{py, s, (d->Hout - py + s - 1) / s, 1, -1, (py + d->pad_t - dy0) / s, dy0, s, nuy, d->Hin};
        k.ax = AxisMap{px, s, (d->Wout - px + s - 1) / s, 1, -1, (px + d->pad_l - dx0) / s, dx0, s, nux, d->Win};
        if (nuy == 0 || nux == 0) { k.ay.nu = 0; k.ax.nu = 0; }
        out[np++] = k;
      }
    }
  }
  for (int i = 0; i < np; ++i) {
    GConvK& k = out[i];
    k.M = (uint32_t)((long long)k.N * k.ay.nt * k.ax.nt);
    k.div_x = make_fastdiv((uint32_t)k.ax.nt);
    k.div_yx = make_fastdiv((uint32_t)(k.ay.nt * k.ax.nt));
    k.div_ct = make_fastdiv((uint32_t)(k.cout_true > 0 ? k.cout_true : 1));
    k.div_s = make_fastdiv((uint32_t)(k.d2s ? k.d2s_s : 1));
  }
  *nphase = np;
  return NLT_OK;
}

// -----------------------------------------------------------------------------
// forward / dgrad kernel
// -----------------------------------------------------------------------------
constexpr int TK = 16;       // K-chunk (channels of one tap of one segment)
constexpr int SA = TK + 4;   // smem row stride of the A tile (odd # of 16B chunks -> conflict-free LDS.128)

struct ChunkIt {
  int uy, ux, s, c0;
};

__device__ __forceinline__ void chunk_advance(const GConvK& g, ChunkIt& it) {
  it.c0 += TK;
  if (it.c0 >= g.seg[it.s].C) {
    it.c0 = 0;
    if (++it.s >= g.nseg) {
      it.s = 0;
      if (++it.ux >= g.ax.nu) { it.ux = 0; ++it.uy; }
    }
  }
}


template <int TM, int TN, int RM, int RN, int NTHR>
__global__ void __launch_bounds__(NTHR, 3)   // 3 CTAs per SM measured best (2: latency-bound, 4: spills)
gconv_kernel(const GConvK g, const float* __restrict__ bias, const int act, const float beta,
             const float* __restrict__ mask_y, const int mask_act, float* __restrict__ out) {
  constexpr int TNT = TN / RN;          // threads along n
  constexpr int TMT = NTHR / TNT;       // threads along m
  static_assert(TMT * RM == TM, "tile/thread mismatch");
  static_assert(RN % 4 == 0 && RM % 2 == 0, "thread tile");
  constexpr int LA = TM * (TK / 4) / NTHR;  // float4 A loads per thread per chunk
  static_assert(LA * NTHR == TM * (TK / 4), "A loader mismatch");
  constexpr int LB = (TK * TN + NTHR - 1) / NTHR;
  constexpr int ROWS_PER_PASS = NTHR / 4;

  __shared__ __align__(16) float As[2][TM * SA];
  __shared__ __align__(16) float Bs[2][TK * TN];

  const int tid = threadIdx.x;
  const int tn = tid % TNT, tm = tid / TNT;
  const uint32_t m0 = blockIdx.x * TM;
  const int n0 = blockIdx.y * TN;

  // ---- per-thread loader rows (fixed over the K loop) ----
  const int c4 = tid & 3;
  int ln[LA], lby[LA], lbx[LA];
#pragma unroll
  for (int i = 0; i < LA; ++i) {
    const uint32_t m = m0 + (tid >> 2) + i * ROWS_PER_PASS;
    if (m < g.M) {
      int n, ty, tx;
      decode_pixel(g, m, n, ty, tx);
      ln[i] = n; lby[i] = ty * g.ay.it + g.ay.i0; lbx[i] = tx * g.ax.it + g.ax.i0;
    } else {
      ln[i] = -1; lby[i] = 0; lbx[i] = 0;
    }
  }

  int nchunk_per_tap = 0;
  for (int s = 0; s < g.nseg; ++s) nchunk_per_tap += (g.seg[s].C + TK - 1) / TK;
  const int nchunks = g.ay.nu * g.ax.nu * nchunk_per_tap;

  float4 ra[LA];
  float rb[LB];

  auto load_chunk = [&](const ChunkIt& it) {
    const Seg sg = g.seg[it.s];
    const int c = it.c0 + c4 * 4;
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int iy = lby[i] + it.uy * g.ay.iu;
      const int ix = lbx[i] + it.ux * g.ax.iu;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ln[i] >= 0 && (unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win && c < sg.C) {
        const size_t pix = ((size_t)(sg.bcast ? 0 : ln[i]) * g.Hin + iy) * g.Win + ix;
        const size_t off = pix * sg.C + c;
        if (sg.vec) {
          v = ld4(sg.ptr + off);
          if (sg.sub) { const float4 u = ld4(sg.sub + off); v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w; }
        } else {
          float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (c + e < sg.C) {
              t[e] = __ldg(sg.ptr + off + e);
              if (sg.sub) t[e] -= __ldg(sg.sub + off + e);
            }
          v = make_float4(t[0], t[1], t[2], t[3]);
        }
      }
      ra[i] = v;
    }
    const int tap = (g.ay.d0 + g.ay.ds * it.uy) * g.kw + (g.ax.d0 + g.ax.ds * it.ux);
    const float* wrow = g.w + (long long)(sg.coff + it.c0) * g.wc;
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int idx = tid + i * NTHR;
      const int kk = idx / TN, nn = n0 + idx % TN;
      float v = 0.f;
      if (idx < TK * TN && it.c0 + kk < sg.C && nn < g.Cout) {
        int t = tap, n = nn;
        if (g.d2s) { t = nn / g.cout_true; n = nn - t * g.cout_true; }
        v = __ldg(wrow + (long long)t * g.wt + (long long)kk * g.wc + (long long)n * g.wn);
      }
      rb[i] = v;
    }
  };
  auto store_chunk = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int row = (tid >> 2) + i * ROWS_PER_PASS;
      *reinterpret_cast<float4*>(&As[buf][row * SA + c4 * 4]) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int idx = tid + i * NTHR;
      if (idx < TK * TN) Bs[buf][idx] = rb[i];
    }
  };

  float acc[RM][RN];
#pragma unroll
  for (int i = 0; i < RM; ++i)
#pragma unroll
    for (int j = 0; j < RN; ++j) acc[i][j] = 0.f;

  ChunkIt it{0, 0, 0, 0};
  if (nchunks > 0) load_chunk(it);
  for (int ch = 0; ch < nchunks; ++ch) {
    const int buf = ch & 1;
    store_chunk(buf);
    __syncthreads();
    if (ch + 1 < nchunks) {
      chunk_advance(g, it);
      load_chunk(it);
    }
    const float* as = As[buf];
    const float* bs = Bs[buf];
#pragma unroll
    for (int kq = 0; kq < TK / 4; ++kq) {
      float4 a[RM];
#pragma unroll
      for (int i = 0; i < RM; ++i)
        a[i] = *reinterpret_cast<const float4*>(&as[(tm + i * TMT) * SA + kq * 4]);
      float b[4][RN];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int jg = 0; jg < RN / 4; ++jg) {
          const float4 t = *reinterpret_cast<const float4*>(&bs[(kq * 4 + kk) * TN + tn * 4 + jg * TNT * 4]);
          b[kk][jg * 4 + 0] = t.x; b[kk][jg * 4 + 1] = t.y; b[kk][jg * 4 + 2] = t.z; b[kk][jg * 4 + 3] = t.w;
        }
#pragma unroll
      for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < RN; ++j) {
          acc[i][j] = fmaf(a[i].x, b[0][j], acc[i][j]);
          acc[i][j] = fmaf(a[i].y, b[1][j], acc[i][j]);
          acc[i][j] = fmaf(a[i].z, b[2][j], acc[i][j]);
          acc[i][j] = fmaf(a[i].w, b[3][j], acc[i][j]);
        }
    }
    // the next iteration writes the other buffer; a thread can be at most one
    // barrier ahead, so buffer `buf` is not overwritten before everyone left it
  }

  // ---- epilogue: two pixel rows at a time; all read-modify-write operands (old
  // gradient for beta, saved activation for the mask) are loaded as one batch
  // before the first store so their latencies overlap ----
  const bool vec_out = (g.cout_true % 4 == 0) && aligned16(out) && (mask_y == nullptr || aligned16(mask_y));
  constexpr int NG = RN / 4;
#pragma unroll
  for (int i0 = 0; i0 < RM; i0 += 2) {
    size_t ob[2][NG];
    int cbv[2][NG];
    bool live[2][NG];
    float4 oldv[2][NG], yv[2][NG];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint32_t m = m0 + tm + (i0 + r) * TMT;
      int n = 0, ty = 0, tx = 0;
      const bool mok = m < g.M;
      if (mok) decode_pixel(g, m, n, ty, tx);
      const int oy0 = g.d2s ? ty * g.d2s_s : g.ay.o0 + g.ay.os * ty;
      const int ox0 = g.d2s ? tx * g.d2s_s : g.ax.o0 + g.ax.os * tx;
#pragma unroll
      for (int jg = 0; jg < NG; ++jg) {
        const int nb = n0 + tn * 4 + jg * TNT * 4;
        int cb = nb, oy = oy0, ox = ox0;     // cb: channel inside the destination pixel
        if (g.d2s) {
          const int t = nb / g.cout_true;
          cb = nb - t * g.cout_true;
          const int dy = t / g.d2s_s;
          oy += dy; ox += t - dy * g.d2s_s;
        }
        live[r][jg] = mok && nb < g.Cout;
        cbv[r][jg] = cb;
        ob[r][jg] = (((size_t)n * g.Hout + oy) * g.Wout + ox) * g.cout_true + cb;
        oldv[r][jg] = make_float4(0.f, 0.f, 0.f, 0.f);
        yv[r][jg] = make_float4(1.f, 1.f, 1.f, 1.f);
        if (live[r][jg] && vec_out) {
          if (beta != 0.f) oldv[r][jg] = *reinterpret_cast<const float4*>(out + ob[r][jg]);
          if (mask_y != nullptr) yv[r][jg] = ld4(mask_y + ob[r][jg]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int jg = 0; jg < NG; ++jg) {
        if (!live[r][jg]) continue;
        const int cb = cbv[r][jg];
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float t = acc[i0 + r][jg * 4 + e];
          if (bias != nullptr && cb + e < g.cout_true) t += __ldg(bias + cb + e);
          v[e] = act_fwd(t, act);
        }
        if (vec_out) {
          const float4 o = oldv[r][jg], y = yv[r][jg];
          v[0] += beta * o.x; v[1] += beta * o.y; v[2] += beta * o.z; v[3] += beta * o.w;
          if (mask_y != nullptr) {
            v[0] *= act_bwd_from_y(y.x, mask_act); v[1] *= act_bwd_from_y(y.y, mask_act);
            v[2] *= act_bwd_from_y(y.z, mask_act); v[3] *= act_bwd_from_y(y.w, mask_act);
          }
          *reinterpret_cast<float4*>(out + ob[r][jg]) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (cb + e >= g.cout_true) continue;
            float t = v[e];
            if (beta != 0.f) t += beta * out[ob[r][jg] + e];
            if (mask_y != nullptr) t *= act_bwd_from_y(__ldg(mask_y + ob[r][jg] + e), mask_act);
            out[ob[r][jg] + e] = t;
          }
        }
      }
  }
}

template <int TM, int TN, int RM, int RN>
static int launch_fwd(const GConvK& k, const float* bias, int act, float beta, const float* mask_y,
                      int mask_act, float* out, cudaStream_t st) {
  constexpr int NTHR = 128;
  dim3 grid((k.M + TM - 1) / TM, (k.Cout + TN - 1) / TN);
  gconv_kernel<TM, TN, RM, RN, NTHR><<<grid, NTHR, 0, st>>>(k, bias, act, beta, mask_y, mask_act, out);
  NLT_CUDA_LAUNCH_CHECK("gconv_kernel");
  return NLT_OK;
}

// -----------------------------------------------------------------------------
// wgrad kernel:  ws[split][k][n] = sum_{p in split} A[p,k] * G[p,n]
// k enumerates "k-groups" of 4 channels: kg = (uy*nux + ux)*GS + gs, plus one
// trailing bias group whose A value is (1,0,0,0).
// -----------------------------------------------------------------------------
constexpr int WTP = 16;  // pixels per smem stage

template <int TKG, int TN, int RK, int RN, int NTHR>
__global__ void __launch_bounds__(NTHR)
gconv_wgrad_kernel(const WgradK w, const float* __restrict__ G, float* __restrict__ ws) {
  constexpr int TKD = TKG * 4;
  constexpr int TNT = TN / RN, TKT = TKD / RK;
  static_assert(TNT * TKT == NTHR, "thread layout");
  static_assert(NTHR % TKG == 0, "loader layout");
  static_assert(RK % 4 == 0 && RN % 4 == 0, "vector tiles");
  constexpr int PP = NTHR / TKG;                 // pixels per loader pass
  constexpr int LA = WTP / PP;                   // A float4 per thread per stage
  static_assert(LA * PP == WTP, "A stage");
  constexpr int GV = TN / 4;                     // float4 per pixel of G
  constexpr int LG = (WTP * GV + NTHR - 1) / NTHR;

  __shared__ __align__(16) float As[2][WTP * TKD];
  __shared__ __align__(16) float Gs[2][WTP * TN];

  const GConvK& g = w.g;
  const int tid = threadIdx.x;
  const int tn = tid % TNT, tk = tid / TNT;
  const int kg0 = blockIdx.x * TKG;
  const int n0 = blockIdx.y * TN;
  const uint32_t p_begin = blockIdx.z * w.pix_per_split;
  const uint32_t p_end = min(g.M, p_begin + w.pix_per_split);

  // loader: fixed k-group per thread
  const int lkg = tid % TKG, lp0 = tid / TKG;
  int uy, ux, s, c;
  decode_kgroup(w, kg0 + lkg, uy, ux, s, c);
  Seg sg;
  sg.ptr = nullptr; sg.sub = nullptr; sg.C = 0; sg.coff = 0; sg.bcast = 0; sg.vec = 0;
  if (s >= 0) sg = g.seg[s];
  const int duy = uy * g.ay.iu + g.ay.i0, dux = ux * g.ax.iu + g.ax.i0;
  const bool g_vec = (g.Cout % 4 == 0) && aligned16(G);

  float4 ra[LA];
  float4 rg[LG];

  auto load_stage = [&](uint32_t pbase) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const uint32_t m = pbase + lp0 + i * PP;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < p_end && s != -2) {
        if (s == -1) {
          v.x = 1.f;
        } else {
          int n, ty, tx;
          decode_pixel(g, m, n, ty, tx);
          const int iy = ty * g.ay.it + duy, ix = tx * g.ax.it + dux;
          if ((unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win) {
            const size_t off = (((size_t)(sg.bcast ? 0 : n) * g.Hin + iy) * g.Win + ix) * sg.C + c;
            if (sg.vec) {
              v = ld4(sg.ptr + off);
              if (sg.sub) { const float4 u = ld4(sg.sub + off); v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w; }
            } else {
              float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (c + e < sg.C) {
                  t[e] = __ldg(sg.ptr + off + e);
                  if (sg.sub) t[e] -= __ldg(sg.sub + off + e);
                }
              v = make_float4(t[0], t[1], t[2], t[3]);
            }
          }
        }
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < LG; ++i) {
      const int idx = tid + i * NTHR;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < WTP * GV) {
        const int pl = idx / GV, n4 = idx % GV;
        const uint32_t m = pbase + pl;
        const int nb = n0 + n4 * 4;
        if (m < p_end && nb < g.Cout) {
          int n, ty, tx;
          decode_pixel(g, m, n, ty, tx);
          const int oy = g.ay.o0 + g.ay.os * ty, ox = g.ax.o0 + g.ax.os * tx;
          const size_t off = (((size_t)n * g.Hout + oy) * g.Wout + ox) * g.Cout + nb;
          if (g_vec) {
            v = ld4(G + off);
          } else {
            float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (nb + e < g.Cout) t[e] = __ldg(G + off + e);
            v = make_float4(t[0], t[1], t[2], t[3]);
          }
        }
      }
      rg[i] = v;
    }
  };
  auto store_stage = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i)
      *reinterpret_cast<float4*>(&As[buf][(lp0 + i * PP) * TKD + lkg * 4]) = ra[i];
#pragma unroll
    for (int i = 0; i < LG; ++i) {
      const int idx = tid + i * NTHR;
      if (idx < WTP * GV) *reinterpret_cast<float4*>(&Gs[buf][idx * 4]) = rg[i];
    }
  };

  float acc[RK][RN];
#pragma unroll
  for (int i = 0; i < RK; ++i)
#pragma unroll
    for (int j = 0; j < RN; ++j) acc[i][j] = 0.f;

  const int nstage = p_end > p_begin ? (int)((p_end - p_begin + WTP - 1) / WTP) : 0;
  if (nstage > 0) load_stage(p_begin);
  for (int st = 0; st < nstage; ++st) {
    const int buf = st & 1;
    store_stage(buf);
    __syncthreads();
    if (st + 1 < nstage) load_stage(p_begin + (uint32_t)(st + 1) * WTP);
    const float* as = As[buf];
    const float* gs = Gs[buf];
#pragma unroll
    for (int p = 0; p < WTP; ++p) {
      float a[RK], b[RN];
#pragma unroll
      for (int ig = 0; ig < RK / 4; ++ig) {
        const float4 t = *reinterpret_cast<const float4*>(&as[p * TKD + tk * 4 + ig * TKT * 4]);
        a[ig * 4 + 0] = t.x; a[ig * 4 + 1] = t.y; a[ig * 4 + 2] = t.z; a[ig * 4 + 3] = t.w;
      }
#pragma unroll
      for (int jg = 0; jg < RN / 4; ++jg) {
        const float4 t = *reinterpret_cast<const float4*>(&gs[p * TN + tn * 4 + jg * TNT * 4]);
        b[jg * 4 + 0] = t.x; b[jg * 4 + 1] = t.y; b[jg * 4 + 2] = t.z; b[jg * 4 + 3] = t.w;
      }
#pragma unroll
      for (int i = 0; i < RK; ++i)
#pragma unroll
        for (int j = 0; j < RN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }

  // partial tile -> workspace [split][KGpad*4][ld]
  const size_t KD_pad = (size_t)gridDim.x * TKD;
  float* wsp = ws + ((size_t)blockIdx.z * KD_pad + (size_t)kg0 * 4) * w.ld;
#pragma unroll
  for (int ig = 0; ig < RK / 4; ++ig)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int krow = tk * 4 + ig * TKT * 4 + e;
#pragma unroll
      for (int jg = 0; jg < RN / 4; ++jg) {
        const int nb = n0 + tn * 4 + jg * TNT * 4;
        if (nb < w.ld)
          *reinterpret_cast<float4*>(&wsp[(size_t)krow * w.ld + nb]) =
              make_float4(acc[ig * 4 + e][jg * 4 + 0], acc[ig * 4 + e][jg * 4 + 1],
                          acc[ig * 4 + e][jg * 4 + 2], acc[ig * 4 + e][jg * 4 + 3]);
      }
    }
}

// second stage: fixed-order sum over splits, scatter to the weight layout.
// 256 threads = 32 split lanes x 8 outputs: every output is summed by 32 lanes (each over its own residue
// class of splits, 2 independent chains), then combined in a fixed order through smem -> deterministic,
// and the latency of walking up to ~1000 partials is spread over 32 lanes instead of one thread.
__global__ void __launch_bounds__(256)
gconv_wgrad_reduce_kernel(const WgradK w, const float* __restrict__ ws, size_t KD_pad,
                          float* __restrict__ dW, float* __restrict__ db, int acc_w, int acc_b) {
  __shared__ float red[32][9];
  const int lane_o = threadIdx.x & 7, lane_s = threadIdx.x >> 3;
  const size_t total = (size_t)w.KG * 4 * w.g.Cout;
  const size_t stride = KD_pad * w.ld;
  for (size_t base = (size_t)blockIdx.x * 8; base < total; base += (size_t)gridDim.x * 8) {
    const size_t idx = base + lane_o;
    float* dst = nullptr;
    int accumulate = acc_w, ntaps_sum = 1, n = 0, k = 0;
    if (idx < total) {
      n = (int)(idx % w.g.Cout);
      k = (int)(idx / w.g.Cout);
      const int kg = k >> 2, e = k & 3;
      int uy, ux, s, c;
      decode_kgroup(w, kg, uy, ux, s, c);
      if (s == -1) {
        // d2s bias: one output channel collects its column in every tap
        if (e == 0 && db != nullptr && (!w.g.d2s || n < w.g.cout_true)) {
          dst = db + n; accumulate = acc_b;
          if (w.g.d2s) ntaps_sum = w.g.d2s_s * w.g.d2s_s;
        }
      } else if (s >= 0 && c + e < w.g.seg[s].C) {
        int tap = (w.g.ay.d0 + w.g.ay.ds * uy) * w.g.kw + (w.g.ax.d0 + w.g.ax.ds * ux), nn = n;
        if (w.g.d2s) { tap = n / w.g.cout_true; nn = n - tap * w.g.cout_true; }
        dst = dW + (long long)tap * w.g.wt + (long long)(w.g.seg[s].coff + c + e) * w.g.wc + (long long)nn * w.g.wn;
      }
    }
    float part = 0.f;
    if (dst != nullptr) {
      for (int tp = 0; tp < ntaps_sum; ++tp) {
        const float* src = ws + (size_t)k * w.ld + n + tp * w.g.cout_true;
        float s0 = 0.f, s1 = 0.f;
        int sp = lane_s;
        for (; sp + 32 < w.nsplit; sp += 64) { s0 += src[(size_t)sp * stride]; s1 += src[(size_t)(sp + 32) * stride]; }
        if (sp < w.nsplit) s0 += src[(size_t)sp * stride];
        part += s0 + s1;
      }
    }
    red[lane_s][lane_o] = part;
    __syncthreads();
    if (lane_s == 0 && dst != nullptr) {
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) sum += red[i][lane_o];
      *dst = accumulate ? (*dst + sum) : sum;
    }
    __syncthreads();
  }
}

// Few partials (the wgmma wgrad of the deep levels: 2-32 splits of a [K_d x N] matrix of up to 4096 x 256):
// one thread per output, splits summed serially in fixed order.  The 32-lane form above keeps 2 of its 32 split
// lanes busy there, tens of microseconds per launch for 2 MB of partials.
__global__ void __launch_bounds__(256)
gconv_wgrad_reduce_flat_kernel(const WgradK w, const float* __restrict__ ws, size_t KD_pad,
                               float* __restrict__ dW, float* __restrict__ db, int acc_w, int acc_b) {
  const size_t total = (size_t)w.KG * 4 * w.g.Cout;
  const size_t stride = KD_pad * w.ld;
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx % w.g.Cout);
  const int k = (int)(idx / w.g.Cout);
  const int kg = k >> 2, e = k & 3;
  int uy, ux, s, c;
  decode_kgroup(w, kg, uy, ux, s, c);
  float* dst = nullptr;
  int accumulate = acc_w, ntaps_sum = 1;
  if (s == -1) {
    if (e == 0 && db != nullptr && (!w.g.d2s || n < w.g.cout_true)) {
      dst = db + n; accumulate = acc_b;
      if (w.g.d2s) ntaps_sum = w.g.d2s_s * w.g.d2s_s;
    }
  } else if (s >= 0 && c + e < w.g.seg[s].C) {
    int tap = (w.g.ay.d0 + w.g.ay.ds * uy) * w.g.kw + (w.g.ax.d0 + w.g.ax.ds * ux), nn = n;
    if (w.g.d2s) { tap = n / w.g.cout_true; nn = n - tap * w.g.cout_true; }
    dst = dW + (long long)tap * w.g.wt + (long long)(w.g.seg[s].coff + c + e) * w.g.wc + (long long)nn * w.g.wn;
  }
  if (dst == nullptr) return;
  float sum = 0.f;
  for (int tp = 0; tp < ntaps_sum; ++tp) {
    const float* src = ws + (size_t)k * w.ld + n + tp * w.g.cout_true;
#pragma unroll 4
    for (int sp = 0; sp < w.nsplit; ++sp) sum += __ldg(src + (size_t)sp * stride);
  }
  *dst = accumulate ? (*dst + sum) : sum;
}

struct WgradPlan {
  int tkg, tn, nthr;
  int kd_tiles, n_tiles, nsplit;
  uint32_t pix_per_split;
  size_t KD_pad;
  int ld, GS, KG;
  size_t ws_floats;
};

static WgradPlan plan_wgrad(const GConvK& k) {
  WgradPlan p;
  p.GS = 0;
  for (int s = 0; s < k.nseg; ++s) p.GS += (k.seg[s].C + 3) / 4;
  p.KG = k.ay.nu * k.ax.nu * p.GS + 1;
  p.tkg = 32;
  p.tn = k.Cout > 32 ? 64 : k.Cout > 16 ? 32 : k.Cout > 8 ? 16 : k.Cout > 4 ? 8 : 4;
  p.nthr = p.tn >= 16 ? 128 : p.tn == 8 ? 64 : 32;
  p.kd_tiles = (p.KG + p.tkg - 1) / p.tkg;
  p.n_tiles = (k.Cout + p.tn - 1) / p.tn;
  p.ld = (k.Cout + 3) / 4 * 4;
  p.KD_pad = (size_t)p.kd_tiles * p.tkg * 4;
  // enough CTAs to fill every SM a few times over, at least 64 pixels per CTA
  const long long tiles = (long long)p.kd_tiles * p.n_tiles;
  long long want = ((long long)sm_count() * 8 + tiles - 1) / tiles;
  long long max_split = ((long long)k.M + 63) / 64;
  if (want > max_split) want = max_split;
  if (want < 1) want = 1;
  if (want > 512) want = 512;
  uint32_t pps = (uint32_t)(((long long)k.M + want - 1) / want);
  pps = (pps + WTP - 1) / WTP * WTP;
  p.pix_per_split = pps;
  p.nsplit = (int)((k.M + pps - 1) / pps);
  if (p.nsplit < 1) p.nsplit = 1;
  p.ws_floats = (size_t)p.nsplit * p.KD_pad * p.ld;
  return p;
}

}  // namespace nlt

using namespace nlt;

namespace nlt {
// launches per kernel label (the string literal of NLT_CUDA_LAUNCH_CHECK; about 60 labels in the library)
static std::mutex g_kl_mutex;
static const char* g_kl_name[128];
static uint64_t g_kl_count[128];
static int g_kl_n = 0;
void count_launch(const char* what) {
  std::lock_guard<std::mutex> lock(g_kl_mutex);
  for (int i = 0; i < g_kl_n; ++i)
    if (g_kl_name[i] == what || strcmp(g_kl_name[i], what) == 0) { ++g_kl_count[i]; return; }
  if (g_kl_n < 128) { g_kl_name[g_kl_n] = what; g_kl_count[g_kl_n++] = 1; }
}

// ---- process-wide switches ----------------------------------------------------------------------------------------
// One row per option, in the order of enum Opt: the nlt_set_option name, the environment variable that gives its first
// value (or none), how that variable is read (CHAR: `val` when its first character is `ch`, else the default; ATOI:
// atoi), the default, and how a value v is stored, from the environment or from nlt_set_option (BOOL: v != 0; INT: v;
// NS: 2 if v == 2, else 1; TC: 0 if v == 0, 2 if v == 2, else 1).
enum class Parse { CHAR, ATOI };
enum class Store { BOOL, INT, NS, TC };
struct OptRow { const char *name, *env; Parse parse; char ch; int val, dflt; Store store; };
static const OptRow kOpts[] = {
    // 1: the wgmma 3xTF32 kernels where eligible; 0: the fp32-FMA kernels only; 2: the wgmma kernel for every shape it
    // can run, ahead of its size heuristics and of the stream kernels (A/B tests)
    {"tc", "NLT_DISABLE_TC", Parse::CHAR, '1', 0, 1, Store::TC},
    {"tc_wgrad", "NLT_DISABLE_TC_WGRAD", Parse::CHAR, '1', 0, 1, Store::BOOL},   // the same for weight gradients
    {"wgrad_rows", nullptr, Parse::CHAR, 0, 0, 1, Store::BOOL},   // row-run form of the warp-stream weight gradient
    {"tcs", "NLT_TCS", Parse::ATOI, 0, 0, 1, Store::BOOL},        // wgmma forward: A operand split in registers
    {"tc_rawhi", "NLT_TC_RAWHI", Parse::CHAR, '0', 0, 1, Store::BOOL},   // 3xTF32: hi truncated (1) or rounded (0)
    {"tc_split_waves", "NLT_TC_SPLIT_WAVES", Parse::CHAR, '1', 1, 0, Store::BOOL},   // see tc_plan
    {"pwx", "NLT_PWX", Parse::CHAR, '0', 0, 1, Store::BOOL},      // the kernels of nlt_pwx.cu (0: the general routes)
    {"pwmma", "NLT_PWMMA", Parse::CHAR, '0', 0, 1, Store::BOOL},  // depth-to-space input gradient on mma.sync (tc on)
    {"tiny", "NLT_TINY", Parse::CHAR, '0', 0, 1, Store::BOOL},    // the row-stream stencil kernel of nlt_tiny.cu
    {"dconv_cw", "NLT_DCONV_CW", Parse::CHAR, '0', 0, 1, Store::BOOL},   // wide stencil weights in constant memory
    // the wide stencil kernel ahead of the quad-per-thread one where both apply (16 / 8 outputs, K <= 32)
    {"dconv_wide_first", "NLT_DCONV_WIDE_FIRST", Parse::CHAR, '0', 0, 1, Store::BOOL},
    // staged-patch forward of the 2x2/s2 convs (nlt_pwx.cu).  H100, cfg4 step: the level-1/2 forward convs take
    // 0.87 ms less on the general kernels
    {"pf", "NLT_PF", Parse::CHAR, '1', 1, 0, Store::BOOL},
    {"pf_s1", "NLT_PF_S1", Parse::CHAR, '1', 1, 0, Store::BOOL},   // with pf: also the stride-1 16 -> 16 stencils
    // the pointwise depth-to-space kernel ahead of the wgmma kernel for the input gradients of 2x2/s2 convs from
    // 64-channel sources.  H100, cfg4 step: the wgmma kernel is faster there (level-3 input gradients 0.64 ms less)
    {"pwd2s_first", "NLT_PWD2S_FIRST", Parse::CHAR, '1', 1, 0, Store::BOOL},
    {"pf_ns", "NLT_PF_NS", Parse::CHAR, '2', 2, 1, Store::NS},     // threads per pixel of the staged-patch forward
    {"pwx_ns", "NLT_PWX_NS", Parse::CHAR, '2', 2, 1, Store::NS},   // ... and of the pointwise forward
    // outer-product weight gradients (nlt_wop.cu): 0 off; 1 the 4 -> 4 and 8 -> 8 stencils and the final 1x1 conv; 2
    // also the 16 -> 16 stencils and the up-convs, where they are slower than the staged-patch / wgmma kernels
    // (16 warps/SM at 128 registers cannot hide the load latency)
    {"wop", "NLT_WOP", Parse::ATOI, 0, 0, 1, Store::INT},
    {"dconv_wide", "NLT_DCONV_WIDE", Parse::ATOI, 0, 0, 1, Store::BOOL},   // wide stencil kernel, 16 outputs
    {"dconv_wide32", "NLT_DCONV_WIDE32", Parse::ATOI, 0, 0, 0, Store::INT},   // 32 outputs: 1 / 2 pixels per thread
    {"dconv_wide8", "NLT_DCONV_WIDE8", Parse::ATOI, 0, 0, 1, Store::INT},     // 8 outputs when > 0
};
static_assert(sizeof(kOpts) / sizeof(kOpts[0]) == (size_t)Opt::COUNT, "one row per option");
static int opt_value[(int)Opt::COUNT];
static bool opt_taken[(int)Opt::COUNT];   // the value has been read from the environment or set

static int opt_index(const char* name) {
  for (int i = 0; i < (int)Opt::COUNT; ++i)
    if (strcmp(kOpts[i].name, name) == 0) return i;
  return -1;
}

static void set_opt(int i, int v) {
  const Store s = kOpts[i].store;
  opt_value[i] = s == Store::INT ? v : s == Store::BOOL ? v != 0
               : s == Store::NS ? (v == 2 ? 2 : 1) : (v == 0 ? 0 : (v == 2 ? 2 : 1));
  opt_taken[i] = true;
}

int opt(Opt o) {
  const int i = (int)o;
  if (!opt_taken[i]) {
    const OptRow& r = kOpts[i];
    const char* e = r.env != nullptr ? getenv(r.env) : nullptr;
    set_opt(i, e == nullptr ? r.dflt : r.parse == Parse::ATOI ? atoi(e) : (e[0] == r.ch ? r.val : r.dflt));
  }
  return opt_value[i];
}

// ---- kernel routes ------------------------------------------------------------------------------------------------
// The route functions apply every option that selects a kernel; the *_applicable / *_plan predicates test shape and
// alignment only.  Options that pick a variant inside one kernel's launch are read where that launch is configured.
enum class Route { NONE, TC, PF, TINY, PWX, PWX_D2S, PWD2S, PWD2S_MMA, PW, DCONV_WIDE, DCONV_SMALL, TILED };

// depth-to-space input gradient: the tensor-core form unless tc = 0 or pwmma = 0 (then the fp32 FMA kernel)
static Route pwd2s_route() { return opt(Opt::TC) && opt(Opt::PWMMA) ? Route::PWD2S_MMA : Route::PWD2S; }

// Kernel of a forward or input-gradient op that runs as one launch, in order of preference; Route::NONE: each phase
// takes its phase_route.  The wgmma kernel needs its workspace within `ws_bytes` (< 0: no workspace, so the op stays
// on the fp32 kernels).
static Route fwd_route(const GConvK* ph, int np, const float* bias, int act, float beta, const float* mask_y,
                       const float* out, int64_t ws_bytes, bool partial_tiles = false) {
  if (np != 1 || ph[0].M == 0) return Route::NONE;
  const GConvK& k = ph[0];
  auto tc = [&] {
    return opt(Opt::TC) && tc_applicable(k, partial_tiles) && ws_bytes >= 0 &&
           (int64_t)tc_workspace_bytes(k, partial_tiles) <= ws_bytes;
  };
  if (opt(Opt::TC) == 2 && tc()) return Route::TC;
  // staged-patch forward; its stride-1 form only with pf_s1
  const bool pf = opt(Opt::PF) && opt(Opt::PWX) && pf_fwd_applicable(k, mask_y, out) && (k.ay.it != 1 || opt(Opt::PF_S1));
  // few-channel stride-1 stencils (4/8/16 -> same): the row-stream kernel of nlt_tiny.cu, ahead of the tensor path
  // (16 -> 16 at 512^2 is a 130 B/pixel stream: the wgmma pipeline's fixed costs exceed its 0.5 kFMA/pixel)
  if (pf && k.ay.it == 1) return Route::PF;
  if (opt(Opt::TINY) && tiny_stencil_applicable(k, out, mask_y)) return Route::TINY;
  // 2x2 / stride-2 convs of levels 1-2 (K = 64 / 128 into 16 / 32 channels)
  if (pf) return Route::PF;
  // up-convs into 4 / 8 channels: depth-to-space pointwise kernel with constant-bank weights (nlt_pwx.cu)
  if (opt(Opt::PWX) && pwx_d2s_fwd_applicable(k, beta, mask_y, out)) return Route::PWX_D2S;
  // input gradients of the 2x2 / stride-2 convs into 32-channel sources with K = 64 (level 3)
  if (opt(Opt::PWD2S_FIRST) && opt(Opt::PWX) && k.d2s && k.nseg == 1 && k.seg[0].C == 64 &&
      pwd2s_applicable(k, bias, act, out, mask_y, nullptr))
    return Route::PWD2S;
  return tc() ? Route::TC : Route::NONE;
}

// kernel of one phase of a forward or input-gradient op
static Route phase_route(const GConvK& k, const float* bias, int act, float beta, const float* mask_y,
                         const float* out) {
  if (opt(Opt::PWX) && pwx_fwd_applicable(k, beta, mask_y, out)) return Route::PWX;
  if (opt(Opt::PWX) && pwd2s_applicable(k, bias, act, out, mask_y, nullptr)) return pwd2s_route();
  if (pw_conv_applicable(k)) return Route::PW;
  if (opt(Opt::TINY) && tiny_stencil_applicable(k, out, mask_y)) return Route::TINY;
  // wide stencil kernel: options dconv_wide / dconv_wide32 / dconv_wide8 for its 16- / 32- / 8-output forms
  const bool wide = dconv_wide_applicable(k, out, mask_y) &&
                    opt(k.Cout == 16 ? Opt::DCONV_WIDE : (k.Cout == 32 ? Opt::DCONV_WIDE32 : Opt::DCONV_WIDE8)) > 0;
  if (dconv_small_applicable(k)) return wide && opt(Opt::DCONV_WIDE_FIRST) ? Route::DCONV_WIDE : Route::DCONV_SMALL;
  return wide ? Route::DCONV_WIDE : Route::TILED;
}

// single-phase pointwise op with a fused pointwise term: the depth-to-space kernel or the pointwise kernel
static Route fused_route(const GConvK& k, const PwExtra& ex, const float* bias, int act, const float* mask_y,
                         const float* out) {
  if (k.M == 0) return Route::NONE;
  if (opt(Opt::PWX) && pwd2s_applicable(k, bias, act, out, mask_y, &ex)) return pwd2s_route();
  return pw_extra_applicable(k, ex, out, mask_y) ? Route::PW : Route::NONE;
}

static int launch_route(Route r, const GConvK& k, const float* bias, int act, float beta, const float* mask_y,
                        int mask_act, float* out, const PwExtra* ex, void* ws, int64_t ws_bytes, bool prepacked,
                        cudaStream_t st, bool partial_tiles = false) {
  switch (r) {
    case Route::TC:
      return launch_tc(k, bias, act, beta, mask_y, mask_act, out, ws, (size_t)ws_bytes, st, prepacked, partial_tiles);
    case Route::PF: return launch_pf_fwd(k, bias, act, beta, mask_y, mask_act, out, st);
    case Route::TINY: return launch_tiny_stencil(k, bias, act, beta, mask_y, mask_act, out, st);
    case Route::PWX: return launch_pwx_fwd(k, bias, act, out, st);
    case Route::PWX_D2S: return launch_pwx_d2s_fwd(k, bias, act, out, st);
    case Route::PWD2S: return launch_pwd2s(k, beta, mask_y, mask_act, out, st, ex);
    case Route::PWD2S_MMA: return launch_pwd2s_mma(k, beta, mask_y, mask_act, out, st, ex);
    case Route::PW: return launch_pw_conv(k, bias, act, beta, mask_y, mask_act, out, st, ex);
    case Route::DCONV_WIDE: return launch_dconv_wide(k, bias, act, beta, mask_y, mask_act, out, st);
    case Route::DCONV_SMALL: return launch_dconv_small(k, bias, act, beta, mask_y, mask_act, out, st);
    case Route::TILED:
      if (k.Cout > 32) return launch_fwd<128, 64, 8, 8>(k, bias, act, beta, mask_y, mask_act, out, st);
      if (k.Cout > 16) return launch_fwd<128, 32, 8, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
      if (k.Cout > 8) return launch_fwd<256, 16, 8, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
      if (k.Cout > 4) return launch_fwd<256, 8, 4, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
      return launch_fwd<256, 4, 2, 4>(k, bias, act, beta, mask_y, mask_act, out, st);
    case Route::NONE: break;
  }
  return set_err(NLT_ERR_INVALID, "no kernel route");
}

enum class WgradRoute { PWX, WOP, WOPN, PWS, TC, TPP, SMALL, TILED };

// outer-product weight gradient: option wop = 1 for shapes into <= 8 channels outside depth-to-space, 2 for all
static bool wop_on(const GConvK& k) { return opt(Opt::WOP) >= 2 || (opt(Opt::WOP) == 1 && !k.d2s && k.Cout <= 8); }

// tensor-core weight gradient for this phase?  The row-run warp-stream kernel takes the shapes it applies to
// (<= 16 gradient channels, K-depth <= 160: the level-1 32 -> 16 down-conv), the wgmma kernel everything else.
static bool use_tc_wgrad(const GConvK& k) {
  return opt(Opt::TC) && opt(Opt::TC_WGRAD) && tc_wgrad_applicable(k) && !wgrad_small_applicable(k);
}

// a k == stride transposed conv keeps its one-pass depth-to-space form when a kernel takes it (the warp-stream
// kernel for narrow tiles, the wgmma kernel from K_d = 128 up); otherwise it runs as s*s phases
static bool wgrad_keeps_d2s(const GConvK& k, const float* G) {
  return (opt(Opt::PWX) && pwx_wgrad_applicable(k, G)) || (wop_on(k) && wop_wgrad_applicable(k, G)) ||
         wgrad_small_applicable(k) || use_tc_wgrad(k);
}

static size_t wgrad_ws_floats(WgradRoute r, const GConvK& k) {
  switch (r) {
    case WgradRoute::PWX: return pwx_wgrad_ws_floats(k);
    case WgradRoute::WOP: return wop_wgrad_ws_floats(k);
    case WgradRoute::WOPN: return wopn_wgrad_ws_floats(k);
    case WgradRoute::PWS: return pws_wgrad_ws_floats(k);
    case WgradRoute::TC: return tc_wgrad_ws_floats(k);
    case WgradRoute::TPP: return wgrad_tpp_ws_floats(k);
    case WgradRoute::SMALL: return wgrad_small_ws_floats(k);
    case WgradRoute::TILED: break;
  }
  return plan_wgrad(k).ws_floats;
}

// Weight-gradient kernel of one phase, in order of preference.  The first four give way to the next route when their
// workspace exceeds `ws_bytes`; the workspace query asks with G = nullptr and no limit.
static WgradRoute wgrad_route(const GConvK& k, const float* G, int64_t ws_bytes) {
  auto fits = [&](WgradRoute r) { return (int64_t)(wgrad_ws_floats(r, k) * sizeof(float)) <= ws_bytes; };
  if (opt(Opt::PWX) && pwx_wgrad_applicable(k, G) && fits(WgradRoute::PWX)) return WgradRoute::PWX;
  // few-channel layers at (near) full resolution: register-tile outer products, one warp per unit kind (nlt_wop.cu)
  if (wop_on(k) && wop_wgrad_applicable(k, G) && fits(WgradRoute::WOP)) return WgradRoute::WOP;
  // final 1x1 conv into <= 4 channels: coalesced (pixel, channel quad) lanes (nlt_wop.cu)
  if (opt(Opt::WOP) > 0 && wopn_wgrad_applicable(k, G) && fits(WgradRoute::WOPN)) return WgradRoute::WOPN;
  if (opt(Opt::PWX) && pws_wgrad_applicable(k, G) && fits(WgradRoute::PWS)) return WgradRoute::PWS;
  if (use_tc_wgrad(k)) return WgradRoute::TC;
  if (wgrad_tpp_applicable(k)) return WgradRoute::TPP;
  if (wgrad_small_applicable(k)) return WgradRoute::SMALL;
  return WgradRoute::TILED;
}

}  // namespace nlt

extern "C" {

const char* nlt_version(void) { return "nlt_b200 0.1 (sm_90a)"; }
const char* nlt_last_error(void) { return nlt::g_err; }
uint64_t nlt_launch_count(void) { return __atomic_load_n(&nlt::g_launches, __ATOMIC_RELAXED); }

uint64_t nlt_kernel_launch_count(const char* name) {
  if (name == nullptr) return 0;
  std::lock_guard<std::mutex> lock(nlt::g_kl_mutex);
  for (int i = 0; i < nlt::g_kl_n; ++i)
    if (strcmp(nlt::g_kl_name[i], name) == 0) return nlt::g_kl_count[i];
  return 0;
}
uint64_t nlt_tc_launch_count(void) { return __atomic_load_n(&nlt::g_tc_launches, __ATOMIC_RELAXED); }

int nlt_set_option(const char* name, int value) {
  NLT_CHECK_ARG(name != nullptr, "null option name");
  const int i = opt_index(name);
  if (i < 0) return set_err(NLT_ERR_INVALID, "unknown option '%s'", name);
  set_opt(i, value);
  return NLT_OK;
}

int nlt_get_option(const char* name, int* value) {
  NLT_CHECK_ARG(name != nullptr && value != nullptr, "null argument");
  const int i = opt_index(name);
  if (i < 0) return set_err(NLT_ERR_INVALID, "unknown option '%s'", name);
  *value = opt((Opt)i);
  return NLT_OK;
}

int64_t nlt_gconv_fwd_workspace_bytes(const nlt_gconv_desc* d) {
  GConvK ph[16];
  int np = 0;
  if (build_phases(d, ph, &np, /*allow_d2s=*/true) != NLT_OK) return -1;
  if (np == 1 && opt(Opt::TC) && tc_applicable(ph[0])) return (int64_t)tc_workspace_bytes(ph[0]);
  return 0;
}

// does the forward of `d` run on the wgmma kernel (which reads packed hi / lo weight planes)?
static bool fwd_takes_tc(const GConvK* ph, int np, float beta, const float* mask_y, const float* out) {
  return fwd_route(ph, np, nullptr, 0, beta, mask_y, out, INT64_MAX) == Route::TC;
}

int64_t nlt_gconv_fwd_pack_bytes(const nlt_gconv_desc* d, float beta, int has_mask) {
  GConvK ph[16];
  int np = 0;
  if (build_phases(d, ph, &np, /*allow_d2s=*/true) != NLT_OK) return -1;
  const float* aligned = reinterpret_cast<const float*>((uintptr_t)256);     // stands for any 16-byte aligned buffer
  if (!fwd_takes_tc(ph, np, beta, has_mask ? aligned : nullptr, aligned)) return 0;
  return (int64_t)tc_workspace_bytes(ph[0]);
}

int nlt_gconv_pack_weights(const nlt_gconv_desc* d, void* packed, int64_t packed_bytes, void* stream) {
  GConvK ph[16];
  int np = 0;
  int rc = build_phases(d, ph, &np, /*allow_d2s=*/true);
  if (rc != NLT_OK) return rc;
  NLT_CHECK_ARG(np == 1 && opt(Opt::TC) && tc_applicable(ph[0]), "this op does not run on the tensor-core kernel");
  return tc_pack(ph[0], packed, (size_t)packed_bytes, (cudaStream_t)stream);
}

static int gconv_fwd_impl(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y,
                          int mask_act, float* out, void* workspace, int64_t workspace_bytes, void* stream, bool prepacked,
                          bool partial_tiles = false) {
  GConvK ph[16];
  int np = 0;
  int rc = build_phases(d, ph, &np, /*allow_d2s=*/true);
  if (rc != NLT_OK) return rc;
  NLT_CHECK_ARG(out != nullptr, "null output");
  NLT_CHECK_ARG(act >= 0 && act <= 3 && mask_act >= 0 && mask_act <= 3, "bad activation code");
  NLT_CHECK_ARG(beta == 0.f || beta == 1.f, "beta must be 0 or 1");
  cudaStream_t st = (cudaStream_t)stream;
  // packed weights are only for an op that nlt_gconv_fwd_pack_bytes puts on the wgmma kernel: route it as that query
  // does (no bias)
  const Route r = fwd_route(ph, np, prepacked ? nullptr : bias, prepacked ? 0 : act, beta, mask_y, out,
                            workspace != nullptr ? workspace_bytes : -1, partial_tiles);
  if (prepacked)
    NLT_CHECK_ARG(r != Route::NONE && r != Route::PWD2S,
                  "nlt_gconv_fwd_packed: this op does not run on the tensor-core kernel (nlt_gconv_fwd_pack_bytes == 0)");
  if (r != Route::NONE)
    return launch_route(r, ph[0], bias, act, beta, mask_y, mask_act, out, nullptr, workspace, workspace_bytes, prepacked,
                        st, partial_tiles);
  for (int i = 0; i < np; ++i) {
    const GConvK& k = ph[i];
    if (k.M == 0) continue;
    rc = launch_route(phase_route(k, bias, act, beta, mask_y, out), k, bias, act, beta, mask_y, mask_act, out, nullptr,
                      nullptr, 0, false, st);
    if (rc != NLT_OK) return rc;
  }
  return NLT_OK;
}

int nlt_gconv_fwd_ws(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y,
                     int mask_act, float* out, void* workspace, int64_t workspace_bytes, void* stream) {
  return gconv_fwd_impl(d, bias, act, beta, mask_y, mask_act, out, workspace, workspace_bytes, stream, false);
}

int nlt_gconv_fwd_packed(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y,
                         int mask_act, float* out, const void* packed, int64_t packed_bytes, void* stream) {
  return gconv_fwd_impl(d, bias, act, beta, mask_y, mask_act, out, const_cast<void*>(packed), packed_bytes, stream, true);
}

static int pw_term_phase(const nlt_gconv_desc* d, const nlt_pw_term* term, GConvK* k, PwExtra* ex) {
  GConvK ph[16];
  int np = 0;
  int rc = build_phases(d, ph, &np, /*allow_d2s=*/true);
  if (rc != NLT_OK) return rc;
  NLT_CHECK_ARG(term != nullptr && term->x != nullptr && term->w != nullptr, "null pointwise term");
  if (np != 1) return NLT_ERR_UNSUPPORTED;
  *k = ph[0];
  ex->x = term->x; ex->K = term->K; ex->w = term->w; ex->wk = term->w_k_stride; ex->wn = term->w_n_stride;
  return NLT_OK;
}

int nlt_gconv_fwd_fused_supported(const nlt_gconv_desc* d, const nlt_pw_term* term, const float* mask_y,
                                  const float* out) {
  GConvK k;
  PwExtra ex;
  if (pw_term_phase(d, term, &k, &ex) != NLT_OK) return 0;
  return fused_route(k, ex, nullptr, 0, mask_y, out) != Route::NONE ? 1 : 0;
}

int nlt_gconv_fwd_fused(const nlt_gconv_desc* d, const nlt_pw_term* term, const float* bias, int act, float beta,
                        const float* mask_y, int mask_act, float* out, void* stream) {
  GConvK k;
  PwExtra ex;
  int rc = pw_term_phase(d, term, &k, &ex);
  if (rc == NLT_ERR_UNSUPPORTED) return set_err(NLT_ERR_UNSUPPORTED, "fused pointwise term: op is not a single-phase pointwise op");
  if (rc != NLT_OK) return rc;
  NLT_CHECK_ARG(out != nullptr, "null output");
  NLT_CHECK_ARG(act >= 0 && act <= 3 && mask_act >= 0 && mask_act <= 3, "bad activation code");
  NLT_CHECK_ARG(beta == 0.f || beta == 1.f, "beta must be 0 or 1");
  const Route r = fused_route(k, ex, bias, act, mask_y, out);
  if (r == Route::NONE) return set_err(NLT_ERR_UNSUPPORTED, "fused pointwise term: shape not served by the pointwise kernel");
  return launch_route(r, k, bias, act, beta, mask_y, mask_act, out, &ex, nullptr, 0, false, (cudaStream_t)stream);
}

int nlt_gconv_fwd(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y,
                  int mask_act, float* out, void* stream) {
  return nlt_gconv_fwd_ws(d, bias, act, beta, mask_y, mask_act, out, nullptr, 0, stream);
}

int64_t nlt_gconv_wgrad_workspace_bytes(const nlt_gconv_desc* d) {
  GConvK ph[16];
  int np = 0;
  if (build_phases(d, ph, &np, /*allow_d2s=*/true) != NLT_OK) return -1;
  if (np == 1 && ph[0].d2s && !wgrad_keeps_d2s(ph[0], nullptr) && build_phases(d, ph, &np, false) != NLT_OK) return -1;
  size_t mx = 0;
  for (int i = 0; i < np; ++i) {
    if (ph[i].M == 0) continue;
    const size_t need = wgrad_ws_floats(wgrad_route(ph[i], nullptr, INT64_MAX), ph[i]);
    if (need > mx) mx = need;
  }
  return (int64_t)(mx * sizeof(float));
}

int nlt_gconv_wgrad(const nlt_gconv_desc* d, const float* G, float* dW, float* db, int accumulate,
                    void* workspace, int64_t workspace_bytes, void* stream) {
  GConvK ph[16];
  int np = 0;
  int rc = build_phases(d, ph, &np, /*allow_d2s=*/true);
  if (rc != NLT_OK) return rc;
  if (np == 1 && ph[0].d2s && !wgrad_keeps_d2s(ph[0], G)) rc = build_phases(d, ph, &np, false);
  if (rc != NLT_OK) return rc;
  NLT_CHECK_ARG(G != nullptr && dW != nullptr && workspace != nullptr, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  bool bias_done = false;
  for (int i = 0; i < np; ++i) {
    const GConvK& k = ph[i];
    if (k.M == 0) continue;
    float* ws = (float*)workspace;
    WgradK w;
    size_t KD_pad = 0;
    const WgradRoute r = wgrad_route(k, G, workspace_bytes);
    const int64_t need = (int64_t)(wgrad_ws_floats(r, k) * sizeof(float));
    NLT_CHECK_ARG(need <= workspace_bytes, "workspace too small: need %lld have %lld", (long long)need,
                  (long long)workspace_bytes);
    switch (r) {
      case WgradRoute::PWX: rc = launch_pwx_wgrad(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::WOP: rc = launch_wop_wgrad(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::WOPN: rc = launch_wopn_wgrad(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::PWS: rc = launch_pws_wgrad(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::TC: rc = launch_tc_wgrad(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::TPP: rc = launch_wgrad_tpp(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::SMALL: rc = launch_wgrad_small(k, G, ws, &w, &KD_pad, st); break;
      case WgradRoute::TILED: {
        WgradPlan p = plan_wgrad(k);
        w.g = k; w.GS = p.GS; w.KG = p.KG; w.ld = p.ld; w.nsplit = p.nsplit; w.pix_per_split = p.pix_per_split;
        KD_pad = p.KD_pad;
        dim3 grid(p.kd_tiles, p.n_tiles, p.nsplit);
        switch (p.tn) {
          case 64: gconv_wgrad_kernel<32, 64, 8, 8, 128><<<grid, 128, 0, st>>>(w, G, ws); break;
          case 32: gconv_wgrad_kernel<32, 32, 8, 4, 128><<<grid, 128, 0, st>>>(w, G, ws); break;
          case 16: gconv_wgrad_kernel<32, 16, 4, 4, 128><<<grid, 128, 0, st>>>(w, G, ws); break;
          case 8: gconv_wgrad_kernel<32, 8, 4, 4, 64><<<grid, 64, 0, st>>>(w, G, ws); break;
          default: gconv_wgrad_kernel<32, 4, 4, 4, 32><<<grid, 32, 0, st>>>(w, G, ws); break;
        }
        NLT_CUDA_LAUNCH_CHECK("gconv_wgrad_kernel");
        break;
      }
    }
    if (rc != NLT_OK) return rc;
    // every phase sees a disjoint subset of lattice pixels, so the bias gradient
    // accumulates across phases; taps are disjoint across phases.
    const size_t total = (size_t)w.KG * 4 * k.Cout;
    if (w.nsplit <= 32) {
      gconv_wgrad_reduce_flat_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, ws, KD_pad, dW, db, accumulate,
                                                                                     bias_done ? 1 : accumulate);
    } else {
      int blocks = (int)((total + 7) / 8);
      if (blocks > sm_count() * 16) blocks = sm_count() * 16;
      gconv_wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(w, ws, KD_pad, dW, db, accumulate,
                                                        bias_done ? 1 : accumulate);
    }
    NLT_CUDA_LAUNCH_CHECK("gconv_wgrad_reduce_kernel");
    bias_done = true;
  }
  return NLT_OK;
}

}  // extern "C"

namespace nlt {

int gconv_run(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y, int mask_act,
              float* out, void* workspace, int64_t workspace_bytes, bool partial_tiles, cudaStream_t st) {
  return gconv_fwd_impl(d, bias, act, beta, mask_y, mask_act, out, workspace, workspace_bytes, st, false, partial_tiles);
}

int64_t gconv_tc_workspace_bytes(const nlt_gconv_desc* d, bool partial_tiles) {
  GConvK ph[16];
  int np = 0;
  if (build_phases(d, ph, &np, /*allow_d2s=*/true) != NLT_OK) return -1;
  return np == 1 && tc_applicable(ph[0], partial_tiles) ? (int64_t)tc_workspace_bytes(ph[0], partial_tiles) : 0;
}

}  // namespace nlt
