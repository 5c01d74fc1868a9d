// Weight gradients of the few-channel layers at (near) full resolution -- levels 10-12 of the decoder and the
// 16 -> 16 second convs of level 1 (nlt/networks/convnet.py:50-76 at depth0 = 16):
//
//   stride-1 2x2 stencils C -> C, C in {4, 8, 16}:        dW[tap, c, n]  = sum_p x[p + tap, c] * dz[p, n]
//   2x2 / stride-2 up-convs K -> CT, CT in {4, 8, 16}:    dW[tap, c, n]  = sum_p x[p, c] * dz[2p + tap, n]
//
// Their [K_d x N] products are tiny (64 ... 10240 numbers) and the pixel streams long (0.5-8 M pixels), so the work
// is cut into OUTER-PRODUCT UNITS: per lattice pixel a unit multiplies one float4 "A" (4 channels of one operand)
// with 16 consecutive floats "B" of the other operand into a 4 x 16 register tile (64 FMAs for 5 LDG.128).  A warp
// owns one unit kind for the whole launch (its accumulators never leave registers): lanes = (pixel slot, channel quad
// of A) with the quad fastest, so that A loads are one contiguous 512-byte run and B loads broadcast inside a pixel.
// Warps stream over row tiles on their own -- no shared memory, no barriers -- and write one fp32 partial per CTA in
// the k-group layout of WgradK; the reduce kernel of nlt_gconv.cu finishes (fixed order: deterministic).
//
// Orientation: A is normally the input-side operand (rows of the partial) and B the 16 gradient columns; when the layer
// has fewer than 16 outputs (4 -> 4, 8 -> 8) the roles swap (A = gradient quad, B = 16 floats of the input patch).
// The bias gradient is one more warp whose constant operand is (1, 0, ...).
#include "nlt_common.cuh"

namespace nlt {

constexpr int WOP_MAX_TASKS = 16;      // warps per CTA
constexpr int WOP_TPX = 128;           // lattice pixels per row tile

struct WopTask {
  const float* a;
  const float* b;
  int a_C, b_C;                // channels per pixel of the A / B image
  int a_s, b_s;                // lattice -> image coordinate scale
  int a_dy, a_dx, a_c0;        // A pixel offset, first channel (the lane adds 4 * quad)
  int a_H, a_W, b_H, b_W;
  int b_dy[2];                 // row offset of B float4 pairs (0, 1) and (2, 3)
  int b_px[4], b_off[4];       // pixel offset (bounds check) and float offset from pixel b_s * x of each B float4
  int lq;                      // log2(lanes per pixel) = log2(quads of A)
  int konst;                   // 1: A = (1, 0, 0, 0) (bias, normal orientation); 2: B = (1, 0, ..., 0) (bias, swapped)
  int swapped;                 // 0: rows <- A, columns <- B;  1: columns <- A, rows <- B
  int base;                    // normal: first partial row of quad 0
  short mmap[16];              // normal: column of B element m; swapped: row of B element m (-1: dropped)
};

struct WopParams {
  WopTask task[WOP_MAX_TASKS];
  int ntask;
  int H, W;                    // lattice rows per image / row length
  int tiles_per_row;
  uint32_t ntiles;
  int kd_pad, ld;
};

__global__ void __launch_bounds__(WOP_MAX_TASKS * 32, 1)
wop_wgrad_kernel(const __grid_constant__ WopParams p, float* __restrict__ ws) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= p.ntask) return;
  const WopTask& tk = p.task[warp];
  const int lq = tk.lq;
  const int cq = lane & ((1 << lq) - 1), slot = lane >> lq;
  const int pw = 32 >> lq;                                     // pixels per warp step
  float2 acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < 8; ++m) acc[i][m] = make_float2(0.f, 0.f);

  const int a_C = tk.a_C, b_C = tk.b_C, a_s = tk.a_s, b_s = tk.b_s, a_dx = tk.a_dx, a_W = tk.a_W, b_W = tk.b_W;
  const int konst = tk.konst;
  int bpx[4], boff[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { bpx[j] = tk.b_px[j]; boff[j] = tk.b_off[j]; }

  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    const uint32_t r = t / (uint32_t)p.tiles_per_row;          // n * H + y
    const int x0 = (int)(t - r * (uint32_t)p.tiles_per_row) * WOP_TPX;
    const int n = (int)(r / (uint32_t)p.H), y = (int)(r - (uint32_t)n * p.H);
    const int ya = a_s * y + tk.a_dy;
    const bool a_row = (unsigned)ya < (unsigned)tk.a_H;
    const float* abase = tk.a + ((size_t)n * tk.a_H + (a_row ? ya : 0)) * a_W * a_C + tk.a_c0 + 4 * cq;
    const float* bbase[2];
    bool b_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int yb = b_s * y + tk.b_dy[h];
      b_row[h] = (unsigned)yb < (unsigned)tk.b_H;
      bbase[h] = tk.b + ((size_t)n * tk.b_H + (b_row[h] ? yb : 0)) * b_W * b_C;
    }
    const int xend = min(x0 + WOP_TPX, p.W);
#pragma unroll 2
    for (int x = x0 + slot; x < xend; x += pw) {
      float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
      if (konst == 1) {
        av.x = cq == 0 ? 1.f : 0.f;
      } else {
        const int xa = a_s * x + a_dx;
        if (a_row && (unsigned)xa < (unsigned)a_W) av = ld4(abase + (size_t)xa * a_C);
      }
      float4 bv[4];
      const int xb = b_s * x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        bv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (konst == 2) {
          if (j == 0) bv[j].x = 1.f;
        } else if (b_row[j >> 1] && (unsigned)(xb + bpx[j]) < (unsigned)b_W) {
          bv[j] = ld4(bbase[j >> 1] + (ptrdiff_t)xb * b_C + boff[j]);
        }
      }
      const float as[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 aa = make_float2(as[i], as[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][2 * j] = ffma2(aa, make_float2(bv[j].x, bv[j].y), acc[i][2 * j]);
          acc[i][2 * j + 1] = ffma2(aa, make_float2(bv[j].z, bv[j].w), acc[i][2 * j + 1]);
        }
      }
    }
  }
  // lanes of one quad: sum over the pixel slots (fixed butterfly order)
  for (int off = 16; off >= (1 << lq); off >>= 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        acc[i][m].x += __shfl_xor_sync(0xffffffffu, acc[i][m].x, off);
        acc[i][m].y += __shfl_xor_sync(0xffffffffu, acc[i][m].y, off);
      }
  }
  if (slot != 0) return;
  float* part = ws + (size_t)blockIdx.x * p.kd_pad * p.ld;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      const float v = (m & 1) ? acc[i][m >> 1].y : acc[i][m >> 1].x;
      const int mm = tk.mmap[m];
      if (mm < 0) continue;
      if (!tk.swapped) part[(size_t)(tk.base + 4 * cq + i) * p.ld + mm] = v;
      else part[(size_t)mm * p.ld + 4 * cq + i] = v;
    }
}

struct WopPlan {
  bool ok;
  WopParams p;
  int GS, KG;
  unsigned grid;
};

static int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }
static bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

static WopPlan wop_plan(const GConvK& k, const float* G) {
  WopPlan pl;
  memset(&pl, 0, sizeof(pl));
  if (k.M == 0) return pl;
  WopParams& p = pl.p;
  for (int s = 0; s < k.nseg; ++s)
    if (!k.seg[s].vec || k.seg[s].sub != nullptr || k.seg[s].bcast) return pl;
  int nt = 0;
  if (k.d2s) {
    // ---- up-conv, one pass over the input lattice: rows = input channels, columns = (tap, n) ----
    const int CT = k.cout_true;
    if (k.d2s_s != 2 || (CT != 4 && CT != 8 && CT != 16) || k.Cout != 4 * CT) return pl;
    if (k.ay.nt != k.Hin || k.ax.nt != k.Win || k.Hout != 2 * k.Hin || k.Wout != 2 * k.Win) return pl;
    const int nsub = 4 * CT / 16;
    int GS = 0;
    for (int s = 0; s < k.nseg; ++s) GS += k.seg[s].C / 4;
    pl.GS = GS; pl.KG = GS + 1;
    p.kd_pad = (GS + 1) * 4; p.ld = 4 * CT;
    int gbase = 0;
    for (int s = -1; s < k.nseg; ++s) {                         // s = -1: the bias warps
      const int Q = s < 0 ? 1 : k.seg[s].C / 4;
      if (!pow2(Q) || Q > 32) return pl;
      for (int sub = 0; sub < nsub; ++sub) {
        if (nt >= WOP_MAX_TASKS) return pl;
        WopTask& t = p.task[nt++];
        t.b = G; t.b_C = CT; t.b_s = 2; t.b_H = k.Hout; t.b_W = k.Wout;
        if (s < 0) { t.a = G; t.konst = 1; t.a_C = 4; t.a_s = 1; t.a_H = k.Hin; t.a_W = k.Win; t.lq = 0; t.base = GS * 4; }
        else {
          t.a = k.seg[s].ptr; t.a_C = k.seg[s].C; t.a_s = 1; t.a_H = k.Hin; t.a_W = k.Win; t.lq = ilog2(Q);
          t.base = gbase * 4;
        }
        // B = elements [16 sub, 16 sub + 16) of the pixel's gradient vector [dy][dx][n]
        for (int j = 0; j < 4; ++j) {
          const int e = 16 * sub + 4 * j;                       // first element of this float4
          const int tap = e / CT, n0 = e - tap * CT;
          const int dy = tap >> 1, dx = tap & 1;
          if (j == 0 || j == 2) t.b_dy[j >> 1] = dy;
          else if (t.b_dy[j >> 1] != dy) return pl;             // (cannot happen: pairs never straddle rows)
          t.b_px[j] = dx; t.b_off[j] = dx * CT + n0;
        }
        for (int m = 0; m < 16; ++m) t.mmap[m] = (short)(16 * sub + m);
      }
      if (s >= 0) gbase += Q;
    }
    p.H = k.Hin; p.W = k.Win;
  } else {
    // ---- stride-1 2x2 stencil C -> C ----
    if (k.nseg != 1) return pl;
    const int C = k.seg[0].C;
    if (C != k.Cout || k.Cout != k.cout_true || (C != 4 && C != 8 && C != 16)) return pl;
    if (k.ay.nu != 2 || k.ax.nu != 2 || k.ay.it != 1 || k.ax.it != 1) return pl;
    if (k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0) return pl;
    if (k.Hin != k.Hout || k.Win != k.Wout || k.ay.nt != k.Hout || k.ax.nt != k.Wout) return pl;
    const int GS = C / 4;
    pl.GS = GS; pl.KG = 4 * GS + 1;
    p.kd_pad = (4 * GS + 1) * 4; p.ld = C;
    const float* X = k.seg[0].ptr;
    const int bias_row = 4 * GS * 4;
    auto tdy = [&](int uy) { return uy * k.ay.iu + k.ay.i0; };
    auto tdx = [&](int ux) { return ux * k.ax.iu + k.ax.i0; };
    if (C == 16) {
      for (int tap = 0; tap < 5; ++tap) {                       // tap 4: bias
        WopTask& t = p.task[nt++];
        t.b = G; t.b_C = 16; t.b_s = 1; t.b_H = k.Hout; t.b_W = k.Wout;
        for (int j = 0; j < 4; ++j) { t.b_px[j] = 0; t.b_off[j] = 4 * j; }
        for (int m = 0; m < 16; ++m) t.mmap[m] = (short)m;
        t.a_C = 16; t.a_s = 1; t.a_H = k.Hin; t.a_W = k.Win;
        if (tap == 4) { t.a = G; t.konst = 1; t.lq = 0; t.base = bias_row; }
        else { t.a = X; t.a_dy = tdy(tap >> 1); t.a_dx = tdx(tap & 1); t.lq = 2; t.base = tap * GS * 4; }
      }
    } else if (C == 8) {
      for (int uy = 0; uy < 3; ++uy) {                          // uy 2: bias
        WopTask& t = p.task[nt++];
        t.swapped = 1;
        t.a = G; t.a_C = 8; t.a_s = 1; t.a_H = k.Hout; t.a_W = k.Wout; t.lq = 1;
        t.b = X; t.b_C = 8; t.b_s = 1; t.b_H = k.Hin; t.b_W = k.Win;
        if (uy == 2) {
          t.konst = 2;
          for (int m = 0; m < 16; ++m) t.mmap[m] = (short)(m == 0 ? bias_row : -1);
        } else {
          t.b_dy[0] = t.b_dy[1] = tdy(uy);
          for (int j = 0; j < 4; ++j) {                         // float4 j: tap ux = j / 2, channels 4 (j % 2) ...
            const int ux = j >> 1;
            t.b_px[j] = tdx(ux); t.b_off[j] = tdx(ux) * 8 + 4 * (j & 1);
            for (int e = 0; e < 4; ++e) t.mmap[4 * j + e] = (short)(((uy * 2 + ux) * GS + (j & 1)) * 4 + e);
          }
        }
      }
    } else {
      for (int q = 0; q < 2; ++q) {                             // q 1: bias
        WopTask& t = p.task[nt++];
        t.swapped = 1;
        t.a = G; t.a_C = 4; t.a_s = 1; t.a_H = k.Hout; t.a_W = k.Wout; t.lq = 0;
        t.b = X; t.b_C = 4; t.b_s = 1; t.b_H = k.Hin; t.b_W = k.Win;
        if (q == 1) {
          t.konst = 2;
          for (int m = 0; m < 16; ++m) t.mmap[m] = (short)(m == 0 ? bias_row : -1);
        } else {
          for (int j = 0; j < 4; ++j) {                         // float4 j: tap (uy, ux) = (j / 2, j % 2)
            const int uy = j >> 1, ux = j & 1;
            t.b_dy[uy] = tdy(uy);
            t.b_px[j] = tdx(ux); t.b_off[j] = tdx(ux) * 4;
            for (int e = 0; e < 4; ++e) t.mmap[4 * j + e] = (short)((uy * 2 + ux) * 4 + e);
          }
        }
      }
    }
    p.H = k.Hout; p.W = k.Wout;
  }
  if (G != nullptr && !aligned16(G)) return pl;
  p.ntask = nt;
  if (p.W < 32) return pl;
  p.tiles_per_row = (p.W + WOP_TPX - 1) / WOP_TPX;
  const long long ntiles = (long long)k.N * p.H * p.tiles_per_row;
  if (ntiles < 1 || ntiles > (1ll << 31)) return pl;
  p.ntiles = (uint32_t)ntiles;
  // 128 registers per thread: 16 resident warps per SM
  const unsigned per_sm = (unsigned)(16 / nt > 0 ? 16 / nt : 1);
  const unsigned cap = (unsigned)sm_count() * per_sm;
  pl.grid = p.ntiles < cap ? (unsigned)p.ntiles : cap;
  pl.ok = true;
  return pl;
}

// ---------------------------------------------------------------------------------------------
// Weight gradient of a 1x1 conv into <= 4 channels (the final conv, nlt/networks/convnet.py:65-70: 36 -> 3 at full
// resolution): dW[c, n] = sum_p x[p, c] * dz[p, n] is 108 numbers over 8 M pixels -- a pure stream of 156 B per
// pixel.  lanes = (pixel slot, channel quad) with the quad fastest, so that a warp's x loads are one contiguous
// 512-byte run (the thread-per-pixel form read 16 of every 64 bytes per instruction and had three K-split CTAs
// re-read every line); 12 accumulators per lane; sources get warps in proportion to their width.
// ---------------------------------------------------------------------------------------------
constexpr int WOPN_MAX_WARPS = 12;

struct WopnParams {
  const float* src[NLT_MAX_SEG];
  int C[NLT_MAX_SEG], lq[NLT_MAX_SEG], row0[NLT_MAX_SEG];       // channels, log2(quads), first partial row
  int w_seg[WOPN_MAX_WARPS], w_phase[WOPN_MAX_WARPS], w_nphase[WOPN_MAX_WARPS];
  int nwarp, N, ld, kd_pad, bias_row;
  uint32_t M;
};

template <int N>
__global__ void __launch_bounds__(WOPN_MAX_WARPS * 32, 3)
wopn_wgrad_kernel(const __grid_constant__ WopnParams p, const float* __restrict__ G, float* __restrict__ ws) {
  __shared__ float red[WOPN_MAX_WARPS][16 * 4 * N];              // [warp][quad <= 16][4][N]
  __shared__ float redb[N];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < p.nwarp) {
    const int sg = p.w_seg[warp];
    const int lq = p.lq[sg], C = p.C[sg];
    const int cq = lane & ((1 << lq) - 1), slot = lane >> lq;
    const uint32_t pw = 32u >> lq;                               // pixels per warp step
    const uint32_t stride = pw * (uint32_t)p.w_nphase[warp] * gridDim.x;
    const float* xb = p.src[sg] + 4 * cq;
    const bool do_bias = (warp == 0) && cq == 0;
    float acc[4][N], gsum[N];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int n = 0; n < N; ++n) acc[i][n] = 0.f;
#pragma unroll
    for (int n = 0; n < N; ++n) gsum[n] = 0.f;
    uint32_t px = (blockIdx.x * (uint32_t)p.w_nphase[warp] + (uint32_t)p.w_phase[warp]) * pw + slot;
#pragma unroll 4
    for (; px < p.M; px += stride) {
      const float4 xv = ld4(xb + (size_t)px * C);
      float g[N];
#pragma unroll
      for (int n = 0; n < N; ++n) g[n] = __ldg(G + (size_t)px * N + n);
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int n = 0; n < N; ++n) acc[i][n] = fmaf(xs[i], g[n], acc[i][n]);
      if (do_bias) {
#pragma unroll
        for (int n = 0; n < N; ++n) gsum[n] += g[n];
      }
    }
    for (int off = 16; off >= (1 << lq); off >>= 1) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int n = 0; n < N; ++n) acc[i][n] += __shfl_xor_sync(0xffffffffu, acc[i][n], off);
    }
    if (warp == 0) {                                             // the bias lanes are the cq == 0 lanes of warp 0
      for (int off = 16; off >= (1 << lq); off >>= 1) {
#pragma unroll
        for (int n = 0; n < N; ++n) gsum[n] += __shfl_xor_sync(0xffffffffu, gsum[n], off);
      }
      if (lane == 0) {
#pragma unroll
        for (int n = 0; n < N; ++n) redb[n] = gsum[n];
      }
    }
    if (slot == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int n = 0; n < N; ++n) red[warp][(cq * 4 + i) * N + n] = acc[i][n];
    }
  }
  __syncthreads();
  // warps of one source in fixed order, one partial per CTA
  float* part = ws + (size_t)blockIdx.x * p.kd_pad * p.ld;
  for (int i = threadIdx.x; i < p.kd_pad * p.ld; i += blockDim.x) part[i] = 0.f;
  __syncthreads();
  for (int sg = 0; sg < NLT_MAX_SEG; ++sg) {
    if (p.C[sg] == 0) continue;
    const int cnt = p.C[sg] * N;                                 // (channel, n) entries of this source
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      float v = 0.f;
      for (int w = 0; w < p.nwarp; ++w)
        if (p.w_seg[w] == sg) v += red[w][i];
      part[(size_t)(p.row0[sg] + i / N) * p.ld + i % N] = v;
    }
  }
  if (threadIdx.x < N) part[(size_t)p.bias_row * p.ld + threadIdx.x] = redb[threadIdx.x];
}

static bool wopn_plan(const GConvK& k, const float* G, WopnParams* p, unsigned* grid, int* GS_out) {
  memset(p, 0, sizeof(*p));
  if (k.d2s || k.M < (1u << 16) || k.Cout != k.cout_true || k.Cout < 1 || k.Cout > 4) return false;
  if (k.ay.nu != 1 || k.ax.nu != 1 || k.ay.it != 1 || k.ax.it != 1 || k.ay.i0 != 0 || k.ax.i0 != 0) return false;
  if (k.ay.os != 1 || k.ax.os != 1 || k.ay.o0 != 0 || k.ax.o0 != 0) return false;
  if (k.Hin != k.Hout || k.Win != k.Wout || k.ay.nt != k.Hout || k.ax.nt != k.Wout) return false;
  (void)G;
  int GS = 0, qmin = 32, qsum = 0;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    if (!sg.vec || sg.sub != nullptr || sg.bcast || sg.C < 4 || sg.C > 64 || !pow2(sg.C / 4)) return false;
    p->src[s] = sg.ptr; p->C[s] = sg.C; p->lq[s] = ilog2(sg.C / 4); p->row0[s] = GS * 4;
    GS += sg.C / 4;
    if (sg.C / 4 < qmin) qmin = sg.C / 4;
    qsum += sg.C / 4;
  }
  int nw = 0;
  for (int s = 0; s < k.nseg; ++s) {
    const int cnt = (k.seg[s].C / 4) / qmin;                     // warps in proportion to the source's width
    for (int ph = 0; ph < cnt; ++ph) {
      if (nw >= WOPN_MAX_WARPS) return false;
      p->w_seg[nw] = s; p->w_phase[nw] = ph; p->w_nphase[nw] = cnt; ++nw;
    }
  }
  if (p->w_seg[0] != 0) return false;
  p->nwarp = nw; p->N = k.Cout; p->ld = (k.Cout + 3) / 4 * 4;
  p->kd_pad = (GS + 1) * 4; p->bias_row = GS * 4; p->M = k.M;
  *grid = (unsigned)sm_count() * (unsigned)(nw <= 4 ? 8 : (nw <= 8 ? 5 : 4));
  *GS_out = GS;
  return true;
}

bool wopn_wgrad_applicable(const GConvK& k, const float* G) {
  WopnParams p; unsigned grid; int GS;
  return wopn_plan(k, G, &p, &grid, &GS);
}

size_t wopn_wgrad_ws_floats(const GConvK& k) {
  WopnParams p; unsigned grid; int GS;
  return wopn_plan(k, nullptr, &p, &grid, &GS) ? (size_t)grid * p.kd_pad * p.ld : 0;
}

int launch_wopn_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  WopnParams p; unsigned grid; int GS;
  if (!wopn_plan(k, G, &p, &grid, &GS)) return set_err(NLT_ERR_INVALID, "wopn_wgrad not applicable");
  w->g = k; w->GS = GS; w->KG = GS + 1; w->ld = p.ld; w->nsplit = (int)grid; w->pix_per_split = 0;
  *KD_pad = (size_t)p.kd_pad;
  const unsigned thr = (unsigned)p.nwarp * 32u;
  switch (p.N) {
    case 1: wopn_wgrad_kernel<1><<<grid, thr, 0, st>>>(p, G, ws); break;
    case 2: wopn_wgrad_kernel<2><<<grid, thr, 0, st>>>(p, G, ws); break;
    case 3: wopn_wgrad_kernel<3><<<grid, thr, 0, st>>>(p, G, ws); break;
    default: wopn_wgrad_kernel<4><<<grid, thr, 0, st>>>(p, G, ws); break;
  }
  NLT_CUDA_LAUNCH_CHECK("wopn_wgrad_kernel");
  return NLT_OK;
}

bool wop_wgrad_applicable(const GConvK& k, const float* G) { return wop_plan(k, G).ok; }

size_t wop_wgrad_ws_floats(const GConvK& k) {
  WopPlan pl = wop_plan(k, nullptr);
  return pl.ok ? (size_t)pl.grid * pl.p.kd_pad * pl.p.ld : 0;
}

int launch_wop_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  WopPlan pl = wop_plan(k, G);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "wop_wgrad not applicable");
  w->g = k; w->GS = pl.GS; w->KG = pl.KG; w->ld = pl.p.ld; w->nsplit = (int)pl.grid; w->pix_per_split = 0;
  *KD_pad = (size_t)pl.p.kd_pad;
  wop_wgrad_kernel<<<pl.grid, pl.p.ntask * 32, 0, st>>>(pl.p, ws);
  NLT_CUDA_LAUNCH_CHECK("wop_wgrad_kernel");
  return NLT_OK;
}

}  // namespace nlt
