// TEST INFRASTRUCTURE (never linked into the product library): runs the per-element functions of
// neural-light-transport_b200/csrc/nlt_barron_core.h -- the exact code the CUDA kernels of nlt_barron.cu call -- in
// plain host loops with the same buffers and the same pass order, so that the index arithmetic (reflecting
// boundaries, odd sizes, the adjoint gather) can be checked against the pinned oracle without a GPU.
// Built on the fly by tests/test_barron_core.py:  g++ -O2 -shared -fPIC -I<csrc> barron_host_check.cpp
#include <cmath>
#include <cstdint>
#include <vector>

#include "nlt_barron_core.h"

using namespace nlt_barron;

namespace {

struct Level {
  int A, B;
  std::vector<float> img, L, H, LH, HL, HH;
};

void rows_pass(const std::vector<float>& x, int P, int A, int B, std::vector<float>& lo, std::vector<float>& hi) {
  const int nl = n_lo(A), nh = n_hi(A);
  lo.assign((size_t)P * nl * B, 0.f);
  hi.assign((size_t)P * nh * B, 0.f);
  for (int p = 0; p < P; ++p)
    for (int j = 0; j < nl; ++j)
      for (int c = 0; c < B; ++c) {
        const float* col = x.data() + (size_t)p * A * B + c;
        lo[((size_t)p * nl + j) * B + c] = analysis_lo(col, A, B, j);
        if (j < nh) hi[((size_t)p * nh + j) * B + c] = analysis_hi(col, A, B, j);
      }
}

// returns the loss contribution of the bands produced here; bands are replaced by their gradients
void cols_pass(const std::vector<float>& src, int P, int R, int B, std::vector<float>& out_lo, std::vector<float>& out_hi,
               bool keep_lo, float inv_scale, float gscale, std::vector<double>& loss_acc) {
  const int nl = n_lo(B), nh = n_hi(B);
  out_lo.assign((size_t)P * R * nl, 0.f);
  out_hi.assign((size_t)P * R * nh, 0.f);
  for (int p = 0; p < P; ++p)
    for (int r = 0; r < R; ++r)
      for (int j = 0; j < nl; ++j) {
        const float* row = src.data() + ((size_t)p * R + r) * B;
        const float l = analysis_lo(row, B, 1, j);
        if (keep_lo) {
          out_lo[((size_t)p * R + r) * nl + j] = l;
        } else {
          loss_acc[p / 3] += charbonnier(l, inv_scale);
          out_lo[((size_t)p * R + r) * nl + j] = gscale * charbonnier_grad(l, inv_scale);
        }
        if (j < nh) {
          const float h = analysis_hi(row, B, 1, j);
          loss_acc[p / 3] += charbonnier(h, inv_scale);
          out_hi[((size_t)p * R + r) * nh + j] = gscale * charbonnier_grad(h, inv_scale);
        }
      }
}

}  // namespace

extern "C" int barron_host(const float* pred, const float* gt, const float* alpha, int32_t Bn, int32_t H, int32_t W,
                           int32_t levels, float scale, float log_z, float loss_scale, float* loss, float* d_pred) {
  const int P = 3 * Bn;
  const long long hw = (long long)H * W;
  const float inv_scale = 1.f / scale, inv_count = 1.f / (float)(hw * 3), gscale = loss_scale * inv_count;
  std::vector<Level> lv(levels + 1);
  lv[0].A = H; lv[0].B = W;
  lv[0].img.assign((size_t)P * hw, 0.f);
  for (long long idx = 0; idx < (long long)Bn * hw; ++idx) {
    const long long b = idx / hw, p = idx - b * hw;
    const float a = alpha ? alpha[idx] : 1.f;
    float y, u, v;
    rgb_to_syuv((gt[idx * 3] - pred[idx * 3]) * a, (gt[idx * 3 + 1] - pred[idx * 3 + 1]) * a,
                (gt[idx * 3 + 2] - pred[idx * 3 + 2]) * a, &y, &u, &v);
    lv[0].img[(b * 3 + 0) * hw + p] = y;
    lv[0].img[(b * 3 + 1) * hw + p] = u;
    lv[0].img[(b * 3 + 2) * hw + p] = v;
  }
  std::vector<double> acc(Bn, 0.0);
  for (int l = 0; l < levels; ++l) {
    Level& c = lv[l];
    rows_pass(c.img, P, c.A, c.B, c.L, c.H);
    lv[l + 1].A = n_lo(c.A); lv[l + 1].B = n_lo(c.B);
    cols_pass(c.L, P, n_lo(c.A), c.B, lv[l + 1].img, c.LH, true, inv_scale, gscale, acc);
    cols_pass(c.H, P, n_hi(c.A), c.B, c.HL, c.HH, false, inv_scale, gscale, acc);
  }
  Level& top = lv[levels];
  for (size_t i = 0; i < top.img.size(); ++i) {
    const int p = (int)(i / ((size_t)top.A * top.B));
    acc[p / 3] += charbonnier(top.img[i], inv_scale);
    top.img[i] = gscale * charbonnier_grad(top.img[i], inv_scale);
  }
  const float constant = std::log(scale) + log_z;             // formed as the kernel forms it
  for (int b = 0; b < Bn; ++b) loss[b] = (float)(acc[b] * (double)inv_count) + constant;
  if (!d_pred) return 0;
  for (int l = levels - 1; l >= 0; --l) {
    Level& c = lv[l];
    const int A = c.A, B = c.B, nlA = n_lo(A), nhA = n_hi(A), nlB = n_lo(B), nhB = n_hi(B);
    std::vector<float> dL((size_t)P * nlA * B), dH((size_t)P * nhA * B);
    for (int p = 0; p < P; ++p) {
      for (int r = 0; r < nlA; ++r)
        for (int i = 0; i < B; ++i) {
          const size_t pr = (size_t)p * nlA + r;
          dL[pr * B + i] = adjoint_at(lv[l + 1].img.data() + pr * nlB, c.LH.data() + pr * nhB, B, 1, 1, i);
        }
      for (int r = 0; r < nhA; ++r)
        for (int i = 0; i < B; ++i) {
          const size_t pr = (size_t)p * nhA + r;
          dH[pr * B + i] = adjoint_at(c.HL.data() + pr * nlB, c.HH.data() + pr * nhB, B, 1, 1, i);
        }
    }
    std::vector<float> dimg((size_t)P * A * B);
    for (int p = 0; p < P; ++p)
      for (int i = 0; i < A; ++i)
        for (int col = 0; col < B; ++col)
          dimg[((size_t)p * A + i) * B + col] =
              adjoint_at(dL.data() + (size_t)p * nlA * B + col, dH.data() + (size_t)p * nhA * B + col, A, B, B, i);
    c.img.swap(dimg);
  }
  for (long long idx = 0; idx < (long long)Bn * hw; ++idx) {
    const long long b = idx / hw, p = idx - b * hw;
    float r, g, bl;
    syuv_to_rgb_transpose(lv[0].img[(b * 3 + 0) * hw + p], lv[0].img[(b * 3 + 1) * hw + p], lv[0].img[(b * 3 + 2) * hw + p],
                          &r, &g, &bl);
    const float a = alpha ? -alpha[idx] : -1.f;
    d_pred[idx * 3 + 0] = a * r;
    d_pred[idx * 3 + 1] = a * g;
    d_pred[idx * 3 + 2] = a * bl;
  }
  return 0;
}

// single steps, for direct comparison with the golden pyramid
extern "C" void barron_host_analysis(const float* x, int32_t n, float* lo, float* hi) {
  for (int j = 0; j < n_lo(n); ++j) lo[j] = analysis_lo(x, n, 1, j);
  for (int j = 0; j < n_hi(n); ++j) hi[j] = analysis_hi(x, n, 1, j);
}
extern "C" void barron_host_adjoint(const float* g_lo, const float* g_hi, int32_t n, float* dx) {
  for (int i = 0; i < n; ++i) dx[i] = adjoint_at(g_lo, g_hi, n, 1, 1, i);
}
