// Per-element arithmetic of the "barron" loss term (nlt/losses.py:90-121 -> third_party/robust_loss): shared by the
// CUDA kernels (nlt_barron.cu) and by the host-compiled checker the CPU tests build from this same header
// (tests/barron_host_check.cpp).  Plain C++ -- no CUDA headers -- so that g++ can compile it too.
//
//   residual (gt - pred)[* alpha]  ->  volume-preserving YUV (util.py:97-115)
//   -> 5-level CDF 9/7 analysis, reflecting boundaries (wavelet.py:33-94, 170-218, 293-334)
//   -> Charbonnier NLL per coefficient: sqrt((w/c)^2 + 1) - 1 + log c + log Z(1)   (general.py:96-122, distribution.py:181-222)
//      (evaluated in a cancellation-free form, see charbonnier())
//
// One analysis step along an axis of length n:  out_lo[j] = sum_t lo[t] * x[R(2j     + t - 4)],  j < ceil(n/2)
//                                               out_hi[j] = sum_t hi[t] * x[R(2j + 1 + t - 3)],  j < floor(n/2)
// with R the reflecting index map (edge sample not repeated, any number of reflections).  The backward pass is
// the exact adjoint of that map, written as a gather: every input position i collects the (j, t) pairs whose
// padded position reflects onto i.
#pragma once

#if defined(__CUDACC__)
#define NLT_HD __host__ __device__ __forceinline__
#else
#define NLT_HD inline
#endif

namespace nlt_barron {

constexpr int LO_TAPS = 9, HI_TAPS = 7;
constexpr int LO_BELOW = 4, HI_BELOW = 3;     // (len - 1) / 2 samples of padding below; the hi filter also skips 1

NLT_HD float lo_tap(int t) {
  // symmetric CDF 9/7 analysis low-pass, centre at t = 4 (wavelet.py:56-64)
  const float h[5] = {0.852698679009f, 0.377402855613f, -0.110624404418f, -0.023849465020f, 0.037828455507f};
  const int d = t < 4 ? 4 - t : t - 4;
  return h[d];
}
NLT_HD float hi_tap(int t) {
  // symmetric CDF 9/7 analysis high-pass, centre at t = 3 (wavelet.py:65-71)
  const float h[4] = {0.788485616406f, -0.418092273222f, -0.040689417609f, 0.064538882629f};
  const int d = t < 3 ? 3 - t : t - 3;
  return h[d];
}

NLT_HD int n_lo(int n) { return (n + 1) / 2; }
NLT_HD int n_hi(int n) { return n / 2; }

// reflecting index map of a length-n axis (wavelet.py:135-147): q in (-inf, inf) -> [0, n)
NLT_HD int reflect(int q, int n) {
  if (n <= 1) return 0;
  const int period = 2 * (n - 1);
  int r = q % period;
  if (r < 0) r += period;
  return r < n ? r : period - r;
}

// ---- forward: one output sample, reading x with element stride `st` ----
NLT_HD float analysis_lo(const float* x, int n, int st, int j) {
  float acc = 0.f;
  for (int t = 0; t < LO_TAPS; ++t) acc += lo_tap(t) * x[(long long)reflect(2 * j + t - LO_BELOW, n) * st];
  return acc;
}
NLT_HD float analysis_hi(const float* x, int n, int st, int j) {
  float acc = 0.f;
  for (int t = 0; t < HI_TAPS; ++t) acc += hi_tap(t) * x[(long long)reflect(2 * j + 1 + t - HI_BELOW, n) * st];
  return acc;
}

// ---- backward: gradient of one INPUT sample i from the gradients of both outputs (exact adjoint) ----
// Padded positions used by the forward pass: q in [-4, n + 3].  Those that reflect onto i are q = +-i + m * period.
NLT_HD float adjoint_at(const float* g_lo, const float* g_hi, int n, int st_lo, int st_hi, int i) {
  const int nl = n_lo(n), nh = n_hi(n);
  if (n <= 1) {
    // every padded position maps to the single sample
    float acc = 0.f;
    for (int j = 0; j < nl; ++j) {
      float s = 0.f;
      for (int t = 0; t < LO_TAPS; ++t) s += lo_tap(t);
      acc += s * g_lo[(long long)j * st_lo];
    }
    for (int j = 0; j < nh; ++j) {
      float s = 0.f;
      for (int t = 0; t < HI_TAPS; ++t) s += hi_tap(t);
      acc += s * g_hi[(long long)j * st_hi];
    }
    return acc;
  }
  const int period = 2 * (n - 1);
  const int q_min = -LO_BELOW, q_max = n - 1 + LO_BELOW;     // widest padded range of the two filters
  float acc = 0.f;
  for (int sign = 0; sign < 2; ++sign) {
    if (sign == 1 && (i == 0 || i == n - 1)) break;          // +i and -i coincide modulo the period at the two edges
    const int base = sign == 0 ? i : -i;
    // smallest q = base + m * period that is >= q_min
    int m = (q_min - base) / period;
    while (base + m * period < q_min) ++m;
    while (base + (m - 1) * period >= q_min) --m;
    for (int q = base + m * period; q <= q_max; q += period) {
      // low-pass: q = 2j + t - 4  ->  t = q + 4 - 2j
      for (int t = 0; t < LO_TAPS; ++t) {
        const int two_j = q + LO_BELOW - t;
        if (two_j >= 0 && (two_j & 1) == 0 && (two_j >> 1) < nl) acc += lo_tap(t) * g_lo[(long long)(two_j >> 1) * st_lo];
      }
      // high-pass: q = 2j + 1 + t - 3  ->  t = q + 2 - 2j
      for (int t = 0; t < HI_TAPS; ++t) {
        const int two_j = q + HI_BELOW - 1 - t;
        if (two_j >= 0 && (two_j & 1) == 0 && (two_j >> 1) < nh) acc += hi_tap(t) * g_hi[(long long)(two_j >> 1) * st_hi];
      }
    }
  }
  return acc;
}

// ---- robust loss at alpha = 1 ----
// sqrt(z^2 + 1) - 1 written as z^2 / (sqrt(z^2 + 1) + 1): the same value without the cancellation that loses every
// digit of the difference below |z| ~ 1e-2 (a converged model's coefficients sit there)
NLT_HD float charbonnier(float w, float inv_scale) {
  const float z = w * inv_scale;
  const float z2 = z * z;
  return z2 / (sqrtf(z2 + 1.f) + 1.f);
}
NLT_HD float charbonnier_grad(float w, float inv_scale) {
  const float z = w * inv_scale;
  return z * inv_scale / sqrtf(z * z + 1.f);
}

// ---- colour: rgb -> scaled YUV and its transpose (tf.image.rgb_to_yuv matrix, util.py:97) ----
constexpr float SYUV = 1.580227820074f;
NLT_HD void rgb_to_syuv(float r, float g, float b, float* y, float* u, float* v) {
  *y = SYUV * (0.299f * r + 0.587f * g + 0.114f * b);
  *u = SYUV * (-0.14714119f * r - 0.28886916f * g + 0.43601035f * b);
  *v = SYUV * (0.61497538f * r - 0.51496512f * g - 0.10001026f * b);
}
NLT_HD void syuv_to_rgb_transpose(float gy, float gu, float gv, float* r, float* g, float* b) {
  *r = SYUV * (0.299f * gy - 0.14714119f * gu + 0.61497538f * gv);
  *g = SYUV * (0.587f * gy - 0.28886916f * gu - 0.51496512f * gv);
  *b = SYUV * (0.114f * gy + 0.43601035f * gu - 0.10001026f * gv);
}

}  // namespace nlt_barron
