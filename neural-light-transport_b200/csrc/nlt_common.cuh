// Shared device/host helpers for the NLT kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "nlt_b200.h"

namespace nlt {

// ---- thread-local error string (nlt_last_error) -----------------------------
extern thread_local char g_err[512];
int set_err(int code, const char* fmt, ...);
#define NLT_CHECK_ARG(cond, ...) \
  do { if (!(cond)) return nlt::set_err(NLT_ERR_INVALID, __VA_ARGS__); } while (0)
extern unsigned long long g_launches;   // kernels launched by this library (diagnostic only)
void count_launch(const char* what);    // per-kernel launch counter behind nlt_kernel_launch_count (diagnostic only)
#define NLT_CUDA_LAUNCH_CHECK(what) \
  do { __atomic_add_fetch(&nlt::g_launches, 1ull, __ATOMIC_RELAXED); nlt::count_launch(what); \
       cudaError_t e_ = cudaGetLastError(); \
       if (e_ != cudaSuccess) return nlt::set_err(NLT_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e_)); } while (0)

// SMs of the current device: grid caps of the grid-stride and persistent kernels (cached per device)
int sm_count();

// process-wide switches, in the order of the option table in nlt_gconv.cu (name, environment variable, default)
enum class Opt {
  TC, TC_WGRAD, WGRAD_ROWS, TCS, TC_RAWHI, TC_SPLIT_WAVES, PWX, PWMMA, TINY, DCONV_CW, DCONV_WIDE_FIRST, PF, PF_S1,
  PWD2S_FIRST, PF_NS, PWX_NS, WOP, DCONV_WIDE, DCONV_WIDE32, DCONV_WIDE8, COUNT
};
// the value of a switch: its environment variable or default on the first read, then whatever nlt_set_option stored
int opt(Opt o);

// two fp32 FMAs on a float pair (a * b + c per component, round-to-nearest)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// ---- 3xTF32 operand split (the wgmma kernels of nlt_tc.cu, the mma.sync kernels of nlt_pwx.cu) ----------------
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// Round-to-nearest TF32 in two integer instructions (cvt.rna.tf32 expands to several instructions with its inf/nan
// handling).  Adding half an ulp to the bit pattern and clearing the low 13 mantissa bits rounds the magnitude to
// nearest (ties away), carries into the exponent correctly, and is only wrong for inf/nan, which the split does not
// need to preserve.
__device__ __forceinline__ float tf32_round(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
// 3xTF32 split of one activation: hi = x truncated (rawhi) or rounded to TF32; lo = x - hi (exact), rounded to TF32
__device__ __forceinline__ void tf32_split(float x, int rawhi, uint32_t& hi, uint32_t& lo) {
  const float h = rawhi ? __uint_as_float(__float_as_uint(x) & 0xFFFFE000u) : tf32_round(x);
  hi = __float_as_uint(h);
  lo = __float_as_uint(tf32_round(x - h));
}

// ---- division by an invariant (Granlund-Montgomery), n < 2^31 ----------------
struct FastDiv {
  uint32_t d, m, l;
};
inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  f.d = d ? d : 1;
  uint32_t l = 0;
  while ((1ull << l) < f.d) ++l;
  f.l = l;
  f.m = (uint32_t)((((1ull << 32) * ((1ull << l) - f.d)) / f.d) + 1);
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, const FastDiv& f) {
  return (__umulhi(n, f.m) + n) >> f.l;
}

// ---- activation ---------------------------------------------------------------
// forward (nlt/networks/elements.py:69-78).  `act` is warp-uniform: the piecewise-linear cases cost
// three instructions per value; ELU (expm1f) sits behind a real call so that its ~30 instructions are
// not if-converted into every epilogue.
static __device__ __noinline__ float elu_slow(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ float act_fwd(float x, int act) {
  if (act == NLT_ACT_ELU) return elu_slow(x);
  const float neg = act == NLT_ACT_LEAKYRELU ? 0.3f : (act == NLT_ACT_RELU ? 0.f : 1.f);
  return x > 0.f ? x : neg * x;
}
// derivative recovered from the saved OUTPUT y (no pre-activation is stored)
__device__ __forceinline__ float act_bwd_from_y(float y, int act) {
  const float neg = act == NLT_ACT_LEAKYRELU ? 0.3f : (act == NLT_ACT_RELU ? 0.f : 1.f);
  return y > 0.f ? 1.f : (act == NLT_ACT_ELU ? y + 1.f : neg);
}

// One axis of the (phase-decomposed) gather map.
//   output coordinate  o = o0 + os * t      t in [0, nt)
//   tap index          d = d0 + ds * u      u in [0, nu)
//   input coordinate   i = t * it + u * iu + i0   (valid iff 0 <= i < n_in)
struct AxisMap {
  int o0, os, nt;
  int it, iu, i0;
  int d0, ds, nu;
  int n_in;
};

struct Seg {
  const float* ptr;
  const float* sub;
  int C;      // channels of this source
  int coff;   // channel offset inside the virtual concat (weight c index)
  int bcast;  // batch-broadcast
  int vec;    // 1: C % 4 == 0 and pointers 16B aligned -> float4 path
};

// Kernel-side description of one phase of a generalised convolution.
struct GConvK {
  AxisMap ay, ax;
  int N, Hin, Win, Hout, Wout, kw;
  int nseg;
  Seg seg[NLT_MAX_SEG];
  int Cout;
  const float* w;
  long long wt, wc, wn;
  uint32_t M;  // lattice pixels in this phase = N * ay.nt * ax.nt
  FastDiv div_x, div_yx;
  // depth-to-space mode (transposed op with k == stride, no padding): ONE pass over
  // the input lattice with N' = k*k*cout_true GEMM columns (n' = tap*cout_true + n),
  // each 4-channel group stored at output pixel (t*s + dy, t*s + dx).  Cout == N'.
  int d2s, d2s_s, cout_true;
  FastDiv div_ct, div_s;   // by cout_true / by d2s_s (tap decode without integer division)
};

__device__ __forceinline__ void decode_pixel(const GConvK& g, uint32_t m, int& n, int& ty, int& tx) {
  uint32_t q = fdiv(m, g.div_yx);
  uint32_t r = m - q * g.div_yx.d;
  uint32_t y = fdiv(r, g.div_x);
  n = (int)q;
  ty = (int)y;
  tx = (int)(r - y * g.div_x.d);
}

// build the per-phase kernel descriptors of a public descriptor (host).
// allow_d2s: fold a k == stride transposed op into one depth-to-space phase.
int build_phases(const nlt_gconv_desc* d, GConvK* out, int* nphase, bool allow_d2s = false);

static __host__ __device__ inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---- wgrad descriptors shared by the tiled and the warp-stream kernels ------------
struct WgradK {
  GConvK g;
  int GS;        // k-groups (4 channels each) per tap
  int KG;        // total k-groups incl. the trailing bias group
  int ld;        // padded Cout (multiple of 4) = workspace row stride
  int nsplit;
  uint32_t pix_per_split;
};

// k-group -> (tap uy,ux ; segment s ; first channel c); s = -1 bias group, -2 padding
__device__ __forceinline__ void decode_kgroup(const WgradK& w, int kg, int& uy, int& ux, int& s, int& c) {
  if (kg >= w.KG) { s = -2; uy = ux = c = 0; return; }
  if (kg == w.KG - 1) { s = -1; uy = ux = c = 0; return; }
  const int tap = kg / w.GS;
  int gs = kg - tap * w.GS;
  uy = tap / w.g.ax.nu; ux = tap - uy * w.g.ax.nu;
  s = 0;
  while (s < w.g.nseg - 1 && gs >= (w.g.seg[s].C + 3) / 4) { gs -= (w.g.seg[s].C + 3) / 4; ++s; }
  c = gs * 4;
}

// specialised small-channel kernels (nlt_small.cu); return NLT_OK or an error
// second, pointwise term of the pointwise kernel's epilogue (see pw_conv_kernel)
constexpr int PW_EX_KMAX = 4;
struct PwExtra {
  const float* x;      // [output pixels][K]
  int K;
  const float* w;      // w[k * wk + c * wn], c < cout_true
  long long wk, wn;
};
bool pw_conv_applicable(const GConvK& k);
bool pw_extra_applicable(const GConvK& k, const PwExtra& ex, const float* out, const float* mask_y);
int launch_pw_conv(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                   float* out, cudaStream_t st, const PwExtra* ex = nullptr);
// wide stencil kernel (pixel x 16, 32 or 8 outputs per thread; options "dconv_wide", "dconv_wide32", "dconv_wide8")
bool dconv_wide_applicable(const GConvK& k, const float* out, const float* mask_y);
int launch_dconv_wide(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                      float* out, cudaStream_t st);
bool dconv_small_applicable(const GConvK& k);
int launch_dconv_small(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                       float* out, cudaStream_t st);
bool wgrad_small_applicable(const GConvK& k);
size_t wgrad_small_ws_floats(const GConvK& k);
// fills w (nsplit, pix_per_split, ld, KG, GS) and *KD_pad for the reduce stage
int launch_wgrad_small(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);

bool wgrad_tpp_applicable(const GConvK& k);
size_t wgrad_tpp_ws_floats(const GConvK& k);
int launch_wgrad_tpp(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);

// wide pointwise conv into 16 channels (nlt_pwx.cu): level 0 of the 64-channel query stack
bool wopn_wgrad_applicable(const GConvK& k, const float* G);
size_t wopn_wgrad_ws_floats(const GConvK& k);
int launch_wopn_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);
bool wop_wgrad_applicable(const GConvK& k, const float* G);
size_t wop_wgrad_ws_floats(const GConvK& k);
int launch_wop_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);
bool tiny_stencil_applicable(const GConvK& k, const float* out, const float* mask_y);
int launch_tiny_stencil(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act,
                        float* out, cudaStream_t st);
bool pwx_fwd_applicable(const GConvK& k, float beta, const float* mask_y, const float* out);
int launch_pwx_fwd(const GConvK& k, const float* bias, int act, float* out, cudaStream_t st);
bool pf_fwd_applicable(const GConvK& k, const float* mask_y, const float* out);
int launch_pf_fwd(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act, float* out,
                  cudaStream_t st);
bool pwx_d2s_fwd_applicable(const GConvK& k, float beta, const float* mask_y, const float* out);
int launch_pwx_d2s_fwd(const GConvK& k, const float* bias, int act, float* out, cudaStream_t st);
bool pwx_wgrad_applicable(const GConvK& k, const float* G);
size_t pwx_wgrad_ws_floats(const GConvK& k);
int launch_pwx_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);

// input gradient of the 2x2 / stride-2 convs into 16-channel sources (depth-to-space pointwise op, nlt_pwx.cu)
bool pwd2s_applicable(const GConvK& k, const float* bias, int act, const float* out, const float* mask_y,
                      const PwExtra* ex);
int launch_pwd2s(const GConvK& k, float beta, const float* mask_y, int mask_act, float* out, cudaStream_t st,
                 const PwExtra* ex);
// the same op on the tensor cores (mma.sync 3xTF32), for every shape pwd2s_applicable accepts; option "pwmma"
int launch_pwd2s_mma(const GConvK& k, float beta, const float* mask_y, int mask_act, float* out, cudaStream_t st,
                     const PwExtra* ex);

// weight gradient of the 2x2 convs of the 16- / 32-channel levels (staged input patch, nlt_pwx.cu)
bool pws_wgrad_applicable(const GConvK& k, const float* G);
size_t pws_wgrad_ws_floats(const GConvK& k);
int launch_pws_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);

// wgmma tensor-core path (nlt_tc.cu)
extern unsigned long long g_tc_launches;
// partial_tiles: also lattices that are not a multiple of the tile shape (edge tiles partly masked)
bool tc_applicable(const GConvK& k, bool partial_tiles = false);
size_t tc_workspace_bytes(const GConvK& k, bool partial_tiles = false);
int launch_tc(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act, float* out,
              void* workspace, size_t workspace_bytes, cudaStream_t st, bool prepacked = false, bool partial_tiles = false);
int tc_pack(const GConvK& k, void* workspace, size_t workspace_bytes, cudaStream_t st, bool partial_tiles = false);

// A forward or input-gradient op of the public descriptor form, routed as nlt_gconv_fwd_ws routes it, for the library's
// own composite ops (nlt_lpips.cu).  partial_tiles: the wgmma kernel also takes lattices that are not a multiple of
// its tile shape.  gconv_tc_workspace_bytes: the scratch that op needs on the wgmma kernel (0 when it cannot run there).
int gconv_run(const nlt_gconv_desc* d, const float* bias, int act, float beta, const float* mask_y, int mask_act,
              float* out, void* workspace, int64_t workspace_bytes, bool partial_tiles, cudaStream_t st);
int64_t gconv_tc_workspace_bytes(const nlt_gconv_desc* d, bool partial_tiles);

bool tc_wgrad_applicable(const GConvK& k);
size_t tc_wgrad_ws_floats(const GConvK& k);
int launch_tc_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st);

}  // namespace nlt
