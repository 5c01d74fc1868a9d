// wgmma tensor-core path of the generalised convolution (sm_90a).
//
// Implicit GEMM  D[128 pixels x BN] += A[128 pixels x KBW ch] * B[KBW ch x BN]  per K-block, where a K-block is
// (tap, segment, KBW-channel chunk).  No im2col: for every tap the A tile is ONE TMA box of the NHWC activation
// tensor, [TH x TW pixels] x [KBW channels], landing in shared memory as 128 rows of 128 B (KBW = 32, 128-byte
// swizzle) or 64 B (KBW = 16, 64-byte swizzle) -- the K-major operand layout wgmma reads.  SAME padding is TMA
// out-of-bounds zero fill (coordinates may be negative); the k == stride "patch" conv is a 5-D view of the same
// tensor (c, dx, x/s, dy, n*H/s + y/s) so that no element stride is needed.
//
// fp32-class accuracy on TF32 tensor cores: 3xTF32.  Weights are split once per call into hi/lo TF32 planes (pack
// kernel); activations are split by the consumer warpgroups (hi = x truncated or rounded to TF32, lo = x - hi
// rounded to TF32) and every 8-channel k-step issues D += Alo*Bhi + Ahi*Blo + Ahi*Bhi with fp32 accumulation in
// registers.
//
// Warp roles (384 threads, 1 CTA / SM, persistent over output tiles):
//   warpgroup 0      warp 0, one thread: TMA producer (A raw tile + Bhi + Blo per stage, mbarrier complete_tx)
//   warpgroups 1-2   consumers of rows [0, 64) / [64, 128) of the tile: operand split, wgmma m64nBNk8, epilogue
// The producer runs ahead into the next tile's stages while the consumers drain their accumulators.
// Two forms of the A operand (option "tcs"): RS = fragments read from the raw tile and split in registers (wgmma
// with A in registers, nothing written back to shared memory); SS = the consumer warpgroup writes hi / lo planes
// of its 64 rows into shared memory (wgmma with both operands in shared memory).
#include <cuda.h>
#include "nlt_common.cuh"

namespace nlt {

constexpr int TC_MAX_STAGES = 8;                // smem ring depth is chosen per shape (2..8): bytes in flight, not math, bound most layers
constexpr int TC_BM = 128;
constexpr int TC_EPI_PAD = 36;                  // floats per staging row (32 columns + 4 pad)
constexpr int TC_EPI_BYTES = 8 * 16 * TC_EPI_PAD * 4;   // epilogue staging: 8 consumer warps x 16 rows
constexpr int TC_THREADS = 384;                 // producer warpgroup + two consumer warpgroups (both kernels)
constexpr uint32_t TC_SPIN_LIMIT = 1u << 28;    // watchdog: trap instead of hanging the GPU
unsigned long long g_tc_launches = 0;           // tensor-core kernel launches (diagnostic)

struct TcParams {
  // lattice / tiling
  int N, Hl, Wl;            // lattice size (pixels this kernel enumerates)
  int TW, TH;               // tile = TH x TW lattice pixels (TW*TH == 128)
  int tiles_x, tiles_y;     // per image
  int n_tiles_n;            // column tiles (Cout / BN)
  int total_tiles;          // N * tiles_y * tiles_x * n_tiles_n
  // K-blocks
  int ntap_y, ntap_x;
  int nseg;
  int seg_chunks[NLT_MAX_SEG];
  int kb_total;
  // TMA coordinate maps: x = tx0*mx + ux*ux_step + x_off (mode A); mode B (patch) uses (ux, tx0, uy, n*Hs + ty0)
  int mode_patch;           // 1: 5-D patch view
  int ux_step, x_off, uy_step, y_off;
  int Hs;                   // mode B: H / s  (rows of the merged n*H/s dimension per image)
  // output
  int Hout, Wout, cout_true, Cout;   // Cout = GEMM columns (d2s: s*s*cout_true)
  int o0y, osy, o0x, osx;            // output pixel = o0 + os * lattice coordinate (non-d2s)
  int d2s, d2s_s;
  // exact multiply-shift division by the run-time tile / channel counts (per-tile coordinate decode of the producer,
  // per-pass address arithmetic of the epilogue): no 32-bit integer division on the critical path of a tile
  FastDiv div_ntn, div_tpi, div_tx, div_tw, div_ct, div_s;
  int act, mask_act;
  int stages;               // smem ring depth
  int rawhi;                // option "tc_rawhi" / NLT_TC_RAWHI (default 1): A-hi = x truncated to TF32 (0: rounded)
  float beta;
  const float* bias;
  const float* mask_y;
  float* out;
};

// ---------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > TC_SPIN_LIMIT) { asm volatile("trap;"); }
  }
}
// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}

// ---- wgmma (m64nNk8, TF32 inputs, fp32 accumulators in registers) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int NR>
__device__ __forceinline__ void acc_fence(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A * B; scale_d == 0 overwrites D.  SS: A and B from shared-memory descriptors; RS: A from registers
// (per warp a 16 x 8 slice: a[0] = (g, t), a[1] = (g + 8, t), a[2] = (g, t + 4), a[3] = (g + 8, t + 4), g = lane / 4,
// t = lane % 4).  D: d[4j + 2h + e] = (row g + 8h, column 8j + 2t + e) of the warp's 16 rows.
__device__ __forceinline__ void wgmma_ss(float (&d)[8], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// K-major swizzled operand tile: rows of ROWB bytes (128 -> SWIZZLE_128B, 64 -> SWIZZLE_64B), 8-row core matrices.
// Stepping K by 8 TF32 values inside the swizzle atom advances the start address by 32 bytes.
template <int ROWB>
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // start address
  d |= (uint64_t)1 << 16;                             // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)((8 * ROWB) >> 4) << 32;             // stride byte offset: 8 rows
  d |= (uint64_t)(ROWB == 128 ? 1 : 2) << 62;         // SWIZZLE_128B / SWIZZLE_64B
  return d;
}

// ---------------------------------------------------------------------------------------------
// weight pack: Bhi/Blo [kb][Cout_pad][KBW] (K-major rows), TF32-rounded split
// ---------------------------------------------------------------------------------------------
__global__ void tc_pack_weights_kernel(const GConvK g, int kbw, int kb_total, int chunks_per_tap, int cout_pad,
                                       float* __restrict__ bhi, float* __restrict__ blo) {
  const size_t total = (size_t)kb_total * cout_pad * kbw;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int kk = (int)(i % kbw);
    const int n = (int)((i / kbw) % cout_pad);
    const int kb = (int)(i / ((size_t)kbw * cout_pad));
    const int tapi = kb / chunks_per_tap;
    int ch = kb - tapi * chunks_per_tap;
    int s = 0;
    while (s < g.nseg - 1 && ch >= g.seg[s].C / kbw) { ch -= g.seg[s].C / kbw; ++s; }
    const int c = g.seg[s].coff + ch * kbw + kk;
    const int uy = tapi / g.ax.nu, ux = tapi - uy * g.ax.nu;
    float v = 0.f;
    if (n < g.Cout) {
      int tap = (g.ay.d0 + g.ay.ds * uy) * g.kw + (g.ax.d0 + g.ax.ds * ux), nn = n;
      if (g.d2s) { tap = n / g.cout_true; nn = n - tap * g.cout_true; }
      v = __ldg(g.w + (long long)tap * g.wt + (long long)c * g.wc + (long long)nn * g.wn);
    }
    const float hi = tf32_rna(v);
    bhi[i] = hi;
    blo[i] = tf32_rna(v - hi);
  }
}

// ---------------------------------------------------------------------------------------------
// main kernel
// ---------------------------------------------------------------------------------------------
struct TcMaps {
  CUtensorMap a[NLT_MAX_SEG];
  CUtensorMap bhi, blo;
};

template <int BN, int KBW, bool RS>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gconv_kernel(const __grid_constant__ TcMaps maps, const TcParams p) {
  constexpr int ROWB = KBW * 4;                   // bytes per operand row
  constexpr int KS = KBW / 8;                     // k-steps per K-block
  constexpr int A_BYTES = TC_BM * ROWB;
  constexpr int A_HALF = 64 * ROWB;               // one consumer warpgroup's rows
  constexpr int B_BYTES = BN * ROWB;
  constexpr int A_PLANES = RS ? 1 : 2;            // raw tile (RS) / hi + lo planes (SS)
  constexpr int STAGE_BYTES = A_PLANES * A_BYTES + 2 * B_BYTES;

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle
  // offset arithmetic on the __shared__ array keeps the address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t bars[2 * TC_MAX_STAGES];
  const int S = p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar0 = smem_u32(bars);
  auto bar_full = [&](int s) { return bar0 + 8u * s; };
  auto bar_empty = [&](int s) { return bar0 + 8u * (TC_MAX_STAGES + s); };
  const uint32_t smem_base = smem_u32(smem);
  auto a_hi = [&](int s) { return smem_base + (uint32_t)s * STAGE_BYTES; };
  auto b_hi = [&](int s) { return smem_base + (uint32_t)s * STAGE_BYTES + A_PLANES * A_BYTES; };
  auto b_lo = [&](int s) { return smem_base + (uint32_t)s * STAGE_BYTES + A_PLANES * A_BYTES + B_BYTES; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), 8);                  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int kb_total = p.kb_total;
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  if (warp < 4) {
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int mt = (int)fdiv((uint32_t)tile, p.div_ntn);
        const int nt = tile - mt * p.n_tiles_n;
        const int n = (int)fdiv((uint32_t)mt, p.div_tpi);
        const int r = mt - n * tiles_per_img;
        const int rq = (int)fdiv((uint32_t)r, p.div_tx);
        const int ty0 = rq * p.TH, tx0 = (r - rq * p.tiles_x) * p.TW;
        int kb = 0;
        for (int uy = 0; uy < p.ntap_y; ++uy)
          for (int ux = 0; ux < p.ntap_x; ++ux)
            for (int s = 0; s < p.nseg; ++s)
              for (int ch = 0; ch < p.seg_chunks[s]; ++ch, ++kb) {
                mbar_wait(bar_empty(stage), phase ^ 1);
                mbar_expect_tx(bar_full(stage), A_BYTES + 2 * B_BYTES);
                if (p.mode_patch)
                  tma_load_5d(a_hi(stage), &maps.a[s], bar_full(stage), ch * KBW, ux, tx0, uy, n * p.Hs + ty0);
                else
                  tma_load_4d(a_hi(stage), &maps.a[s], bar_full(stage), ch * KBW, tx0 + ux * p.ux_step + p.x_off,
                              ty0 + uy * p.uy_step + p.y_off, n);
                tma_load_3d(b_hi(stage), &maps.bhi, bar_full(stage), 0, nt * BN, kb);
                tma_load_3d(b_lo(stage), &maps.blo, bar_full(stage), 0, nt * BN, kb);
                if (++stage == S) { stage = 0; phase ^= 1; }
              }
      }
    }
    return;
  }

  // ================= consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =================
  const int wg = (warp >> 2) - 1;
  const int wq = warp & 3;                        // warp inside the warpgroup: rows [64 wg + 16 wq, +16)
  const int g = lane >> 2, t = lane & 3;
  const int r0 = 64 * wg + 16 * wq + g;           // this thread's accumulator rows: r0, r0 + 8
  // RS: physical 16-byte chunk of logical chunk c in rows r0 / r0 + 8 (the same for both: TMA swizzle by row)
  auto swz = [&](int c) { return ROWB == 128 ? (c ^ (r0 & 7)) : (c ^ ((r0 >> 1) & 3)); };

  // epilogue geometry: accumulator -> bias / activation -> per-warp smem staging [16 rows x 32 columns] -> transposed
  // read (QPR lanes = one pixel's contiguous columns) -> beta / derivative mask -> coalesced float4 stores
  float* stg = reinterpret_cast<float*>(smem + (size_t)S * STAGE_BYTES) + (warp - 4) * 16 * TC_EPI_PAD;
  const bool rmw = (p.beta != 0.f) || (p.mask_y != nullptr);
  constexpr int NCH = (BN + 31) / 32;             // 32-column chunks per tile (BN == 16: one half-used chunk)
  constexpr int CW = BN < 32 ? BN : 32;           // columns per chunk
  constexpr int QPR = CW / 4;                     // float4 quads per pixel row of a chunk
  constexpr int RPI = 32 / QPR;                   // pixel rows covered per pass of the warp
  constexpr int NPASS = 16 / RPI;                 // passes per chunk
  const int lq = lane % QPR, lr = lane / QPR;
  // output offset(tile, pass i, column) = tile base + row_off[i] + col_off(column): row_off depends only on the lane
  const int sxy = p.d2s ? p.d2s_s : 1;
  int row_off[NPASS], row_y[NPASS], row_x[NPASS];   // row_y / row_x: the pass's pixel inside the tile
#pragma unroll
  for (int i = 0; i < NPASS; ++i) {
    const int row = 64 * wg + 16 * wq + i * RPI + lr;
    const int rty = (int)fdiv((uint32_t)row, p.div_tw), rtx = row - rty * p.TW;
    row_y[i] = rty; row_x[i] = rtx;
    row_off[i] = p.d2s ? (rty * sxy * p.Wout + rtx * sxy) * p.cout_true
                       : (p.osy * rty * p.Wout + p.osx * rtx) * p.cout_true;
  }
  // tile origin -> output offset of its first pixel; rem_y / rem_x: lattice rows / columns left from the origin (the
  // last tiles of a lattice that is not a multiple of the tile shape are partly outside it)
  auto tile_base = [&](int tile, int& nt, int& rem_y, int& rem_x) -> size_t {
    const int mt = (int)fdiv((uint32_t)tile, p.div_ntn);
    nt = tile - mt * p.n_tiles_n;
    const int n = (int)fdiv((uint32_t)mt, p.div_tpi);
    const int r = mt - n * tiles_per_img;
    const int rq = (int)fdiv((uint32_t)r, p.div_tx);
    const int ty0 = rq * p.TH, tx0 = (r - rq * p.tiles_x) * p.TW;
    rem_y = p.Hl - ty0; rem_x = p.Wl - tx0;
    const int oy = p.d2s ? ty0 * sxy : p.o0y + p.osy * ty0, ox = p.d2s ? tx0 * sxy : p.o0x + p.osx * tx0;
    return (((size_t)n * p.Hout + oy) * p.Wout + ox) * p.cout_true;
  };
  // offset of GEMM column nb inside an output pixel group (d2s: which of the s x s pixels, which channel)
  auto col_off = [&](int nb) -> int {
    if (!p.d2s) return nb;
    const int tap = (int)fdiv((uint32_t)nb, p.div_ct);
    const int dy = (int)fdiv((uint32_t)tap, p.div_s);
    return (dy * p.Wout + (tap - dy * p.d2s_s)) * p.cout_true + (nb - tap * p.cout_true);
  };
  const int act = p.act;
  const float neg = act == NLT_ACT_LEAKYRELU ? 0.3f : (act == NLT_ACT_RELU ? 0.f : 1.f);

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    for (int kb = 0; kb < kb_total; ++kb) {
      mbar_wait(bar_full(stage), phase);
      const uint32_t bh0 = b_hi(stage), bl0 = b_lo(stage);
      if constexpr (RS) {
        const uint8_t* at = smem + (size_t)stage * STAGE_BYTES + (size_t)r0 * ROWB + t * 4;
        uint32_t ah[KS][4], al[KS][4];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float x = *reinterpret_cast<const float*>(at + (e & 1) * 8 * ROWB + swz(2 * ks + (e >> 1)) * 16);
            tf32_split(x, p.rawhi, ah[ks][e], al[ks][e]);
          }
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          const uint64_t bh = wgmma_desc<ROWB>(bh0 + ks * 32), bl = wgmma_desc<ROWB>(bl0 + ks * 32);
          wgmma_rs(acc, al[ks], bh, (kb | ks) != 0);   // small terms first
          wgmma_rs(acc, ah[ks], bl, 1);
          wgmma_rs(acc, ah[ks], bh, 1);
        }
      } else {
        // split this warpgroup's 64 rows: the raw tile becomes the hi plane in place, lo goes to the second plane
        // (elementwise over physical 16-byte chunks: swizzle-agnostic)
        float4* ah = reinterpret_cast<float4*>(smem + (size_t)stage * STAGE_BYTES + wg * A_HALF);
        float4* al = reinterpret_cast<float4*>(smem + (size_t)stage * STAGE_BYTES + A_BYTES + wg * A_HALF);
        const int tw = threadIdx.x - 128 - 128 * wg;
#pragma unroll
        for (int i = 0; i < A_HALF / 16 / 128; ++i) {
          const int q = tw + i * 128;
          const float4 v = ah[q];
          uint32_t h[4], l[4];
          tf32_split(v.x, p.rawhi, h[0], l[0]); tf32_split(v.y, p.rawhi, h[1], l[1]);
          tf32_split(v.z, p.rawhi, h[2], l[2]); tf32_split(v.w, p.rawhi, h[3], l[3]);
          ah[q] = make_float4(__uint_as_float(h[0]), __uint_as_float(h[1]), __uint_as_float(h[2]), __uint_as_float(h[3]));
          al[q] = make_float4(__uint_as_float(l[0]), __uint_as_float(l[1]), __uint_as_float(l[2]), __uint_as_float(l[3]));
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma reads
        named_bar_sync(1 + wg, 128);
        const uint32_t ahi0 = a_hi(stage) + wg * A_HALF, alo0 = ahi0 + A_BYTES;
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          const uint64_t dah = wgmma_desc<ROWB>(ahi0 + ks * 32), dal = wgmma_desc<ROWB>(alo0 + ks * 32);
          const uint64_t bh = wgmma_desc<ROWB>(bh0 + ks * 32), bl = wgmma_desc<ROWB>(bl0 + ks * 32);
          wgmma_ss(acc, dal, bh, (kb | ks) != 0);      // small terms first
          wgmma_ss(acc, dah, bl, 1);
          wgmma_ss(acc, dah, bh, 1);
        }
      }
      wgmma_commit();
      // wait for this K-block's MMAs before the next one: in the RS form the next split writes the registers these
      // MMAs still read (keeping one group in flight would need a second fragment set and 32 more registers per
      // thread at BN = 128); the TMA ring and the other warpgroup cover the wait
      wgmma_wait_all();
      acc_fence(acc);
      // the stage is free once this warp's MMAs have read it
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty(stage));
      if (++stage == S) { stage = 0; phase ^= 1; }
    }

    // ================= epilogue =================
    int nt, rem_y, rem_x;
    const size_t tbase = tile_base(tile, nt, rem_y, rem_x);
    bool valid[NPASS];
#pragma unroll
    for (int i = 0; i < NPASS; ++i) valid[i] = row_y[i] < rem_y && row_x[i] < rem_x;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int col0 = nt * BN + ch * 32;         // GEMM column of this chunk
      const size_t cbase = tbase + (size_t)col_off(col0 + lq * 4);
      float4 rm_old[NPASS], rm_y[NPASS];
      if (rmw) {                                  // read-modify-write operands first: their latency overlaps the staging
#pragma unroll
        for (int i = 0; i < NPASS; ++i) {
          const size_t ob = cbase + (size_t)row_off[i];
          rm_old[i] = (p.beta != 0.f && valid[i]) ? *reinterpret_cast<const float4*>(p.out + ob) : make_float4(0.f, 0.f, 0.f, 0.f);
          rm_y[i] = (p.mask_y != nullptr && valid[i]) ? ld4(p.mask_y + ob) : make_float4(1.f, 1.f, 1.f, 1.f);
        }
      }
#pragma unroll
      for (int jj = 0; jj < CW / 8; ++jj) {
        const int j = ch * 4 + jj;                // 8-column group of the accumulator
        int cb = col0 + jj * 8 + 2 * t;
        if (p.d2s) cb -= (int)fdiv((uint32_t)cb, p.div_ct) * p.cout_true;
        float b0 = 0.f, b1 = 0.f;
        if (p.bias != nullptr) { b0 = __ldg(p.bias + cb); b1 = __ldg(p.bias + cb + 1); }
        float o[4] = {acc[4 * j] + b0, acc[4 * j + 1] + b1, acc[4 * j + 2] + b0, acc[4 * j + 3] + b1};
        if (act == NLT_ACT_ELU) {                 // warp-uniform
#pragma unroll
          for (int e = 0; e < 4; ++e) o[e] = elu_slow(o[e]);
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) o[e] = o[e] > 0.f ? o[e] : neg * o[e];
        }
        *reinterpret_cast<float2*>(stg + g * TC_EPI_PAD + jj * 8 + 2 * t) = make_float2(o[0], o[1]);
        *reinterpret_cast<float2*>(stg + (g + 8) * TC_EPI_PAD + jj * 8 + 2 * t) = make_float2(o[2], o[3]);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < NPASS; ++i) {
        const int row = i * RPI + lr;
        float4 o = *reinterpret_cast<const float4*>(stg + row * TC_EPI_PAD + lq * 4);
        if (rmw) {
          o.x += p.beta * rm_old[i].x; o.y += p.beta * rm_old[i].y; o.z += p.beta * rm_old[i].z; o.w += p.beta * rm_old[i].w;
          if (p.mask_y != nullptr) {
            o.x *= act_bwd_from_y(rm_y[i].x, p.mask_act); o.y *= act_bwd_from_y(rm_y[i].y, p.mask_act);
            o.z *= act_bwd_from_y(rm_y[i].z, p.mask_act); o.w *= act_bwd_from_y(rm_y[i].w, p.mask_act);
          }
        }
        if (valid[i]) *reinterpret_cast<float4*>(p.out + cbase + (size_t)row_off[i]) = o;
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)sym;
  }
  return fn;
}

struct TcPlan {
  bool ok;
  bool ts;      // RS form of the A operand (option tcs)
  int bn;
  int kbw;
  TcParams p;
  int chunks_per_tap;
  int cout_pad;
  size_t pack_floats;   // per plane
  size_t smem_bytes;
};

static int pick_bn(int cout) {
  if (cout % 128 == 0) return 128;
  if (cout % 64 == 0) return 64;
  if (cout % 32 == 0) return 32;
  if (cout % 16 == 0) return 16;
  return 0;
}

// Which single-phase GConvK shapes the tensor path takes (everything else stays on the SIMT kernels).
static TcPlan tc_plan(const GConvK& k, bool partial_tiles) {
  TcPlan pl;
  memset(&pl, 0, sizeof(pl));
  pl.ok = false;
  // option "tcs": 1 = RS form (A operand split in registers), 0 = SS form (hi / lo planes in shared memory)
  const bool ts = opt(Opt::TCS) == 1;
  // option "tc" = 2 (A/B testing): every shape the kernel can run takes it, ignoring the size heuristics below
  const bool force = opt(Opt::TC) == 2;
  pl.ts = ts;
  if (k.cout_true % 4 != 0) return pl;
  pl.bn = pick_bn(k.Cout);
  if (pl.bn == 0) return pl;
  int ctot = 0;
  pl.kbw = 32;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    if (sg.C % 16 != 0 || sg.sub != nullptr || sg.bcast || !aligned16(sg.ptr)) return pl;
    if (sg.C % 32 != 0) pl.kbw = 16;
    ctot += sg.C;
  }
  const int TC_KB = pl.kbw;
  if (!aligned16(k.w)) { /* weights are only read by the pack kernel: no alignment needed */ }
  if (!force) {
    // with less than 64 contraction terms the op is a pure stream: the pointwise / fp32 kernels are faster there
    if (k.ay.nu * k.ax.nu * ctot < 64) return pl;
    // 16-channel (64-byte-row) K-blocks only from K = 128 up: below that the FFMA stream kernels take these layers
    if (pl.kbw == 16 && k.ay.nu * k.ax.nu * ctot < 128) return pl;
  }
  if (k.ay.nu < 1 || k.ax.nu < 1) return pl;
  TcParams& p = pl.p;
  p.N = k.N; p.Hl = k.ay.nt; p.Wl = k.ax.nt;
  // tile shape
  // tile shape: TW = 128 lattice columns, or the smallest power of two >= Wl; partial tiles at the right / bottom
  // edge load zeros (TMA out-of-bounds fill) or rows that only feed masked outputs, and store nothing outside.
  // Only option tc = 2 and callers that ask for partial tiles take lattices that are not a multiple of the tile shape:
  // at the 1x1 .. 4x4 bottleneck levels most rows of a tile would be masked, and the fp32 kernels serve those layers
  if (p.Hl < 1 || p.Wl < 1) return pl;
  p.TW = TC_BM;
  while (p.TW / 2 >= p.Wl) p.TW /= 2;
  p.TH = TC_BM / p.TW;
  if (!force && !partial_tiles && (p.Wl % p.TW != 0 || p.Hl % p.TH != 0)) return pl;
  p.tiles_x = (p.Wl + p.TW - 1) / p.TW; p.tiles_y = (p.Hl + p.TH - 1) / p.TH;
  // coordinate map
  const bool stride1 = (k.ay.it == 1 && k.ax.it == 1);
  const bool patch = (!k.d2s && k.ay.it > 1 && k.ay.it == k.ax.it && k.ay.iu == 1 && k.ax.iu == 1 && k.ay.i0 == 0 &&
                      k.ax.i0 == 0 && k.ay.nu == k.ay.it && k.ax.nu == k.ax.it && k.Hin == k.ay.nt * k.ay.it &&
                      k.Win == k.ax.nt * k.ax.it);
  if (!stride1 && !patch) return pl;
  p.mode_patch = patch ? 1 : 0;
  p.ux_step = k.ax.iu; p.x_off = k.ax.i0; p.uy_step = k.ay.iu; p.y_off = k.ay.i0;
  p.Hs = patch ? k.Hin / k.ay.it : 0;
  if (patch && (k.ay.it > 256 || p.TW > 256)) return pl;
  p.ntap_y = k.ay.nu; p.ntap_x = k.ax.nu;
  p.nseg = k.nseg;
  pl.chunks_per_tap = 0;
  for (int s = 0; s < k.nseg; ++s) { p.seg_chunks[s] = k.seg[s].C / TC_KB; pl.chunks_per_tap += p.seg_chunks[s]; }
  p.kb_total = p.ntap_y * p.ntap_x * pl.chunks_per_tap;
  p.Hout = k.Hout; p.Wout = k.Wout; p.cout_true = k.cout_true; p.Cout = k.Cout;
  p.o0y = k.ay.o0; p.osy = k.ay.os; p.o0x = k.ax.o0; p.osx = k.ax.os;
  p.d2s = k.d2s; p.d2s_s = k.d2s_s;
  // few output tiles: narrower column tiles so that more SMs get work (A is re-read from L2), but only while the finer
  // tiling still fits ONE wave of persistent CTAs: every tile pays the pipeline fill / drain of the kernel again
  // (option "tc_split_waves" = 1: split whenever there are fewer tiles than SMs)
  const bool split_waves = opt(Opt::TC_SPLIT_WAVES) == 1;
  while (pl.bn > 32) {
    const long long tiles = (long long)p.N * p.tiles_x * p.tiles_y * (k.Cout / pl.bn);
    if (split_waves ? tiles >= sm_count() : 2 * tiles > sm_count()) break;
    pl.bn /= 2;
  }
  p.n_tiles_n = k.Cout / pl.bn;
  p.div_ntn = make_fastdiv((uint32_t)p.n_tiles_n); p.div_tpi = make_fastdiv((uint32_t)(p.tiles_x * p.tiles_y));
  p.div_tx = make_fastdiv((uint32_t)p.tiles_x); p.div_tw = make_fastdiv((uint32_t)p.TW);
  p.div_ct = make_fastdiv((uint32_t)p.cout_true); p.div_s = make_fastdiv((uint32_t)(p.d2s ? p.d2s_s : 1));
  const long long tt = (long long)p.N * p.tiles_x * p.tiles_y * p.n_tiles_n;
  if (tt > (1ll << 30)) return pl;
  p.total_tiles = (int)tt;
  pl.cout_pad = k.Cout;
  pl.pack_floats = (size_t)p.kb_total * pl.cout_pad * TC_KB;
  {
    const size_t stage_bytes = (ts ? 1 : 2) * (size_t)TC_BM * TC_KB * 4 + 2 * (size_t)pl.bn * TC_KB * 4;
    int st = (int)((227 * 1024 - TC_EPI_BYTES - 2048) / stage_bytes);
    if (st > TC_MAX_STAGES) st = TC_MAX_STAGES;
    if (st < 2) return pl;
    p.stages = st;
    pl.smem_bytes = (size_t)st * stage_bytes + TC_EPI_BYTES + 1024;
  }
  if (get_encode() == nullptr) return pl;
  p.rawhi = opt(Opt::TC_RAWHI);
  pl.ok = true;
  return pl;
}

static int encode_maps(const GConvK& k, const TcPlan& pl, const float* bhi, const float* blo, TcMaps* maps) {
  EncodeTiledFn enc = get_encode();
  const TcParams& p = pl.p;
  const int TC_KB = pl.kbw;
  const CUtensorMapSwizzle swz = pl.kbw == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    const cuuint64_t C = sg.C, W = k.Win, H = k.Hin, N = k.N;
    CUresult r;
    if (p.mode_patch) {
      const cuuint64_t st = k.ay.it;
      cuuint64_t dims[5] = {C, st, W / st, st, N * (H / st)};
      cuuint64_t strides[4] = {C * 4, st * C * 4, W * C * 4, st * W * C * 4};
      cuuint32_t box[5] = {(cuuint32_t)TC_KB, 1, (cuuint32_t)p.TW, 1, (cuuint32_t)p.TH};
      cuuint32_t es[5] = {1, 1, 1, 1, 1};
      r = enc(&maps->a[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)sg.ptr, dims, strides, box, es,
              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      cuuint64_t dims[4] = {C, W, H, N};
      cuuint64_t strides[3] = {C * 4, W * C * 4, H * W * C * 4};
      cuuint32_t box[4] = {(cuuint32_t)TC_KB, (cuuint32_t)p.TW, (cuuint32_t)p.TH, 1};
      cuuint32_t es[4] = {1, 1, 1, 1};
      r = enc(&maps->a[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)sg.ptr, dims, strides, box, es,
              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) return set_err(NLT_ERR_CUDA, "cuTensorMapEncodeTiled(A seg %d) failed: %d", s, (int)r);
  }
  const float* planes[2] = {bhi, blo};
  CUtensorMap* bm[2] = {&maps->bhi, &maps->blo};
  for (int i = 0; i < 2; ++i) {
    cuuint64_t dims[3] = {(cuuint64_t)TC_KB, (cuuint64_t)pl.cout_pad, (cuuint64_t)p.kb_total};
    cuuint64_t strides[2] = {(cuuint64_t)TC_KB * 4, (cuuint64_t)TC_KB * 4 * pl.cout_pad};
    cuuint32_t box[3] = {(cuuint32_t)TC_KB, (cuuint32_t)pl.bn, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = enc(bm[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)planes[i], dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_err(NLT_ERR_CUDA, "cuTensorMapEncodeTiled(B) failed: %d", (int)r);
  }
  return NLT_OK;
}

// =============================================================================================
// wgmma weight gradient:  dW[Kd x N] = sum_p A[p, Kd]^T * G[p, N]   (3xTF32, fp32 accumulate in registers)
//
// The contraction runs over PIXELS.  TF32 wgmma operands must be K-major, so the two consumer warpgroups
// TRANSPOSE while they split: TMA brings raw [32 pixels x w channels] pieces (w <= 32, hardware-swizzled so the
// transposing reads are bank-conflict free), the consumers write hi/lo planes [channel row][32 pixels = 128 B] in
// the K-major SWIZZLE_128B layout, and each warpgroup issues 4 K-steps x 3 products per 32-pixel stage into its
// [64 x BN] half of ONE [128 x BN] accumulator that lives in registers for the CTA's whole pixel range.  The
// planes are double-buffered: the split of stage i + 1 overlaps the MMAs of stage i.  Works for any channel
// counts that are multiples of 4.  The bias gradient (column sums of G) is accumulated on the way.  One fp32
// partial per CTA goes to the workspace; the fp32 path's fixed-order reduce kernel sums the partials
// (deterministic) and scatters them into the Keras weight layout.
// =============================================================================================
constexpr int WG_PT = 32;             // pixels per stage (= 128 B of fp32 per transposed row)
constexpr int WG_MAX_PIECES = 36;     // raw pieces per stage: <= 32 for A (128 rows / 4) + <= 2 for G (+ slack)
constexpr int WG_PLANE_A = TC_BM * 128;   // one transposed A plane: 128 rows x 128 B

struct WgPiece {
  int16_t is_g, seg, uy, ux;   // source
  int16_t c0, w;               // channel range inside the source
  int16_t row, pad;            // first transposed row (A: row of the M tile; G: row of the N tile)
  int32_t raw_off;             // byte offset of the raw tile inside a raw stage (1024-aligned)
};

struct WgParams {
  int N, Hl, Wl, TW, TH, tiles_x, tiles_y, total_ptiles;
  int mode_patch, ux_step, x_off, uy_step, y_off, Hs;     // A coordinate map (as TcParams)
  int g_patch, g_px, g_py, g_Hs;                          // G on a strided sub-lattice (transposed phases); g_patch == 2: depth-to-space
  int g_ct, g_s;                                          // depth-to-space: channels of the gradient tensor, stride
  int ntap_x, nseg, ctot, Kd;
  int seg_C[NLT_MAX_SEG], seg_coff[NLT_MAX_SEG];
  int n_mtiles, n_ntiles;
  FastDiv div_tpi, div_tx;                                // multiply-shift division by tiles per image / per row
  int raw_stages, raw_stage_bytes;
  int Cout, ld, KD_pad, bias_row;
  float* ws;
};

struct WgMaps {
  CUtensorMap a[NLT_MAX_SEG][4];   // per source, per piece width class: 4, 8, 16, 32 channels
  CUtensorMap g;                   // G pieces (width BN <= 32 -> BN, else 32)
};

__device__ __forceinline__ int wg_wclass(int w) { return w == 32 ? 3 : w == 16 ? 2 : w == 8 ? 1 : 0; }

// physical 16-byte chunk of logical chunk `cq` in pixel row `p` of a raw [32 x w] tile (TMA swizzle by row bytes)
__device__ __forceinline__ int wg_raw_chunk(int w, int p, int cq) {
  return w == 32 ? (cq ^ (p & 7)) : w == 16 ? (cq ^ ((p >> 1) & 3)) : w == 8 ? (cq ^ ((p >> 2) & 1)) : cq;
}

template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_wgrad_kernel(const __grid_constant__ WgMaps maps, const WgParams p) {
  constexpr int PLANE_G = BN * 128;
  constexpr int PLANES_BYTES = 2 * WG_PLANE_A + 2 * PLANE_G;      // Ahi, Alo, Ghi, Glo

  extern __shared__ uint8_t smem_raw[];
  // offset arithmetic on the __shared__ array keeps the address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t bars[2 * TC_MAX_STAGES];
  __shared__ WgPiece pieces[WG_MAX_PIECES];
  __shared__ uint16_t items[64];            // work items of the split: (piece << 8) | channel quad
  __shared__ int n_pieces_s, n_items_s, raw_bytes_s;
  __shared__ float bias_part[64];

  const int S = p.raw_stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar0 = smem_u32(bars);
  auto bar_rfull = [&](int s) { return bar0 + 8u * s; };
  auto bar_rempty = [&](int s) { return bar0 + 8u * (TC_MAX_STAGES + s); };
  uint8_t* planes = smem;                                         // 2 x PLANES_BYTES
  uint8_t* raw = smem + 2 * PLANES_BYTES;                         // S x raw_stage_bytes
  const uint32_t planes_u32 = smem_u32(planes), raw_u32 = smem_u32(raw);

  const int mtile = blockIdx.y, ntile = blockIdx.z;
  const int k_lo = mtile * TC_BM, k_hi = min(p.Kd, k_lo + TC_BM);

  if (threadIdx.x == 0) {
    // piece table of this (M tile, N tile): A pieces in flattened (tap, concat-channel) order, then G pieces
    int np = 0, off = 0, k = k_lo;
    while (k < k_hi) {
      const int tap = k / p.ctot, c = k - tap * p.ctot;
      int s = 0;
      while (s < p.nseg - 1 && c >= p.seg_coff[s] + p.seg_C[s]) ++s;
      const int cin = c - p.seg_coff[s];
      int w = p.seg_C[s] - cin;
      if (w > 32) w = 32;
      if (w > k_hi - k) w = k_hi - k;
      w = w >= 32 ? 32 : w >= 16 ? 16 : w >= 8 ? 8 : 4;         // power-of-two piece widths (all sizes are multiples of 4)
      WgPiece& pc = pieces[np++];
      pc.is_g = 0; pc.seg = (int16_t)s; pc.uy = (int16_t)(tap / p.ntap_x); pc.ux = (int16_t)(tap % p.ntap_x);
      pc.c0 = (int16_t)cin; pc.w = (int16_t)w; pc.row = (int16_t)(k - k_lo); pc.pad = 0; pc.raw_off = off;
      off += (WG_PT * w * 4 + 1023) & ~1023;
      k += w;
    }
    const int gw = p.g_patch == 2 ? min(min(BN, 32), p.g_ct) : (BN < 32 ? BN : 32);
    for (int c = 0; c < BN; c += gw) {
      WgPiece& pc = pieces[np++];
      pc.is_g = 1; pc.seg = 0; pc.uy = 0; pc.ux = 0; pc.c0 = (int16_t)(ntile * BN + c); pc.w = (int16_t)gw;
      if (p.g_patch == 2) {
        // depth-to-space weight gradient: GEMM column n' = tap * cout + n is channel n of the gradient pixel
        // (s*y + dy, s*x + dx) above lattice pixel (y, x)
        const int ncol = ntile * BN + c, tap = ncol / p.g_ct;
        pc.c0 = (int16_t)(ncol - tap * p.g_ct);
        pc.uy = (int16_t)(tap / p.g_s); pc.ux = (int16_t)(tap % p.g_s);
      }
      pc.row = (int16_t)c; pc.pad = 0; pc.raw_off = off;
      off += (WG_PT * gw * 4 + 1023) & ~1023;
    }
    n_pieces_s = np;
    int bytes = 0, ni = 0;
    for (int i = 0; i < np; ++i) {
      bytes += WG_PT * pieces[i].w * 4;
      for (int cq = 0; cq < pieces[i].w / 4; ++cq) items[ni++] = (uint16_t)((i << 8) | cq);
    }
    n_items_s = ni;
    raw_bytes_s = bytes;
    for (int s = 0; s < S; ++s) { mbar_init(bar_rfull(s), 1); mbar_init(bar_rempty(s), 8); }      // one arrival per consumer warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // transposed planes start as zero: rows beyond this tile's Kd / BN stay zero for the whole kernel
  for (int i = threadIdx.x; i < 2 * PLANES_BYTES / 16; i += TC_THREADS)
    reinterpret_cast<float4*>(planes)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int n_pieces = n_pieces_s;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  int my_tiles = 0;
  for (int t = blockIdx.x; t < p.total_ptiles; t += gridDim.x) ++my_tiles;

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  if (warp < 4) {
    // ================= TMA producer =================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < p.total_ptiles; t += gridDim.x) {
        const int n = (int)fdiv((uint32_t)t, p.div_tpi);
        const int r = t - n * tiles_per_img;
        const int rq = (int)fdiv((uint32_t)r, p.div_tx);
        const int ty0 = rq * p.TH, tx0 = (r - rq * p.tiles_x) * p.TW;
        mbar_wait(bar_rempty(stage), phase ^ 1);
        mbar_expect_tx(bar_rfull(stage), (uint32_t)raw_bytes_s);
        const uint32_t base = raw_u32 + (uint32_t)stage * p.raw_stage_bytes;
        for (int i = 0; i < n_pieces; ++i) {
          const WgPiece pc = pieces[i];
          if (pc.is_g) {
            if (p.g_patch == 2)
              tma_load_5d(base + pc.raw_off, &maps.g, bar_rfull(stage), pc.c0, pc.ux, tx0, pc.uy, n * p.g_Hs + ty0);
            else if (p.g_patch)
              tma_load_5d(base + pc.raw_off, &maps.g, bar_rfull(stage), pc.c0, p.g_px, tx0, p.g_py, n * p.g_Hs + ty0);
            else
              tma_load_4d(base + pc.raw_off, &maps.g, bar_rfull(stage), pc.c0, tx0, ty0, n);
          } else {
            const CUtensorMap* m = &maps.a[pc.seg][wg_wclass(pc.w)];
            if (p.mode_patch)
              tma_load_5d(base + pc.raw_off, m, bar_rfull(stage), pc.c0, pc.ux, tx0, pc.uy, n * p.Hs + ty0);
            else
              tma_load_4d(base + pc.raw_off, m, bar_rfull(stage), pc.c0, tx0 + pc.ux * p.ux_step + p.x_off,
                          ty0 + pc.uy * p.uy_step + p.y_off, n);
          }
        }
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ================= transpose + split, then wgmma: both consumer warpgroups (warps 4..11) =================
    // every thread takes two independent items per stage (dependent LDS -> split -> STS chains need the parallelism)
    const int wg = (warp >> 2) - 1;
    const int t = threadIdx.x - 128;              // 0..255 ; pixel = t % 32, item lane = t / 32
    const int px = t & 31, ql = t >> 5;
    const int n_items = n_items_s;
    constexpr int MAXI = 6;                       // items per thread: 48 items / 8 lanes
    float gsum[MAXI][4];
#pragma unroll
    for (int i = 0; i < MAXI; ++i) { gsum[i][0] = gsum[i][1] = gsum[i][2] = gsum[i][3] = 0.f; }
    const int pxc = px >> 2, pxo = (px & 3) << 2;
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int b = it & 1;
      mbar_wait(bar_rfull(stage), phase);
      const uint8_t* rbase = raw + (size_t)stage * p.raw_stage_bytes;
      uint8_t* pl = planes + (size_t)b * PLANES_BYTES;
#pragma unroll
      for (int i = 0; i < MAXI; ++i) {
        const int j = ql + 8 * i;
        if (j >= n_items) break;
        const int itm = items[j];
        const WgPiece pc = pieces[itm >> 8];
        const int cq = itm & 0xff;
        uint8_t* hi = pl + (pc.is_g ? 2 * WG_PLANE_A : 0);
        const int lo_off = pc.is_g ? PLANE_G : WG_PLANE_A;
        const float4 v = *reinterpret_cast<const float4*>(rbase + pc.raw_off + (size_t)px * pc.w * 4 +
                                                          wg_raw_chunk(pc.w, px, cq) * 16);
        const float vv[4] = {v.x, v.y, v.z, v.w};
        if (pc.is_g) { gsum[i][0] += v.x; gsum[i][1] += v.y; gsum[i][2] += v.z; gsum[i][3] += v.w; }
        const int row0 = pc.row + cq * 4;           // multiple of 4: (row0 + e) & 7 == (row0 & 7) + e
        const int r7 = row0 & 7;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // K-major SWIZZLE_128B: 16-byte chunk index XOR (row % 8)
          const int o = (row0 + e) * 128 + (((pxc ^ (r7 + e)) << 4) | pxo);
          const float h = tf32_round(vv[e]);
          *reinterpret_cast<float*>(hi + o) = h;
          *reinterpret_cast<float*>(hi + lo_off + o) = tf32_round(vv[e] - h);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma reads
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_rempty(stage));                  // raw stage consumed
      // this warpgroup's MMAs of stage it - 1 are done; after the barrier, so are the other warpgroup's, and every
      // warp has written planes b (planes b ^ 1 may be overwritten from the next stage on)
      wgmma_wait_all();
      acc_fence(acc);
      named_bar_sync(1, 256);
      const uint32_t ahi = planes_u32 + (uint32_t)b * PLANES_BYTES + (uint32_t)wg * (64 * 128), alo = ahi + WG_PLANE_A;
      const uint32_t ghi = planes_u32 + (uint32_t)b * PLANES_BYTES + 2 * WG_PLANE_A, glo = ghi + PLANE_G;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < WG_PT / 8; ++ks) {
        const uint64_t dah = wgmma_desc<128>(ahi + ks * 32), dal = wgmma_desc<128>(alo + ks * 32);
        const uint64_t dgh = wgmma_desc<128>(ghi + ks * 32), dgl = wgmma_desc<128>(glo + ks * 32);
        wgmma_ss(acc, dal, dgh, 1);
        wgmma_ss(acc, dah, dgl, 1);
        wgmma_ss(acc, dah, dgh, 1);
      }
      wgmma_commit();
      if (++stage == S) { stage = 0; phase ^= 1; }
    }
    wgmma_wait_all();
    acc_fence(acc);
    // bias partial: reduce the 32 pixel lanes of each warp in a fixed butterfly order
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int j = ql + 8 * i;
      const bool isg = j < n_items && pieces[items[j < n_items ? j : 0] >> 8].is_g;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = gsum[i][e];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (isg && px == 0) {
          const int itm = items[j];
          bias_part[pieces[itm >> 8].row + (itm & 0xff) * 4 + e] = v;
        }
      }
    }
  }
  // ---- all partials are ready: accumulators (registers of the consumers) and bias sums ----
  __syncthreads();
  if (warp >= 4) {
    const int wg = (warp >> 2) - 1, wq = warp & 3, g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = k_lo + 64 * wg + 16 * wq + g + 8 * h;         // accumulator row
      if (k < k_hi) {
        float* dst = p.ws + ((size_t)blockIdx.x * p.KD_pad + k) * p.ld + ntile * BN + 2 * t4;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
    const int r = threadIdx.x - 128;
    if (mtile == 0 && r < BN)
      p.ws[((size_t)blockIdx.x * p.KD_pad + p.bias_row) * p.ld + ntile * BN + r] = my_tiles > 0 ? bias_part[r] : 0.f;
  }
}

struct WgPlan {
  bool ok;
  int bn;
  WgParams p;
  size_t smem_bytes;
  int nsplit;
};

static WgPlan wg_plan(const GConvK& k) {
  WgPlan pl;
  memset(&pl, 0, sizeof(pl));
  if (k.M == 0 || k.Cout % 16 != 0) return pl;
  if (k.d2s && (k.cout_true % 4 != 0 || (k.cout_true & (k.cout_true - 1)) != 0) && k.cout_true % 32 != 0) return pl;
  int ctot = 0;
  for (int s = 0; s < k.nseg; ++s) {
    const Seg& sg = k.seg[s];
    if (sg.C % 4 != 0 || sg.sub != nullptr || sg.bcast || !aligned16(sg.ptr)) return pl;
    ctot += sg.C;
  }
  if (k.ay.nu < 1 || k.ax.nu < 1) return pl;
  pl.bn = k.Cout % 64 == 0 ? 64 : k.Cout % 32 == 0 ? 32 : 16;
  WgParams& p = pl.p;
  p.N = k.N; p.Hl = k.ay.nt; p.Wl = k.ax.nt;
  if (p.Wl >= WG_PT) {
    if (p.Wl % WG_PT) return pl;
    p.TW = WG_PT; p.TH = 1;
  } else {
    if (WG_PT % p.Wl) return pl;
    p.TW = p.Wl; p.TH = WG_PT / p.Wl;
    if (p.Hl % p.TH) return pl;
  }
  p.tiles_x = p.Wl / p.TW; p.tiles_y = p.Hl / p.TH;
  p.div_tpi = make_fastdiv((uint32_t)(p.tiles_x * p.tiles_y)); p.div_tx = make_fastdiv((uint32_t)p.tiles_x);
  const long long tt = (long long)p.N * p.tiles_x * p.tiles_y;
  if (tt > (1ll << 30) || tt < 4) return pl;
  p.total_ptiles = (int)tt;
  const bool stride1 = (k.ay.it == 1 && k.ax.it == 1);
  const bool patch = (k.ay.it > 1 && k.ay.it == k.ax.it && k.ay.iu == 1 && k.ax.iu == 1 && k.ay.i0 == 0 && k.ax.i0 == 0 &&
                      k.ay.nu == k.ay.it && k.ax.nu == k.ax.it && k.Hin == k.ay.nt * k.ay.it && k.Win == k.ax.nt * k.ax.it);
  if (!stride1 && !patch) return pl;
  p.mode_patch = patch ? 1 : 0;
  p.ux_step = k.ax.iu; p.x_off = k.ax.i0; p.uy_step = k.ay.iu; p.y_off = k.ay.i0;
  p.Hs = patch ? k.Hin / k.ay.it : 0;
  if (k.ay.os != k.ax.os) return pl;
  if (k.d2s) {
    // ONE pass over the input lattice for all s*s taps (instead of s*s phases that each re-read the input):
    // the gradient pieces of a stage come from the s*s pixels above each lattice pixel
    if (k.Hout != p.Hl * k.d2s_s || k.Wout != p.Wl * k.d2s_s) return pl;
    p.g_patch = 2; p.g_py = 0; p.g_px = 0; p.g_Hs = k.Hout / k.d2s_s; p.g_ct = k.cout_true; p.g_s = k.d2s_s;
  } else if (k.ay.os == 1) {
    if (k.ay.o0 != 0 || k.ax.o0 != 0 || k.Hout != p.Hl || k.Wout != p.Wl) return pl;
    p.g_patch = 0;
  } else {
    const int os = k.ay.os;
    if (k.Hout != p.Hl * os || k.Wout != p.Wl * os) return pl;
    p.g_patch = 1; p.g_py = k.ay.o0; p.g_px = k.ax.o0; p.g_Hs = k.Hout / os;
  }
  p.ntap_x = k.ax.nu; p.nseg = k.nseg; p.ctot = ctot;
  p.Kd = k.ay.nu * k.ax.nu * ctot;
  if (p.Kd < 128) return pl;      // below one full M tile the warp-stream fp32 kernel takes the shape
  int coff = 0;
  for (int s = 0; s < k.nseg; ++s) { p.seg_C[s] = k.seg[s].C; p.seg_coff[s] = coff; coff += k.seg[s].C; }
  p.n_mtiles = (p.Kd + TC_BM - 1) / TC_BM;
  p.n_ntiles = k.Cout / pl.bn;
  p.Cout = k.Cout; p.ld = k.Cout;
  p.bias_row = p.Kd; p.KD_pad = p.Kd + 4;
  // raw stage: worst case 32 A pieces of 4 channels (1 KB each after rounding) or 4 of 32 (4 KB each): <= 32 KB; G <= 8 KB
  p.raw_stage_bytes = 32 * 1024 + 8 * 1024;
  {
    // tighter bound: pieces never exceed max(16 KB of payload, #pieces KB); recompute exactly for M tile 0 (the fullest)
    int bytes = 0, kk = 0;
    const int k_hi = p.Kd < TC_BM ? p.Kd : TC_BM;
    int worst = 0;
    for (int mt = 0; mt < p.n_mtiles; ++mt) {
      bytes = 0; kk = mt * TC_BM;
      const int hi = (kk + TC_BM < p.Kd) ? kk + TC_BM : p.Kd;
      while (kk < hi) {
        const int tap = kk / ctot, c = kk - tap * ctot;
        int s = 0;
        while (s < k.nseg - 1 && c >= p.seg_coff[s] + p.seg_C[s]) ++s;
        int w = p.seg_C[s] - (c - p.seg_coff[s]);
        if (w > 32) w = 32;
        if (w > hi - kk) w = hi - kk;
        w = w >= 32 ? 32 : w >= 16 ? 16 : w >= 8 ? 8 : 4;
        bytes += (WG_PT * w * 4 + 1023) & ~1023;
        kk += w;
      }
      if (bytes > worst) worst = bytes;
    }
    (void)k_hi;
    int gw = pl.bn < 32 ? pl.bn : 32;
    if (k.d2s && k.cout_true < gw) gw = k.cout_true;
    worst += (pl.bn / gw) * ((WG_PT * gw * 4 + 1023) & ~1023);
    p.raw_stage_bytes = worst;
  }
  const size_t planes = 2 * (2 * (size_t)WG_PLANE_A + 2 * (size_t)pl.bn * 128);
  int st = (int)((227 * 1024 - 2048 - (long long)planes - 4096) / p.raw_stage_bytes);
  if (st > TC_MAX_STAGES) st = TC_MAX_STAGES;
  if (st < 2) return pl;
  p.raw_stages = st;
  pl.smem_bytes = planes + (size_t)st * p.raw_stage_bytes + 1024;
  long long want = sm_count() / ((long long)p.n_mtiles * p.n_ntiles);
  if (want < 1) want = 1;
  if (want > tt / 4) want = tt / 4;
  if (want < 1) want = 1;
  pl.nsplit = (int)want;
  if (get_encode() == nullptr) return pl;
  pl.ok = true;
  return pl;
}

bool tc_wgrad_applicable(const GConvK& k) { return wg_plan(k).ok; }

size_t tc_wgrad_ws_floats(const GConvK& k) {
  WgPlan pl = wg_plan(k);
  return pl.ok ? (size_t)pl.nsplit * pl.p.KD_pad * pl.p.ld : 0;
}

template <int BN>
static int wg_launch(const WgMaps& maps, const WgPlan& pl, cudaStream_t st) {
  static bool attr_set[64] = {false};     // per device: the attribute is not process-wide
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(tc_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 4096);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  dim3 grid(pl.nsplit, pl.p.n_mtiles, pl.p.n_ntiles);
  tc_wgrad_kernel<BN><<<grid, TC_THREADS, pl.smem_bytes, st>>>(maps, pl.p);
  NLT_CUDA_LAUNCH_CHECK("tc_wgrad_kernel");
  __atomic_add_fetch(&g_tc_launches, 1ull, __ATOMIC_RELAXED);
  return NLT_OK;
}

// raw [pixels x w channels] tile of an NHWC tensor, swizzled by its row bytes (bank-conflict-free transposing reads)
static CUresult wg_encode(EncodeTiledFn enc, CUtensorMap* m, const float* ptr, int C, int W, int H, int N, int w, int TW,
                          int TH, int patch_s) {
  const CUtensorMapSwizzle swz = w == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : w == 16 ? CU_TENSOR_MAP_SWIZZLE_64B
                                 : w == 8 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  const cuuint64_t c = C, ww = W, h = H, n = N;
  if (patch_s > 1) {
    const cuuint64_t st_ = patch_s;
    cuuint64_t dims[5] = {c, st_, ww / st_, st_, n * (h / st_)};
    cuuint64_t strides[4] = {c * 4, st_ * c * 4, ww * c * 4, st_ * ww * c * 4};
    cuuint32_t box[5] = {(cuuint32_t)w, 1, (cuuint32_t)TW, 1, (cuuint32_t)TH};
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)ptr, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
               swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  cuuint64_t dims[4] = {c, ww, h, n};
  cuuint64_t strides[3] = {c * 4, ww * c * 4, h * ww * c * 4};
  cuuint32_t box[4] = {(cuuint32_t)w, (cuuint32_t)TW, (cuuint32_t)TH, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)ptr, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

int launch_tc_wgrad(const GConvK& k, const float* G, float* ws, WgradK* w, size_t* KD_pad, cudaStream_t st) {
  WgPlan pl = wg_plan(k);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "tensor-core wgrad not applicable");
  NLT_CHECK_ARG(aligned16(G), "dz must be 16-byte aligned");
  EncodeTiledFn enc = get_encode();
  WgMaps maps;
  memset(&maps, 0, sizeof(maps));
  const WgParams& p = pl.p;
  static const int widths[4] = {4, 8, 16, 32};
  for (int s = 0; s < k.nseg; ++s)
    for (int wi = 0; wi < 4; ++wi) {
      if (widths[wi] > k.seg[s].C) continue;
      CUresult r = wg_encode(enc, &maps.a[s][wi], k.seg[s].ptr, k.seg[s].C, k.Win, k.Hin, k.N, widths[wi], p.TW, p.TH,
                             p.mode_patch ? k.ay.it : 1);
      if (r != CUDA_SUCCESS) return set_err(NLT_ERR_CUDA, "cuTensorMapEncodeTiled(wgrad A %d/%d) failed: %d", s, widths[wi], (int)r);
    }
  {
    int gw = pl.bn < 32 ? pl.bn : 32;
    if (k.d2s && k.cout_true < gw) gw = k.cout_true;
    CUresult r = k.d2s ? wg_encode(enc, &maps.g, G, k.cout_true, k.Wout, k.Hout, k.N, gw, p.TW, p.TH, k.d2s_s)
                       : wg_encode(enc, &maps.g, G, k.Cout, k.Wout, k.Hout, k.N, gw, p.TW, p.TH, p.g_patch ? k.ay.os : 1);
    if (r != CUDA_SUCCESS) return set_err(NLT_ERR_CUDA, "cuTensorMapEncodeTiled(wgrad G) failed: %d", (int)r);
  }
  pl.p.ws = ws;
  w->g = k;
  w->GS = p.ctot / 4;
  w->KG = k.ay.nu * k.ax.nu * w->GS + 1;
  w->ld = p.ld; w->nsplit = pl.nsplit; w->pix_per_split = 0;
  *KD_pad = (size_t)p.KD_pad;
  switch (pl.bn) {
    case 64: return wg_launch<64>(maps, pl, st);
    case 32: return wg_launch<32>(maps, pl, st);
    default: return wg_launch<16>(maps, pl, st);
  }
}

bool tc_applicable(const GConvK& k, bool partial_tiles) { return tc_plan(k, partial_tiles).ok; }

size_t tc_workspace_bytes(const GConvK& k, bool partial_tiles) {
  TcPlan pl = tc_plan(k, partial_tiles);
  return pl.ok ? 2 * pl.pack_floats * sizeof(float) + 256 : 0;
}

template <int BN, int KBW>
static int tc_launch_bn(const TcMaps& maps, const TcPlan& pl, cudaStream_t st) {
  // the opt-in to > 48 KB of dynamic shared memory is a per-device attribute
  static bool attr_set[2][64] = {{false}};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[pl.ts ? 1 : 0][dev]) {
    cudaError_t e = pl.ts ? cudaFuncSetAttribute(tc_gconv_kernel<BN, KBW, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 227 * 1024 - 1024)
                          : cudaFuncSetAttribute(tc_gconv_kernel<BN, KBW, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 227 * 1024 - 1024);
    if (e != cudaSuccess) return set_err(NLT_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    if (dev >= 0 && dev < 64) attr_set[pl.ts ? 1 : 0][dev] = true;
  }
  const int grid = pl.p.total_tiles < sm_count() ? pl.p.total_tiles : sm_count();
  if (pl.ts) tc_gconv_kernel<BN, KBW, true><<<grid, TC_THREADS, pl.smem_bytes, st>>>(maps, pl.p);
  else tc_gconv_kernel<BN, KBW, false><<<grid, TC_THREADS, pl.smem_bytes, st>>>(maps, pl.p);
  NLT_CUDA_LAUNCH_CHECK("tc_gconv_kernel");
  __atomic_add_fetch(&g_tc_launches, 1ull, __ATOMIC_RELAXED);
  return NLT_OK;
}

// hi / lo planes of the weights in K-block layout (what the B tensor maps of the conv kernel read)
int tc_pack(const GConvK& k, void* workspace, size_t workspace_bytes, cudaStream_t st, bool partial_tiles) {
  TcPlan pl = tc_plan(k, partial_tiles);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "tensor-core path not applicable");
  const size_t need = 2 * pl.pack_floats * sizeof(float) + 256;
  NLT_CHECK_ARG(workspace != nullptr && workspace_bytes >= need, "tc workspace too small: need %zu", need);
  float* bhi = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  float* blo = bhi + pl.pack_floats;
  const size_t total = pl.pack_floats;
  int blocks = (int)((total + 255) / 256);
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  tc_pack_weights_kernel<<<blocks, 256, 0, st>>>(k, pl.kbw, pl.p.kb_total, pl.chunks_per_tap, pl.cout_pad, bhi, blo);
  NLT_CUDA_LAUNCH_CHECK("tc_pack_weights_kernel");
  return NLT_OK;
}

int launch_tc(const GConvK& k, const float* bias, int act, float beta, const float* mask_y, int mask_act, float* out,
              void* workspace, size_t workspace_bytes, cudaStream_t st, bool prepacked, bool partial_tiles) {
  TcPlan pl = tc_plan(k, partial_tiles);
  if (!pl.ok) return set_err(NLT_ERR_INVALID, "tensor-core path not applicable");
  const size_t need = 2 * pl.pack_floats * sizeof(float) + 256;
  NLT_CHECK_ARG(workspace != nullptr && workspace_bytes >= need, "tc workspace too small: need %zu", need);
  float* bhi = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  float* blo = bhi + pl.pack_floats;
  if (!prepacked) {
    const int rc0 = tc_pack(k, workspace, workspace_bytes, st, partial_tiles);
    if (rc0 != NLT_OK) return rc0;
  }
  TcMaps maps;
  int rc = encode_maps(k, pl, bhi, blo, &maps);
  if (rc != NLT_OK) return rc;
  pl.p.act = act; pl.p.mask_act = mask_act; pl.p.beta = beta; pl.p.bias = bias; pl.p.mask_y = mask_y; pl.p.out = out;
  if (pl.kbw == 32) {
    switch (pl.bn) {
      case 128: return tc_launch_bn<128, 32>(maps, pl, st);
      case 64: return tc_launch_bn<64, 32>(maps, pl, st);
      case 32: return tc_launch_bn<32, 32>(maps, pl, st);
      default: return tc_launch_bn<16, 32>(maps, pl, st);
    }
  }
  switch (pl.bn) {
    case 128: return tc_launch_bn<128, 16>(maps, pl, st);
    case 64: return tc_launch_bn<64, 16>(maps, pl, st);
    case 32: return tc_launch_bn<32, 16>(maps, pl, st);
    default: return tc_launch_bn<16, 16>(maps, pl, st);
  }
}

}  // namespace nlt
