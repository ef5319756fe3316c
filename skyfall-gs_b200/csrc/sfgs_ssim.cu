// sfgs_ssim.cu — fused SSIM (value map + the three partial-derivative maps, and the gradient w.r.t. img1).
//
// Replaces fusedssim / fusedssim_backward of the reference's fused-ssim submodule (SSIM/ssim.h:7-26; what they
// compute: 11-tap sigma = 1.5 separable Gaussian window with "same" zero padding, C1/C2 passed by the caller,
// only img1 differentiable).  The kernels are new, designed around what Hopper offers for a tile-movement problem of
// this shape:
//
//   * the zero-padded (tile + 5-pixel halo) boxes of the input planes are fetched by TMA
//     (cp.async.bulk.tensor.3d, one elected thread, completion on an mbarrier): the tensor map's out-of-bounds
//     fill IS the "same" zero padding, so there is no per-pixel bounds test and no address arithmetic on the load
//     side at all;
//   * the five windowed moments E[x], E[y], E[x^2], E[y^2], E[xy] are carried as two pairs + one scalar:
//     (x, y) and (x^2, y^2) share their filter weight, which is loaded once per tap for both lanes of a pair; the
//     pair arithmetic is written with the round-to-nearest intrinsics, so no multiply is contracted into an add and
//     every lane is rounded exactly like a separate multiply / add / fused multiply-add;
//   * 64x32-pixel tiles (1.5x halo read amplification against L2; 2.6x for the reference's 16x16 tiles), the
//     horizontal pass register-blocked four outputs per thread from 128-bit shared-memory loads, the vertical pass
//     streaming down 2 columns x 4 rows per thread with the partial sums in registers;
//   * every global access is 64 or 128 bits wide.
//
// Images whose rows are not 16-byte multiples (W % 4 != 0) or whose base is unaligned cannot be described by a
// tensor map; they take the same kernels with a cooperative bounds-checked tile load instead of TMA.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <mutex>
#include "sfgs_common.cuh"

namespace {

constexpr int TW = 64, TH = 32, HALO = 5;
// The TMA box starts on a 16-byte boundary of the row (x0 - 8 rather than x0 - 5), so it is fetched from x0 - HX with
// HX = 8 and is 64 + 2*8 = 80 floats wide: output column c
// reads box columns c + 3 .. c + 13.  Rows have no such constraint (the box starts at y0 - 5).
constexpr int HX = 8;
constexpr int BOX_W = TW + 2 * HX;        // 80 floats = 320 bytes per row
constexpr int BOX_H = TH + 2 * HALO;      // 42
constexpr int BOX_FLOATS = BOX_W * BOX_H; // 3360 floats = 13440 bytes = 105 x 128: consecutive boxes stay 128-byte aligned
constexpr int BOX_STRIDE = BOX_FLOATS;
constexpr int SSIM_THREADS = 256;

// sigma = 1.5, 11 taps, normalised (the window of SSIM/ssim.cu:12-24 and of utils/loss_utils.py:gaussian)
__constant__ float c_w[11] = {0.001028380123898387f, 0.0075987582094967365f, 0.036000773310661316f,
                              0.10936068743467331f,  0.21300552785396576f,   0.26601171493530273f,
                              0.21300552785396576f,  0.10936068743467331f,   0.036000773310661316f,
                              0.0075987582094967365f, 0.001028380123898387f};

using u64 = unsigned long long;
using f2 = float2;
__device__ __forceinline__ f2 pk(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk(f2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

__device__ __forceinline__ void mbar_init(u64* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, unsigned parity) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  } while (!ok);
}
// one box {BOX_W, BOX_H, 1} of a [planes, H, W] float tensor, corner (x, y, plane); out-of-range elements arrive as 0
__device__ __forceinline__ void tma_load_box(float* dst, const CUtensorMap* tm, int x, int y, int plane, u64* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(tm), "r"(x), "r"(y), "r"(plane),
                 "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}

// cooperative fallback for images a tensor map cannot describe: same box, zero padding by bounds test
__device__ __forceinline__ void load_box_generic(float* dst, const float* __restrict__ plane, int x0, int y0, int W, int H) {
  for (int i = threadIdx.x; i < BOX_H * BOX_W; i += SSIM_THREADS) {
    const int r = i / BOX_W, c = i - r * BOX_W;
    const int gx = x0 + c, gy = y0 + r;
    dst[i] = (gx >= 0 && gx < W && gy >= 0 && gy < H) ? plane[(size_t)gy * W + gx] : 0.f;
  }
}

struct Maps4 { CUtensorMap m[4]; };

// ---------------------------------------------------------------------------------------------------- forward
struct FwdSmem {
  float box[2][2][BOX_STRIDE];       // [stage][img1, img2] tile + halo (TMA destination, dense rows of BOX_W floats)
  float2 h12[BOX_H][TW];             // horizontally filtered (x, y)
  float2 h34[BOX_H][TW];             // horizontally filtered (x^2, y^2)
  float h5[BOX_H][TW];               // horizontally filtered x*y
  u64 bar[2];
};

// Persistent CTAs: CTA b takes tiles b, b + grid, ...; the boxes of tile i+1 are requested from the TMA unit before
// tile i is touched (two box stages, one mbarrier each), so the fetch latency hides behind a whole tile of arithmetic.
struct TileIter {
  int tiles_x, tiles_y, ntiles;
  __device__ __forceinline__ void decode(int tile, int& x0, int& y0, int& plane) const {
    const int per_plane = tiles_x * tiles_y;
    plane = tile / per_plane;
    const int r = tile - plane * per_plane;
    const int ty = r / tiles_x;
    x0 = (r - ty * tiles_x) * TW; y0 = ty * TH;
  }
};

template <bool TRAIN, bool USE_TMA>
__global__ void __launch_bounds__(SSIM_THREADS, 2)
ssim_fwd_kernel(const __grid_constant__ Maps4 tm, int H, int W, int planes, float C1, float C2, const float* __restrict__ img1,
                const float* __restrict__ img2, float* __restrict__ ssim_map, float* __restrict__ dm_dmu1,
                float* __restrict__ dm_dsigma1_sq, float* __restrict__ dm_dsigma12) {
  extern __shared__ __align__(128) unsigned char ssim_smem[];
  FwdSmem& S = *reinterpret_cast<FwdSmem*>(ssim_smem);
  const int t = threadIdx.x;
  TileIter it;
  it.tiles_x = (W + TW - 1) / TW; it.tiles_y = (H + TH - 1) / TH; it.ntiles = it.tiles_x * it.tiles_y * planes;

  auto request = [&](int tile, int stage) {      // thread 0 only
    int bx, by, pl;
    it.decode(tile, bx, by, pl);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic-proxy reads of this stage are ordered before the async writes
    mbar_expect_tx(&S.bar[stage], 2u * BOX_FLOATS * sizeof(float));
    tma_load_box(S.box[stage][0], &tm.m[0], bx - HX, by - HALO, pl, &S.bar[stage]);
    tma_load_box(S.box[stage][1], &tm.m[1], bx - HX, by - HALO, pl, &S.bar[stage]);
  };
  if (USE_TMA) {
    if (t == 0) {
      mbar_init(&S.bar[0], 1); mbar_init(&S.bar[1], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      if ((int)blockIdx.x < it.ntiles) request(blockIdx.x, 0);
    }
    __syncthreads();            // the barrier words are initialised before anyone polls them
  }

  int iter = 0;
  for (int tile = blockIdx.x; tile < it.ntiles; tile += gridDim.x, iter++) {
  const int stage = iter & 1;
  int x0, y0, plane;
  it.decode(tile, x0, y0, plane);
  const size_t poff = (size_t)plane * H * W;
  if (USE_TMA) {
    // the other stage was last read by the previous tile's horizontal pass, which every thread left two barriers ago
    if (t == 0 && tile + (int)gridDim.x < it.ntiles) request(tile + gridDim.x, stage ^ 1);
    mbar_wait(&S.bar[stage], (unsigned)(iter >> 1) & 1u);
  } else {
    load_box_generic(S.box[stage][0], img1 + poff, x0 - HX, y0 - HALO, W, H);
    load_box_generic(S.box[stage][1], img2 + poff, x0 - HX, y0 - HALO, W, H);
    __syncthreads();
  }

  // ---- horizontal pass: unit = (box row, group of 4 output columns); 14 inputs per image from five 128-bit loads
  for (int u = t; u < BOX_H * (TW / 4); u += SSIM_THREADS) {
    const int row = u >> 4, xg = u & 15;
    const float4* px = reinterpret_cast<const float4*>(&S.box[stage][0][row * BOX_W + 4 * xg]);
    const float4* py = reinterpret_cast<const float4*>(&S.box[stage][1][row * BOX_W + 4 * xg]);
    float X[20], Y[20];                       // box columns 4xg .. 4xg+19; the four outputs use columns 4xg+3 .. 4xg+16
#pragma unroll
    for (int q = 0; q < 5; q++) {
      const float4 a = px[q], b = py[q];
      X[4 * q] = a.x; X[4 * q + 1] = a.y; X[4 * q + 2] = a.z; X[4 * q + 3] = a.w;
      Y[4 * q] = b.x; Y[4 * q + 1] = b.y; Y[4 * q + 2] = b.z; Y[4 * q + 3] = b.w;
    }
    f2 P1[14], P2[14];
    float PXY[14];
#pragma unroll
    for (int i = 0; i < 14; i++) {
      P1[i] = pk(X[i + HX - HALO], Y[i + HX - HALO]); P2[i] = mul2(P1[i], P1[i]); PXY[i] = X[i + HX - HALO] * Y[i + HX - HALO];
    }
    float2 o12[4], o34[4];
    float o5[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float wc = c_w[HALO];
      const f2 wc2 = pk(wc, wc);
      f2 a1 = mul2(P1[j + HALO], wc2), a2 = mul2(P2[j + HALO], wc2);
      float a5 = PXY[j + HALO] * wc;
#pragma unroll
      for (int d = 1; d <= HALO; d++) {
        const float w = c_w[HALO - d];
        const f2 w2 = pk(w, w);
        a1 = fma2(add2(P1[j + HALO - d], P1[j + HALO + d]), w2, a1);
        a2 = fma2(add2(P2[j + HALO - d], P2[j + HALO + d]), w2, a2);
        a5 = fmaf(PXY[j + HALO - d] + PXY[j + HALO + d], w, a5);
      }
      upk(a1, o12[j].x, o12[j].y);
      upk(a2, o34[j].x, o34[j].y);
      o5[j] = a5;
    }
    float4* d12 = reinterpret_cast<float4*>(&S.h12[row][4 * xg]);
    float4* d34 = reinterpret_cast<float4*>(&S.h34[row][4 * xg]);
    d12[0] = make_float4(o12[0].x, o12[0].y, o12[1].x, o12[1].y);
    d12[1] = make_float4(o12[2].x, o12[2].y, o12[3].x, o12[3].y);
    d34[0] = make_float4(o34[0].x, o34[0].y, o34[1].x, o34[1].y);
    d34[1] = make_float4(o34[2].x, o34[2].y, o34[3].x, o34[3].y);
    *reinterpret_cast<float4*>(&S.h5[row][4 * xg]) = make_float4(o5[0], o5[1], o5[2], o5[3]);
  }
  __syncthreads();

  // ---- vertical pass: 2 columns x 4 output rows per thread, streaming down the 14 rows it needs
  const int cg = t & 31, rg = t >> 5;         // column group (2 columns), row group (4 rows)
  const int lx = 2 * cg, ly = 4 * rg;
  f2 v1[4][2], v2[4][2];
  float v5[4][2];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int c = 0; c < 2; c++) { v1[r][c] = pk(0.f, 0.f); v2[r][c] = pk(0.f, 0.f); v5[r][c] = 0.f; }
#pragma unroll
  for (int i = 0; i < 14; i++) {              // box row ly + i feeds output row ly + r with weight c_w[i - r]
    const float4 a = *reinterpret_cast<const float4*>(&S.h12[ly + i][lx]);
    const float4 b = *reinterpret_cast<const float4*>(&S.h34[ly + i][lx]);
    const float2 c5 = *reinterpret_cast<const float2*>(&S.h5[ly + i][lx]);
    const f2 a0 = pk(a.x, a.y), a1 = pk(a.z, a.w), b0 = pk(b.x, b.y), b1 = pk(b.z, b.w);
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int k = i - r;
      if (k >= 0 && k <= 10) {
        const float w = c_w[k];
        const f2 w2 = pk(w, w);
        v1[r][0] = fma2(a0, w2, v1[r][0]); v1[r][1] = fma2(a1, w2, v1[r][1]);
        v2[r][0] = fma2(b0, w2, v2[r][0]); v2[r][1] = fma2(b1, w2, v2[r][1]);
        v5[r][0] = fmaf(c5.x, w, v5[r][0]); v5[r][1] = fmaf(c5.y, w, v5[r][1]);
      }
    }
  }

  // ---- SSIM and its partial derivatives (the formulas of the SSIM index; cf. utils/loss_utils.py:_ssim)
  const int gx = x0 + lx;
  const bool vec_ok = (W & 1) == 0;           // 8-byte stores need even rows (bases are checked on the host)
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int gy = y0 + ly + r;
    if (gy >= H || gx >= W) continue;
    float val[2], dmu[2], ds1[2], ds12[2];
#pragma unroll
    for (int c = 0; c < 2; c++) {
      float mu1, mu2, ex2, ey2;
      upk(v1[r][c], mu1, mu2);
      upk(v2[r][c], ex2, ey2);
      const float exy = v5[r][c];
      const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
      const float sigma1_sq = ex2 - mu1_sq, sigma2_sq = ey2 - mu2_sq, sigma12 = exy - mu12;
      const float A = mu1_sq + mu2_sq + C1, B = sigma1_sq + sigma2_sq + C2;
      const float Cn = 2.f * mu12 + C1, Dn = 2.f * sigma12 + C2;
      float iA, iB;       // A, B >= C1, C2 > 0: the approximate reciprocal (1 ulp) needs no special cases
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(iA) : "f"(A));
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(iB) : "f"(B));
      const float iAB = iA * iB;
      val[c] = Cn * Dn * iAB;
      if (TRAIN) {
        // d/dmu1 of (Cn Dn)/(A B) with sigma1_sq, sigma12 depending on mu1:  2 mu2 (Dn - Cn)/(AB) - 2 mu1 Cn Dn (1/A - 1/B)/(AB)
        dmu[c] = 2.f * iAB * (mu2 * (Dn - Cn) - mu1 * Cn * Dn * (iA - iB));
        ds1[c] = -Cn * Dn * iAB * iB;
        ds12[c] = 2.f * Cn * iAB;
      }
    }
    const size_t o = poff + (size_t)gy * W + gx;
    if (vec_ok && gx + 1 < W) {
      *reinterpret_cast<float2*>(ssim_map + o) = make_float2(val[0], val[1]);
      if (TRAIN) {
        *reinterpret_cast<float2*>(dm_dmu1 + o) = make_float2(dmu[0], dmu[1]);
        *reinterpret_cast<float2*>(dm_dsigma1_sq + o) = make_float2(ds1[0], ds1[1]);
        *reinterpret_cast<float2*>(dm_dsigma12 + o) = make_float2(ds12[0], ds12[1]);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 2; c++)
        if (gx + c < W) {
          ssim_map[o + c] = val[c];
          if (TRAIN) { dm_dmu1[o + c] = dmu[c]; dm_dsigma1_sq[o + c] = ds1[c]; dm_dsigma12[o + c] = ds12[c]; }
        }
    }
  }
  __syncthreads();      // the vertical pass is done with h12/h34/h5 before the next tile's horizontal pass rewrites them
  }   // tile loop
}

// ---------------------------------------------------------------------------------------------------- backward
// dL/dimg1 = G * (dmu1 dL) + 2 img1 . G * (dsigma1_sq dL) + img2 . G * (dsigma12 dL),  G = the 2-D window
// (mu1 = G*x, sigma1_sq = G*x^2 - mu1^2, sigma12 = G*xy - mu1 mu2; the mu1 terms are inside dm_dmu1).
struct BwdSmem {
  float box[1][4][BOX_STRIDE];       // [dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12] tiles + halo (one stage: see below)
  float2 h01[BOX_H][TW];             // horizontally filtered (dmu1 dL, dsigma1_sq dL)
  float h2[BOX_H][TW];               // horizontally filtered dsigma12 dL
  u64 bar[2];
};

// Four input planes leave no room for two box stages at two CTAs per SM, so the boxes are single-buffered and the next
// tile's fetch is issued as soon as the horizontal pass has consumed them: it overlaps the vertical pass and the stores.
template <bool USE_TMA>
__global__ void __launch_bounds__(SSIM_THREADS, 2)
ssim_bwd_kernel(const __grid_constant__ Maps4 tm, int H, int W, int planes, const float* __restrict__ img1,
                const float* __restrict__ img2, const float* __restrict__ dL_dmap, const float* __restrict__ dm_dmu1,
                const float* __restrict__ dm_dsigma1_sq, const float* __restrict__ dm_dsigma12,
                float* __restrict__ dL_dimg1) {
  extern __shared__ __align__(128) unsigned char ssim_smem[];
  BwdSmem& S = *reinterpret_cast<BwdSmem*>(ssim_smem);
  const int t = threadIdx.x;
  TileIter it;
  it.tiles_x = (W + TW - 1) / TW; it.tiles_y = (H + TH - 1) / TH; it.ntiles = it.tiles_x * it.tiles_y * planes;

  auto request = [&](int tile, int stage) {      // thread 0 only
    int bx, by, pl;
    it.decode(tile, bx, by, pl);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_expect_tx(&S.bar[stage], 4u * BOX_FLOATS * sizeof(float));
#pragma unroll
    for (int k = 0; k < 4; k++) tma_load_box(S.box[stage][k], &tm.m[k], bx - HX, by - HALO, pl, &S.bar[stage]);
  };
  if (USE_TMA) {
    if (t == 0) {
      mbar_init(&S.bar[0], 1); mbar_init(&S.bar[1], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      if ((int)blockIdx.x < it.ntiles) request(blockIdx.x, 0);
    }
    __syncthreads();
  }

  int iter = 0;
  for (int tile = blockIdx.x; tile < it.ntiles; tile += gridDim.x, iter++) {
  constexpr int stage = 0;
  int x0, y0, plane;
  it.decode(tile, x0, y0, plane);
  const size_t poff = (size_t)plane * H * W;
  if (USE_TMA) {
    mbar_wait(&S.bar[0], (unsigned)iter & 1u);
  } else {
    load_box_generic(S.box[stage][0], dL_dmap + poff, x0 - HX, y0 - HALO, W, H);
    load_box_generic(S.box[stage][1], dm_dmu1 + poff, x0 - HX, y0 - HALO, W, H);
    load_box_generic(S.box[stage][2], dm_dsigma1_sq + poff, x0 - HX, y0 - HALO, W, H);
    load_box_generic(S.box[stage][3], dm_dsigma12 + poff, x0 - HX, y0 - HALO, W, H);
    __syncthreads();
  }

  for (int u = t; u < BOX_H * (TW / 4); u += SSIM_THREADS) {
    const int row = u >> 4, xg = u & 15;
    f2 P[14];
    float Q[14];
#pragma unroll
    for (int q = 0; q < 5; q++) {             // box columns 4xg .. 4xg+19, of which 4xg+3 .. 4xg+16 are used
      const float4 g = *reinterpret_cast<const float4*>(&S.box[stage][0][row * BOX_W + 4 * xg + 4 * q]);
      const float4 a = *reinterpret_cast<const float4*>(&S.box[stage][1][row * BOX_W + 4 * xg + 4 * q]);
      const float4 b = *reinterpret_cast<const float4*>(&S.box[stage][2][row * BOX_W + 4 * xg + 4 * q]);
      const float4 c = *reinterpret_cast<const float4*>(&S.box[stage][3][row * BOX_W + 4 * xg + 4 * q]);
      const float gg[4] = {g.x, g.y, g.z, g.w}, aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w},
                  cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int i = 4 * q + e - (HX - HALO);
        if (i >= 0 && i < 14) { P[i] = mul2(pk(aa[e], bb[e]), pk(gg[e], gg[e])); Q[i] = cc[e] * gg[e]; }
      }
    }
    float2 o01[4];
    float o2[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float wc = c_w[HALO];
      f2 a1 = mul2(P[j + HALO], pk(wc, wc));
      float a2 = Q[j + HALO] * wc;
#pragma unroll
      for (int d = 1; d <= HALO; d++) {
        const float w = c_w[HALO - d];
        a1 = fma2(add2(P[j + HALO - d], P[j + HALO + d]), pk(w, w), a1);
        a2 = fmaf(Q[j + HALO - d] + Q[j + HALO + d], w, a2);
      }
      upk(a1, o01[j].x, o01[j].y);
      o2[j] = a2;
    }
    float4* d01 = reinterpret_cast<float4*>(&S.h01[row][4 * xg]);
    d01[0] = make_float4(o01[0].x, o01[0].y, o01[1].x, o01[1].y);
    d01[1] = make_float4(o01[2].x, o01[2].y, o01[3].x, o01[3].y);
    *reinterpret_cast<float4*>(&S.h2[row][4 * xg]) = make_float4(o2[0], o2[1], o2[2], o2[3]);
  }
  __syncthreads();
  if (USE_TMA && t == 0 && tile + (int)gridDim.x < it.ntiles) request(tile + gridDim.x, 0);   // boxes are free again

  const int cg = t & 31, rg = t >> 5;
  const int lx = 2 * cg, ly = 4 * rg;
  f2 v01[4][2];
  float v2[4][2];
#pragma unroll
  for (int r = 0; r < 4; r++)
#pragma unroll
    for (int c = 0; c < 2; c++) { v01[r][c] = pk(0.f, 0.f); v2[r][c] = 0.f; }
#pragma unroll
  for (int i = 0; i < 14; i++) {
    const float4 a = *reinterpret_cast<const float4*>(&S.h01[ly + i][lx]);
    const float2 c2 = *reinterpret_cast<const float2*>(&S.h2[ly + i][lx]);
    const f2 a0 = pk(a.x, a.y), a1 = pk(a.z, a.w);
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int k = i - r;
      if (k >= 0 && k <= 10) {
        const float w = c_w[k];
        const f2 w2 = pk(w, w);
        v01[r][0] = fma2(a0, w2, v01[r][0]); v01[r][1] = fma2(a1, w2, v01[r][1]);
        v2[r][0] = fmaf(c2.x, w, v2[r][0]); v2[r][1] = fmaf(c2.y, w, v2[r][1]);
      }
    }
  }
  const int gx = x0 + lx;
  const bool vec_ok = (W & 1) == 0;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int gy = y0 + ly + r;
    if (gy >= H || gx >= W) continue;
    const size_t o = poff + (size_t)gy * W + gx;
    float s0[2], s1[2];
    upk(v01[r][0], s0[0], s1[0]);
    upk(v01[r][1], s0[1], s1[1]);
    if (vec_ok && gx + 1 < W) {
      const float2 p1 = *reinterpret_cast<const float2*>(img1 + o), p2 = *reinterpret_cast<const float2*>(img2 + o);
      *reinterpret_cast<float2*>(dL_dimg1 + o) = make_float2(s0[0] + (2.f * p1.x) * s1[0] + p2.x * v2[r][0],
                                                             s0[1] + (2.f * p1.y) * s1[1] + p2.y * v2[r][1]);
    } else {
#pragma unroll
      for (int c = 0; c < 2; c++)
        if (gx + c < W) dL_dimg1[o + c] = s0[c] + (2.f * img1[o + c]) * s1[c] + img2[o + c] * v2[r][c];
    }
  }
  __syncthreads();      // the vertical pass is done with h01/h2 before the next tile's horizontal pass rewrites them
  }   // tile loop
}

// ---- tensor maps ----------------------------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

// [planes, H, W] float tensor, box {BOX_W, BOX_H, 1}, zero fill outside
bool make_map(CUtensorMap* m, const float* base, int planes, int H, int W) {
  auto fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes};
  const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
  const cuuint32_t box[3] = {BOX_W, BOX_H, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool tma_ok(const void* p, int W) { return (W % 4) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int sm_count() {
  static int n[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (n[dev] == 0) { int v = 132; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev); n[dev] = v > 0 ? v : 132; }
  return n[dev];
}

template <typename K>
void opt_in(K kernel, size_t smem) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); }

}  // namespace

extern "C" {

const char* sfgs_last_error(void);
int sfgs_set_error(int code, const char* what, int cuda_error);   // sfgs_api.cu

int sfgs_fusedssim_forward(float C1, float C2, int B, int CH, int H, int W, const float* img1, const float* img2,
                           int train, float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12,
                           void* stream) {
  if (B < 0 || CH < 0 || H < 0 || W < 0) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_forward: bad sizes", 0);
  if (B == 0 || CH == 0 || H == 0 || W == 0) return SFGS_OK;   // empty batch: nothing to write
  if (!img1 || !img2 || !ssim_map) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_forward: null pointer", 0);
  if (train && (!dm_dmu1 || !dm_dsigma1_sq || !dm_dsigma12)) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_forward: null derivative map", 0);
  for (const void* p : {(const void*)ssim_map, (const void*)dm_dmu1, (const void*)dm_dsigma1_sq, (const void*)dm_dsigma12})
    if (p && (reinterpret_cast<uintptr_t>(p) & 7)) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_forward: outputs must be 8-byte aligned", 0);
  const int planes = B * CH;
  const long long ntiles = (long long)((W + TW - 1) / TW) * ((H + TH - 1) / TH) * planes;
  const int grid = (int)(ntiles < 2LL * sm_count() ? ntiles : 2LL * sm_count());   // persistent: two CTAs per SM
  Maps4 tm = {};
  const bool use_tma = tma_ok(img1, W) && tma_ok(img2, W) && make_map(&tm.m[0], img1, planes, H, W) &&
                       make_map(&tm.m[1], img2, planes, H, W);
  static SfgsPerDeviceOnce once;
  if (once.first_use()) {
    opt_in(ssim_fwd_kernel<true, true>, sizeof(FwdSmem));  opt_in(ssim_fwd_kernel<true, false>, sizeof(FwdSmem));
    opt_in(ssim_fwd_kernel<false, true>, sizeof(FwdSmem)); opt_in(ssim_fwd_kernel<false, false>, sizeof(FwdSmem));
  }
  cudaStream_t st = (cudaStream_t)stream;
  SFGS_COUNT_LAUNCH();
#define SSIM_FWD(TR, TM) ssim_fwd_kernel<TR, TM><<<grid, SSIM_THREADS, sizeof(FwdSmem), st>>>( \
      tm, H, W, planes, C1, C2, img1, img2, ssim_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
  if (train) { if (use_tma) SSIM_FWD(true, true); else SSIM_FWD(true, false); }
  else { if (use_tma) SSIM_FWD(false, true); else SSIM_FWD(false, false); }
#undef SSIM_FWD
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : sfgs_set_error(SFGS_E_CUDA, "fusedssim_forward", (int)e);
}

int sfgs_fusedssim_backward(float C1, float C2, int B, int CH, int H, int W, const float* img1, const float* img2,
                            const float* dL_dmap, const float* dm_dmu1, const float* dm_dsigma1_sq,
                            const float* dm_dsigma12, float* dL_dimg1, void* stream) {
  (void)C1; (void)C2;
  if (B < 0 || CH < 0 || H < 0 || W < 0) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_backward: bad sizes", 0);
  if (B == 0 || CH == 0 || H == 0 || W == 0) return SFGS_OK;
  if (!img1 || !img2 || !dL_dmap || !dm_dmu1 || !dm_dsigma1_sq || !dm_dsigma12 || !dL_dimg1)
    return sfgs_set_error(SFGS_E_BADARG, "fusedssim_backward: null pointer", 0);
  for (const void* p : {(const void*)img1, (const void*)img2, (const void*)dL_dimg1})
    if (reinterpret_cast<uintptr_t>(p) & 7) return sfgs_set_error(SFGS_E_BADARG, "fusedssim_backward: images must be 8-byte aligned", 0);
  const int planes = B * CH;
  const long long ntiles = (long long)((W + TW - 1) / TW) * ((H + TH - 1) / TH) * planes;
  const int grid = (int)(ntiles < 2LL * sm_count() ? ntiles : 2LL * sm_count());   // persistent: two CTAs per SM
  Maps4 tm = {};
  const float* src[4] = {dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12};
  bool use_tma = true;
  for (int k = 0; k < 4 && use_tma; k++) use_tma = tma_ok(src[k], W) && make_map(&tm.m[k], src[k], planes, H, W);
  static SfgsPerDeviceOnce once;
  if (once.first_use()) { opt_in(ssim_bwd_kernel<true>, sizeof(BwdSmem)); opt_in(ssim_bwd_kernel<false>, sizeof(BwdSmem)); }
  cudaStream_t st = (cudaStream_t)stream;
  SFGS_COUNT_LAUNCH();
  if (use_tma)
    ssim_bwd_kernel<true><<<grid, SSIM_THREADS, sizeof(BwdSmem), st>>>(tm, H, W, planes, img1, img2, dL_dmap, dm_dmu1,
                                                                     dm_dsigma1_sq, dm_dsigma12, dL_dimg1);
  else
    ssim_bwd_kernel<false><<<grid, SSIM_THREADS, sizeof(BwdSmem), st>>>(tm, H, W, planes, img1, img2, dL_dmap, dm_dmu1,
                                                                      dm_dsigma1_sq, dm_dsigma12, dL_dimg1);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : sfgs_set_error(SFGS_E_CUDA, "fusedssim_backward", (int)e);
}

}  // extern "C"
