// sfgs_gauss_bwd.cu — per-Gaussian adjoint: conic -> cov2D -> cov3D -> scale/rot,
// projected mean -> 3D mean, depth -> mean, RGB -> SH (+ view direction -> mean),
// normal -> rotation.
//
// Fuses computeCov2DCUDA and the backward preprocessCUDA
// (RAST/cuda_rasterizer/backward.cu:144-310, 433-506) with the twelve
// torch::zeros fills of RasterizeGaussiansBackwardCUDA
// (RAST/rasterize_points.cu:180-196): one thread per Gaussian reads the 14
// blend-adjoint sums produced by the tile kernel, runs the whole chain in
// registers; the block first zero-fills its span of every output array with
// coalesced stores, so no output needs a prior memset, then only the visible
// Gaussians — compacted into dense warps — run the adjoint chain and overwrite
// their rows.
#include "sfgs_common.cuh"
#include <cstdlib>

namespace {

constexpr int GB_THREADS = 128;
constexpr int GB_SPAN = 256;   // Gaussians per block (two per thread in the cheap phases)

__device__ __forceinline__ void rot_from_quat(float r, float x, float y, float z, float R[3][3]) {
  R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
  R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
  R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// d(v/|v|)/dv applied to dv — auxiliary.h:108-119
__device__ __forceinline__ float3 dnormvdv3(float3 v, float3 dv) {
  const float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
  const float invsum32 = 1.0f / sqrt(sum2 * sum2 * sum2);
  float3 o;
  o.x = ((+sum2 - v.x * v.x) * dv.x - v.y * v.x * dv.y - v.z * v.x * dv.z) * invsum32;
  o.y = (-v.x * v.y * dv.x + (sum2 - v.y * v.y) * dv.y - v.z * v.y * dv.z) * invsum32;
  o.z = (-v.x * v.z * dv.x - v.y * v.z * dv.y + (sum2 - v.z * v.z) * dv.z) * invsum32;
  return o;
}

template <bool WRITE_SH, int MIN_CTAS>
__global__ void __launch_bounds__(GB_THREADS, MIN_CTAS)
gauss_bwd_kernel(int g_begin, int g_end, int acc_row0, int D, int M, const float* __restrict__ means3D, const int* __restrict__ radii,
                 const float* __restrict__ shs, const unsigned char* __restrict__ clamped,
                 const float* __restrict__ scales, const float* __restrict__ rotations, float scale_modifier,
                 const float* __restrict__ cov3Ds, const float* __restrict__ rec,
                 const float* __restrict__ norm3D_precomp, const float* __restrict__ view,
                 const float* __restrict__ proj, float h_x, float h_y, float tan_fovx, float tan_fovy,
                 float kernel_size, const float* __restrict__ campos, const float* __restrict__ acc,
                 float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity,
                 float* __restrict__ dL_dcolor, float* __restrict__ dL_ddepth, float* __restrict__ dL_dmean3D,
                 float* __restrict__ dL_dcov3D, float* __restrict__ dL_dnorm3D, float* __restrict__ dL_dsh,
                 float* __restrict__ dL_dscale, float* __restrict__ dL_drot) {
  // 24 KB tile: column t of a [12][128] float4 array receives thread t's SH coefficients by cp.async
  // (fast path), or 19 floats of per-thread scratch for the generic dL_dsh store
  __shared__ __align__(128) float s_tile[WRITE_SH ? GB_THREADS * 48 : 4];
  __shared__ unsigned short s_list[GB_SPAN];
  __shared__ unsigned char s_vis[GB_SPAN];
  __shared__ int s_cnt[2 * GB_THREADS / 32];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int base = g_begin + blockIdx.x * GB_SPAN;           // Gaussians [g_begin, g_end) are this launch's share
  const int nspan = min(GB_SPAN, g_end - base);

  // ---------------- phase A: which Gaussians of the span were rasterized ----------------
  // Culled Gaussians (64 % of the 1M-Gaussian benchmark frame) only need zeros.  Running the adjoint chain
  // thread-per-Gaussian left 36 % of the lanes of every warp doing useful work; instead the visible ones are
  // compacted (in index order) and processed by dense warps.
  bool vis[2];
  unsigned bal[2];
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int g = r * GB_THREADS + t;
    vis[r] = g < nspan && radii[base + g] > 0;
    bal[r] = __ballot_sync(0xffffffffu, vis[r]);
    s_vis[g] = vis[r] ? 1 : 0;
    if (lane == 0) s_cnt[r * (GB_THREADS / 32) + wid] = __popc(bal[r]);
  }
  __syncthreads();
  int nvis = 0;
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int seg = r * (GB_THREADS / 32) + wid;
    int off = 0;
#pragma unroll
    for (int q = 0; q < 2 * GB_THREADS / 32; q++) off += q < seg ? s_cnt[q] : 0;
    if (vis[r]) s_list[off + __popc(bal[r] & ((1u << lane) - 1u))] = (unsigned short)(r * GB_THREADS + t);
  }
#pragma unroll
  for (int q = 0; q < 2 * GB_THREADS / 32; q++) nvis += s_cnt[q];

  // every output row of the span starts as zeros: contiguous, 16-byte stores wherever the caller's buffer allows
  if (nvis < nspan) {
    auto zero_fill = [&](float* dst, int width) {
      const int nfl = nspan * width;
      float* d = dst + (size_t)base * width;
      const int nv4 = ((reinterpret_cast<uintptr_t>(d) & 15) == 0) ? (nfl >> 2) : 0;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int i = t; i < nv4; i += GB_THREADS) reinterpret_cast<float4*>(d)[i] = z;
      for (int i = (nv4 << 2) + t; i < nfl; i += GB_THREADS) d[i] = 0.f;
    };
    zero_fill(dL_dmean2D, 3);
    zero_fill(dL_dconic, 4);
    zero_fill(dL_dopacity, 1);
    zero_fill(dL_dcolor, 3);
    zero_fill(dL_ddepth, 1);
    zero_fill(dL_dmean3D, 3);
    zero_fill(dL_dcov3D, 6);
    zero_fill(dL_dnorm3D, 3);
    zero_fill(dL_dscale, 3);
    zero_fill(dL_drot, 4);
    if (WRITE_SH) {
      // dL_dsh is 2/3 of the output bytes: its rows are whole 16-byte units when M is a multiple of 4 and the
      // buffer is aligned, so the rows the dense warps are about to write anyway are skipped
      float* d = dL_dsh + (size_t)base * 3 * M;
      if ((M & 3) == 0 && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
        const int q_per_row = 3 * M / 4, nq = nspan * q_per_row;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = t; i < nq; i += GB_THREADS)
          if (!s_vis[i / q_per_row]) reinterpret_cast<float4*>(d)[i] = z;
      } else {
        zero_fill(dL_dsh, 3 * M);
      }
    }
  }
  __syncthreads();   // orders the zero fill before the row stores below, and publishes s_list

  const bool sh_fast = WRITE_SH && shs != nullptr && M == 16 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(dL_dsh) & 15) == 0;
  const bool sh_staged = sh_fast;
  const int sh_nq = D == 0 ? 1 : (D == 1 ? 3 : (D == 2 ? 7 : 12));   // float4s covering (D+1)^2 coefficients

  // ---------------- phase B: dense warps over the visible Gaussians ----------------
  for (int k = t; k < nvis; k += GB_THREADS) {
    const int idx = base + (int)s_list[k];
    const size_t i = (size_t)idx;
    float o_mean2D[3] = {0, 0, 0}, o_conic[4] = {0, 0, 0, 0}, o_opac = 0, o_color[3] = {0, 0, 0}, o_depth = 0;
    float o_mean[3] = {0, 0, 0}, o_cov[6] = {0, 0, 0, 0, 0, 0}, o_norm[3] = {0, 0, 0};
    float o_scale[3] = {0, 0, 0}, o_rot[4] = {0, 0, 0, 0};
    float dsh_scale[16];   // dRGB/dsh_k for k < (D+1)^2, else 0
#pragma unroll
    for (int q = 0; q < 16; q++) dsh_scale[q] = 0.f;
    float dL_dRGB[3] = {0, 0, 0};

    if (sh_staged) {
      const float4* g4 = reinterpret_cast<const float4*>(shs + i * 48);
      float4* s4 = reinterpret_cast<float4*>(s_tile);
#pragma unroll
      for (int q = 0; q < 12; q++)
        if (q < sh_nq) {
          const unsigned sa = (unsigned)__cvta_generic_to_shared(&s4[q * GB_THREADS + threadIdx.x]);
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(g4 + q));
        }
      asm volatile("cp.async.commit_group;\n" ::);
    }
    const float mx = means3D[3 * i], my = means3D[3 * i + 1], mz = means3D[3 * i + 2];
    float4 q_in = make_float4(0.f, 0.f, 0.f, 0.f);
    float scx = 0.f, scy = 0.f, scz = 0.f;
    if (scales != nullptr) {
      q_in = *reinterpret_cast<const float4*>(rotations + 4 * i);
      scx = scales[3 * i]; scy = scales[3 * i + 1]; scz = scales[3 * i + 2];
    }
    const unsigned cm = shs != nullptr ? clamped[idx] : 0u;
    const float4* a4 = reinterpret_cast<const float4*>(acc + (i - (size_t)acc_row0) * 16);
    const float4 A0 = a4[0], A1 = a4[1], A2 = a4[2], A3 = a4[3];
    const float4 rec1 = *reinterpret_cast<const float4*>(rec + i * REC_FLOATS + 4);    // con.z, opacity*coef, depth
    const float4 rec2 = *reinterpret_cast<const float4*>(rec + i * REC_FLOATS + 8);    // r, g, b, nx
    const float4 rec3 = *reinterpret_cast<const float4*>(rec + i * REC_FLOATS + 12);   // ny, nz
    o_color[0] = A0.x; o_color[1] = A0.y; o_color[2] = A0.z; o_depth = A0.w;
    o_norm[0] = A1.x; o_norm[1] = A1.y; o_norm[2] = A1.z;
    o_mean2D[0] = A1.w; o_mean2D[1] = A2.x; o_mean2D[2] = A2.y;
    o_conic[0] = A2.z; o_conic[1] = A2.w; o_conic[3] = A3.x;
    o_opac = A3.y;

    const float* cov3D = cov3Ds + 6 * i;
    const float combined_opacity = rec1.y;

    // ---------------- conic -> cov2D -> cov3D, t (computeCov2DCUDA) ----------------
    {
      const float dLcx = o_conic[0], dLcy = o_conic[1], dLcz = o_conic[3];
      float tx = view[0] * mx + view[4] * my + view[8] * mz + view[12];
      float ty = view[1] * mx + view[5] * my + view[9] * mz + view[13];
      const float tz = view[2] * mx + view[6] * my + view[10] * mz + view[14];
      const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
      const float txtz = tx / tz, tytz = ty / tz;
      tx = min(limx, max(-limx, txtz)) * tz;
      ty = min(limy, max(-limy, tytz)) * tz;
      const float x_grad_mul = txtz < -limx || txtz > limx ? 0 : 1;
      const float y_grad_mul = tytz < -limy || tytz > limy ? 0 : 1;

      const float a0 = h_x / tz, a2 = -(h_x * tx) / (tz * tz);
      const float b1 = h_y / tz, b2 = -(h_y * ty) / (tz * tz);
      // W[c][r]
      const float Wm[3][3] = {{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}};
      float T[3][3];   // T[c][r]
#pragma unroll
      for (int r = 0; r < 3; r++) {
        T[0][r] = Wm[0][r] * a0 + Wm[1][r] * 0.0f + Wm[2][r] * a2;
        T[1][r] = Wm[0][r] * 0.0f + Wm[1][r] * b1 + Wm[2][r] * b2;
        T[2][r] = 0.f;
      }
      const float Vrk[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}};
      // X[c][r] = T[r][0]*Vrk[0][c] + T[r][1]*Vrk[1][c] + T[r][2]*Vrk[2][c]
      float X[3][2];
#pragma unroll
      for (int c = 0; c < 3; c++) {
        X[c][0] = T[0][0] * Vrk[0][c] + T[0][1] * Vrk[1][c] + T[0][2] * Vrk[2][c];
        X[c][1] = T[1][0] * Vrk[0][c] + T[1][1] * Vrk[1][c] + T[1][2] * Vrk[2][c];
      }
      const float c00 = X[0][0] * T[0][0] + X[1][0] * T[0][1] + X[2][0] * T[0][2];
      const float c01 = X[0][1] * T[0][0] + X[1][1] * T[0][1] + X[2][1] * T[0][2];
      const float c11 = X[0][1] * T[1][0] + X[1][1] * T[1][1] + X[2][1] * T[1][2];

      const float det_0 = fmax(1e-6, (double)(c00 * c11 - c01 * c01));
      const float det_1 = fmax(1e-6, (double)((c00 + kernel_size) * (c11 + kernel_size) - c01 * c01));
      const float coef = sqrt(det_0 / (det_1 + 1e-6) + 1e-6);
      const float opacity = combined_opacity / (coef + 1e-6);
      const float dL_dcoef = o_opac * opacity;
      const float dL_dsqrtcoef = dL_dcoef * 0.5 * 1. / (coef + 1e-6);
      const float dL_ddet0 = dL_dsqrtcoef / (det_1 + 1e-6);
      const float dL_ddet1 = dL_dsqrtcoef * det_0 * (-1.f / (det_1 * det_1 + 1e-6));
      const float dcoef_da = dL_ddet0 * c11 + dL_ddet1 * (c11 + kernel_size);
      const float dcoef_db = dL_ddet0 * (-2. * c01) + dL_ddet1 * (-2. * c01);
      const float dcoef_dc = dL_ddet0 * c00 + dL_ddet1 * (c00 + kernel_size);

      const float a = c00 + kernel_size, b = c01, c = c11 + kernel_size;
      const float denom = a * c - b * b;
      float dL_da = 0, dL_db = 0, dL_dc = 0;
      const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
      if (denom2inv != 0) {
        dL_da = denom2inv * (-c * c * dLcx + 2 * b * c * dLcy + (denom - a * c) * dLcz);
        dL_dc = denom2inv * (-a * a * dLcz + 2 * a * b * dLcy + (denom - a * c) * dLcx);
        dL_db = denom2inv * 2 * (b * c * dLcx - (denom + 2 * b * b) * dLcy + a * b * dLcz);
        if (det_0 <= 1e-6 || det_1 <= 1e-6) {
          o_opac = 0;
        } else {
          dL_da += dcoef_da; dL_dc += dcoef_dc; dL_db += dcoef_db;
          o_opac = o_opac * coef;
        }
        o_cov[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
        o_cov[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
        o_cov[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
        o_cov[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][1] * dL_dc;
        o_cov[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][2] * dL_dc;
        o_cov[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db + 2 * T[1][1] * T[1][2] * dL_dc;
      }
      // dL/dT (upper 2x3), dL/dJ, dL/dt
      const float dL_dT00 = 2 * (T[0][0] * Vrk[0][0] + T[0][1] * Vrk[0][1] + T[0][2] * Vrk[0][2]) * dL_da +
                            (T[1][0] * Vrk[0][0] + T[1][1] * Vrk[0][1] + T[1][2] * Vrk[0][2]) * dL_db;
      const float dL_dT01 = 2 * (T[0][0] * Vrk[1][0] + T[0][1] * Vrk[1][1] + T[0][2] * Vrk[1][2]) * dL_da +
                            (T[1][0] * Vrk[1][0] + T[1][1] * Vrk[1][1] + T[1][2] * Vrk[1][2]) * dL_db;
      const float dL_dT02 = 2 * (T[0][0] * Vrk[2][0] + T[0][1] * Vrk[2][1] + T[0][2] * Vrk[2][2]) * dL_da +
                            (T[1][0] * Vrk[2][0] + T[1][1] * Vrk[2][1] + T[1][2] * Vrk[2][2]) * dL_db;
      const float dL_dT10 = 2 * (T[1][0] * Vrk[0][0] + T[1][1] * Vrk[0][1] + T[1][2] * Vrk[0][2]) * dL_dc +
                            (T[0][0] * Vrk[0][0] + T[0][1] * Vrk[0][1] + T[0][2] * Vrk[0][2]) * dL_db;
      const float dL_dT11 = 2 * (T[1][0] * Vrk[1][0] + T[1][1] * Vrk[1][1] + T[1][2] * Vrk[1][2]) * dL_dc +
                            (T[0][0] * Vrk[1][0] + T[0][1] * Vrk[1][1] + T[0][2] * Vrk[1][2]) * dL_db;
      const float dL_dT12 = 2 * (T[1][0] * Vrk[2][0] + T[1][1] * Vrk[2][1] + T[1][2] * Vrk[2][2]) * dL_dc +
                            (T[0][0] * Vrk[2][0] + T[0][1] * Vrk[2][1] + T[0][2] * Vrk[2][2]) * dL_db;
      const float dL_dJ00 = Wm[0][0] * dL_dT00 + Wm[0][1] * dL_dT01 + Wm[0][2] * dL_dT02;
      const float dL_dJ02 = Wm[2][0] * dL_dT00 + Wm[2][1] * dL_dT01 + Wm[2][2] * dL_dT02;
      const float dL_dJ11 = Wm[1][0] * dL_dT10 + Wm[1][1] * dL_dT11 + Wm[1][2] * dL_dT12;
      const float dL_dJ12 = Wm[2][0] * dL_dT10 + Wm[2][1] * dL_dT11 + Wm[2][2] * dL_dT12;
      const float tzi = 1.f / tz, tz2 = tzi * tzi, tz3 = tz2 * tzi;
      const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
      const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
      const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * tx) * tz3 * dL_dJ02 + (2 * h_y * ty) * tz3 * dL_dJ12;
      // view^T (3x3 part)
      o_mean[0] = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
      o_mean[1] = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
      o_mean[2] = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;
    }

    // ---------------- projected centre and depth -> mean (preprocessCUDA bwd) ----------------
    {
      const float hw = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
      const float m_w = 1.0f / (hw + 0.0000001f);
      const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
      const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
      const float gx = o_mean2D[0], gy = o_mean2D[1];
      const float d0 = (proj[0] * m_w - proj[3] * mul1) * gx + (proj[1] * m_w - proj[3] * mul2) * gy;
      const float d1 = (proj[4] * m_w - proj[7] * mul1) * gx + (proj[5] * m_w - proj[7] * mul2) * gy;
      const float d2 = (proj[8] * m_w - proj[11] * mul1) * gx + (proj[9] * m_w - proj[11] * mul2) * gy;
      o_mean[0] += d0; o_mean[1] += d1; o_mean[2] += d2;
      const float mul3 = view[2] * mx + view[6] * my + view[10] * mz + view[14];
      const float e0 = (view[2] - view[3] * mul3) * o_depth;
      const float e1 = (view[6] - view[7] * mul3) * o_depth;
      const float e2 = (view[10] - view[11] * mul3) * o_depth;
      o_mean[0] += e0; o_mean[1] += e1; o_mean[2] += e2;
    }

    // ---------------- RGB -> SH and view direction -> mean ----------------
    if (shs != nullptr) {
      const float ox = mx - campos[0], oy = my - campos[1], oz = mz - campos[2];
      const float len = sqrt(ox * ox + oy * oy + oz * oz);
      const float x = ox / len, y = oy / len, z = oz / len;
      dL_dRGB[0] = o_color[0] * ((cm & 1u) ? 0 : 1);
      dL_dRGB[1] = o_color[1] * ((cm & 2u) ? 0 : 1);
      dL_dRGB[2] = o_color[2] * ((cm & 4u) ? 0 : 1);
      auto sh_adjoint = [&](auto sh) {
        float dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0};
        dsh_scale[0] = SH_C0;
        if (D > 0) {
          dsh_scale[1] = -SH_C1 * y; dsh_scale[2] = SH_C1 * z; dsh_scale[3] = -SH_C1 * x;
  #pragma unroll
          for (int ch = 0; ch < 3; ch++) {
            dRGBdx[ch] = -SH_C1 * sh(3 * 3 + ch);
            dRGBdy[ch] = -SH_C1 * sh(1 * 3 + ch);
            dRGBdz[ch] = SH_C1 * sh(2 * 3 + ch);
          }
          if (D > 1) {
            const float xx = x * x, yy = y * y, zz = z * z;
            const float xy = x * y, yz = y * z, xz = x * z;
            dsh_scale[4] = SH_C2_0 * xy; dsh_scale[5] = SH_C2_1 * yz; dsh_scale[6] = SH_C2_2 * (2.f * zz - xx - yy);
            dsh_scale[7] = SH_C2_3 * xz; dsh_scale[8] = SH_C2_4 * (xx - yy);
  #pragma unroll
            for (int ch = 0; ch < 3; ch++) {
              const float s4 = sh(4 * 3 + ch), s5 = sh(5 * 3 + ch), s6 = sh(6 * 3 + ch), s7 = sh(7 * 3 + ch), s8 = sh(8 * 3 + ch);
              dRGBdx[ch] += SH_C2_0 * y * s4 + SH_C2_2 * 2.f * -x * s6 + SH_C2_3 * z * s7 + SH_C2_4 * 2.f * x * s8;
              dRGBdy[ch] += SH_C2_0 * x * s4 + SH_C2_1 * z * s5 + SH_C2_2 * 2.f * -y * s6 + SH_C2_4 * 2.f * -y * s8;
              dRGBdz[ch] += SH_C2_1 * y * s5 + SH_C2_2 * 2.f * 2.f * z * s6 + SH_C2_3 * x * s7;
            }
            if (D > 2) {
              dsh_scale[9] = SH_C3_0 * y * (3.f * xx - yy);
              dsh_scale[10] = SH_C3_1 * xy * z;
              dsh_scale[11] = SH_C3_2 * y * (4.f * zz - xx - yy);
              dsh_scale[12] = SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy);
              dsh_scale[13] = SH_C3_4 * x * (4.f * zz - xx - yy);
              dsh_scale[14] = SH_C3_5 * z * (xx - yy);
              dsh_scale[15] = SH_C3_6 * x * (xx - 3.f * yy);
  #pragma unroll
              for (int ch = 0; ch < 3; ch++) {
                const float s9 = sh(9 * 3 + ch), s10 = sh(10 * 3 + ch), s11 = sh(11 * 3 + ch), s12 = sh(12 * 3 + ch);
                const float s13 = sh(13 * 3 + ch), s14 = sh(14 * 3 + ch), s15 = sh(15 * 3 + ch);
                dRGBdx[ch] += (SH_C3_0 * s9 * 3.f * 2.f * xy + SH_C3_1 * s10 * yz + SH_C3_2 * s11 * -2.f * xy +
                               SH_C3_3 * s12 * -3.f * 2.f * xz + SH_C3_4 * s13 * (-3.f * xx + 4.f * zz - yy) +
                               SH_C3_5 * s14 * 2.f * xz + SH_C3_6 * s15 * 3.f * (xx - yy));
                dRGBdy[ch] += (SH_C3_0 * s9 * 3.f * (xx - yy) + SH_C3_1 * s10 * xz +
                               SH_C3_2 * s11 * (-3.f * yy + 4.f * zz - xx) + SH_C3_3 * s12 * -3.f * 2.f * yz +
                               SH_C3_4 * s13 * -2.f * xy + SH_C3_5 * s14 * -2.f * yz + SH_C3_6 * s15 * -3.f * 2.f * xy);
                dRGBdz[ch] += (SH_C3_1 * s10 * xy + SH_C3_2 * s11 * 4.f * 2.f * yz +
                               SH_C3_3 * s12 * 3.f * (2.f * zz - xx - yy) + SH_C3_4 * s13 * 4.f * 2.f * xz +
                               SH_C3_5 * s14 * (xx - yy));
              }
            }
          }
        }
        float3 dL_ddir;
        dL_ddir.x = dRGBdx[0] * dL_dRGB[0] + dRGBdx[1] * dL_dRGB[1] + dRGBdx[2] * dL_dRGB[2];
        dL_ddir.y = dRGBdy[0] * dL_dRGB[0] + dRGBdy[1] * dL_dRGB[1] + dRGBdy[2] * dL_dRGB[2];
        dL_ddir.z = dRGBdz[0] * dL_dRGB[0] + dRGBdz[1] * dL_dRGB[1] + dRGBdz[2] * dL_dRGB[2];
        const float3 dm = dnormvdv3(make_float3(ox, oy, oz), dL_ddir);
        o_mean[0] += dm.x; o_mean[1] += dm.y; o_mean[2] += dm.z;
      };
      if (sh_staged) {
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        const float* sf = s_tile + 4 * threadIdx.x;   // coefficient j = word (j & 3) of float4 [j >> 2][t]
        sh_adjoint([&](int j) { return sf[(j >> 2) * (4 * GB_THREADS) + (j & 3)]; });
      } else {
        const float* shg = shs + i * M * 3;
        sh_adjoint([&](int j) { return shg[j]; });
      }
    }

    // ---------------- cov3D -> scale / rotation, normal -> rotation ----------------
    if (scales != nullptr) {
      const float r = q_in.x, x = q_in.y, y = q_in.z, z = q_in.w;
      float R[3][3];
      rot_from_quat(r, x, y, z, R);
      const float s[3] = {scale_modifier * scx, scale_modifier * scy, scale_modifier * scz};
      float Mm[3][3];   // M = S * R : M[c][r] = s[r] * R[c][r]
#pragma unroll
      for (int c = 0; c < 3; c++) { Mm[c][0] = s[0] * R[c][0]; Mm[c][1] = s[1] * R[c][1]; Mm[c][2] = s[2] * R[c][2]; }
      const float* g = o_cov;
      // dL_dSigma (symmetric, off-diagonals halved), columns
      const float Sg[3][3] = {{g[0], 0.5f * g[1], 0.5f * g[2]}, {0.5f * g[1], g[3], 0.5f * g[4]}, {0.5f * g[2], 0.5f * g[4], g[5]}};
      // dL_dM = 2 * M * dL_dSigma : (2M)[c][r] = 2*M[c][r]; out[c][r] = sum_k (2M)[k][r] * Sg[c][k]
      float dM[3][3];
#pragma unroll
      for (int c = 0; c < 3; c++)
#pragma unroll
        for (int rr = 0; rr < 3; rr++)
          dM[c][rr] = (2.0f * Mm[0][rr]) * Sg[c][0] + (2.0f * Mm[1][rr]) * Sg[c][1] + (2.0f * Mm[2][rr]) * Sg[c][2];
      // Rt[c][r] = R[r][c]; dMt[c][r] = dM[r][c]
      float dMt[3][3];
#pragma unroll
      for (int c = 0; c < 3; c++)
#pragma unroll
        for (int rr = 0; rr < 3; rr++) dMt[c][rr] = dM[rr][c];
      o_scale[0] = R[0][0] * dMt[0][0] + R[1][0] * dMt[0][1] + R[2][0] * dMt[0][2];
      o_scale[1] = R[0][1] * dMt[1][0] + R[1][1] * dMt[1][1] + R[2][1] * dMt[1][2];
      o_scale[2] = R[0][2] * dMt[2][0] + R[1][2] * dMt[2][1] + R[2][2] * dMt[2][2];
#pragma unroll
      for (int k = 0; k < 3; k++) { dMt[0][k] *= s[0]; dMt[1][k] *= s[1]; dMt[2][k] *= s[2]; }
      o_rot[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
      o_rot[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
      o_rot[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
      o_rot[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);

      if (norm3D_precomp == nullptr) {
        // normal -> rotation (computeNorm3D bwd, backward.cu:380-428); the raw (unscaled) scales pick the axis
        float ax0, ax1, ax2;
        if (scx > scz && scy > scz) { ax0 = 0.f; ax1 = 0.f; ax2 = 1.f; }
        else if (scx > scy && scz > scy) { ax0 = 0.f; ax1 = 1.f; ax2 = 0.f; }
        else { ax0 = 1.f; ax1 = 0.f; ax2 = 0.f; }
        const float n3x = rec2.w, n3y = rec3.x, n3z = rec3.y;
        // R * axis : out[r] = R[0][r]*ax0 + R[1][r]*ax1 + R[2][r]*ax2
        const float rn0 = R[0][0] * ax0 + R[1][0] * ax1 + R[2][0] * ax2;
        const float rn1 = R[0][1] * ax0 + R[1][1] * ax1 + R[2][1] * ax2;
        const float rn2 = R[0][2] * ax0 + R[1][2] * ax1 + R[2][2] * ax2;
        if (rn0 * n3x + rn1 * n3y + rn2 * n3z < 0) { ax0 = -ax0; ax1 = -ax1; ax2 = -ax2; }
        const float dn[3] = {o_norm[0], o_norm[1], o_norm[2]};
        const float ax[3] = {ax0, ax1, ax2};
        // dL_dR[c][r] = dn[c]*ax[r]; dRt[c][r] = dL_dR[r][c] = dn[r]*ax[c]
        float dRt[3][3];
#pragma unroll
        for (int c = 0; c < 3; c++)
#pragma unroll
          for (int rr = 0; rr < 3; rr++) dRt[c][rr] = dn[rr] * ax[c];
        o_rot[0] += 2 * z * (dRt[0][1] - dRt[1][0]) + 2 * y * (dRt[2][0] - dRt[0][2]) + 2 * x * (dRt[1][2] - dRt[2][1]);
        o_rot[1] += 2 * y * (dRt[1][0] + dRt[0][1]) + 2 * z * (dRt[2][0] + dRt[0][2]) + 2 * r * (dRt[1][2] - dRt[2][1]) - 4 * x * (dRt[2][2] + dRt[1][1]);
        o_rot[2] += 2 * x * (dRt[1][0] + dRt[0][1]) + 2 * r * (dRt[2][0] - dRt[0][2]) + 2 * z * (dRt[1][2] + dRt[2][1]) - 4 * y * (dRt[2][2] + dRt[0][0]);
        o_rot[3] += 2 * r * (dRt[0][1] - dRt[1][0]) + 2 * x * (dRt[2][0] + dRt[0][2]) + 2 * y * (dRt[1][2] + dRt[2][1]) - 4 * z * (dRt[1][1] + dRt[0][0]);
      }
    }

    // ---------------- this Gaussian's rows ----------------
    auto store3 = [&](float* dst, const float* v) { float* d = dst + 3 * i; d[0] = v[0]; d[1] = v[1]; d[2] = v[2]; };
    auto store4 = [&](float* dst, float v0, float v1, float v2, float v3) {
      float* d = dst + 4 * i;
      if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) *reinterpret_cast<float4*>(d) = make_float4(v0, v1, v2, v3);
      else { d[0] = v0; d[1] = v1; d[2] = v2; d[3] = v3; }
    };
    store3(dL_dmean2D, o_mean2D);
    store4(dL_dconic, o_conic[0], o_conic[1], o_conic[2], o_conic[3]);
    dL_dopacity[i] = o_opac;
    store3(dL_dcolor, o_color);
    dL_ddepth[i] = o_depth;
    store3(dL_dmean3D, o_mean);
    {
      float* d = dL_dcov3D + 6 * i;
      if ((reinterpret_cast<uintptr_t>(d) & 7) == 0) {
        reinterpret_cast<float2*>(d)[0] = make_float2(o_cov[0], o_cov[1]);
        reinterpret_cast<float2*>(d)[1] = make_float2(o_cov[2], o_cov[3]);
        reinterpret_cast<float2*>(d)[2] = make_float2(o_cov[4], o_cov[5]);
      } else {
#pragma unroll
        for (int q = 0; q < 6; q++) d[q] = o_cov[q];
      }
    }
    store3(dL_dnorm3D, o_norm);
    store3(dL_dscale, o_scale);
    store4(dL_drot, o_rot[0], o_rot[1], o_rot[2], o_rot[3]);
    if (WRITE_SH) {
      // dL_dsh[g][k][ch] = dRGB/dsh_k(g) * dL_dRGB[ch](g)
      if (sh_fast) {
        float4* d4 = reinterpret_cast<float4*>(dL_dsh + i * 48);
#pragma unroll
        for (int k4 = 0; k4 < 12; k4++) {
          float v[4];
#pragma unroll
          for (int c = 0; c < 4; c++) { const int r = 4 * k4 + c; v[c] = dsh_scale[r / 3] * dL_dRGB[r % 3]; }
          d4[k4] = make_float4(v[0], v[1], v[2], v[3]);
        }
      } else {
        float* sc = s_tile + 19 * t;   // per-thread scratch: dynamic indexing without local memory
#pragma unroll
        for (int q = 0; q < 16; q++) sc[q] = dsh_scale[q];
        sc[16] = dL_dRGB[0]; sc[17] = dL_dRGB[1]; sc[18] = dL_dRGB[2];
        float* d = dL_dsh + i * 3 * M;
        for (int r = 0; r < 3 * M; r++) { const int kk = r / 3, ch = r - 3 * kk; d[r] = (kk < 16 ? sc[kk] : 0.f) * sc[16 + ch]; }
      }
    }
  }
}

}  // namespace

// Clears the [P,16] accumulator rows of rasterized Gaussians only (the blend adjoint touches no other row and the
// per-Gaussian adjoint reads no other row): 64 B x V instead of a 64 B x P memset, and less of the L2 spent on rows
// nobody will use.  Runs right before the blend adjoint, so the lines it writes are L2-resident for the reductions.
namespace {
__global__ void __launch_bounds__(256)
acc_clear_visible_kernel(int P, const int* __restrict__ radii, float* __restrict__ acc) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P || radii[i] <= 0) return;
  float4* a = reinterpret_cast<float4*>(acc + (size_t)i * 16);
  a[0] = a[1] = a[2] = a[3] = make_float4(0.f, 0.f, 0.f, 0.f);
}
}  // namespace

void sfgs_launch_acc_clear_visible(int P, const int* radii, float* acc, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  acc_clear_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, radii, acc);
}

void sfgs_launch_gauss_bwd(const sfgs_backward_args* a, const GeomLayout& g, float focal_x, float focal_y,
                           const float* acc, int g_begin, int g_end, int acc_row0, cudaStream_t st) {
  if (g_end <= g_begin) return;
  const int blocks = (g_end - g_begin + GB_SPAN - 1) / GB_SPAN;
  const float* cov3D_ptr = a->cov3D_precomp != nullptr ? a->cov3D_precomp : g.cov3D;
  SFGS_COUNT_LAUNCH();
#define GB_ARGS                                                                                                       \
  g_begin, g_end, acc_row0, a->D, a->M, a->means3D, a->radii, a->shs, g.clamped, a->scales, a->rotations,             \
      a->scale_modifier, cov3D_ptr, g.rec, a->norm3D_precomp, a->viewmatrix, a->projmatrix, focal_x, focal_y,         \
      a->tan_fovx, a->tan_fovy, a->kernel_size, a->cam_pos, acc, a->dL_dmean2D, a->dL_dconic, a->dL_dopacity,         \
      a->dL_dcolor, a->dL_ddepth, a->dL_dmean3D, a->dL_dcov3D, a->dL_dnorm3D, a->dL_dsh, a->dL_dscale, a->dL_drot
  // resident CTAs per SM of the SH-writing variant: 5 (96 registers); 6 / 7 CTAs would cap it at 80 / 72 registers and
  // spill, 4 CTAs leave fewer warps to hide the gathers.
  if (a->M > 0 && a->dL_dsh != nullptr) {
    gauss_bwd_kernel<true, 5><<<blocks, GB_THREADS, 0, st>>>(GB_ARGS);
  } else {
    gauss_bwd_kernel<false, 5><<<blocks, GB_THREADS, 0, st>>>(GB_ARGS);
  }
#undef GB_ARGS
}
