// sfgs_gauss_bwd.cu — per-Gaussian adjoint: conic -> cov2D -> cov3D -> scale/rot,
// projected mean -> 3D mean, depth -> mean, RGB -> SH (+ view direction -> mean),
// normal -> rotation.
//
// Fuses computeCov2DCUDA and the backward preprocessCUDA
// (RAST/cuda_rasterizer/backward.cu:144-310, 433-506) with the twelve
// torch::zeros fills of RasterizeGaussiansBackwardCUDA
// (RAST/rasterize_points.cu:180-196), so no output needs a prior memset.
//
// The stage moves data more than it computes: every row of every output is written (culled Gaussians get zeros),
// and each rasterized Gaussian reads ~370 B of inputs.  Persistent CTAs therefore walk their share of spans of
// GB_SPAN consecutive Gaussians as a two-stage pipeline:
//   - compaction: each span's radii are ballot-compacted into slots for its rasterized Gaussians (in index order);
//     a stage takes whole spans while their visible Gaussians fit in its GB_SLOTS slots (a fully visible span
//     always fits), so sparse frames still give the adjoint full warps;
//   - gather: cp.async copies the slots' input rows into shared memory, issued one stage ahead so the round trip
//     overlaps the current stage's adjoint and stores;
//   - adjoint: dense threads run the chain (gauss_adjoint) slot by slot from shared memory;
//   - epilogue, span by span: the results are staged in shared memory over the consumed inputs (culled Gaussians
//     as zeros), the ten fixed-width arrays as images of their global ranges and dL_dsh as 19 factors per
//     Gaussian; then the whole CTA writes every output array's contiguous range of the span once, in 16-byte
//     stores.
#include "sfgs_common.cuh"
#include <cstdlib>

namespace {

constexpr int GB_THREADS = 96;
constexpr int GB_SPAN = 96;         // Gaussians per span: one per thread in the compaction
constexpr int GB_SLOTS = 96;        // visible Gaussians per pipeline stage: a span that is entirely visible fits
constexpr int GB_MAX_SPANS = 8;       // spans per stage when few of their Gaussians are visible
constexpr int GB_CTAS_PER_SM = 3;     // three GbShared of 75 KB fit the 228 KB of an SM

// outputs of one Gaussian as the adjoint returns them: the 31 fixed-width gradients, then the 16 dRGB/dsh_k factors and
// the 3 clamp-masked dL/dRGB whose products form dL_dsh
constexpr int O_MEAN2D = 0, O_CONIC = 3, O_OPAC = 7, O_COLOR = 8, O_DEPTH = 11, O_MEAN3D = 12, O_COV = 15,
              O_NORM = 21, O_SCALE = 24, O_ROT = 27, O_SHF = 31, O_RGB = 47, GB_ROW = 50;
constexpr int GB_FIXED = 31;       // fixed-width gradient floats per Gaussian
constexpr int GB_SH_ROW = 19;      // staged dL_dsh factors per Gaussian (odd: rows start in different banks)
constexpr int GB_NFIXED = 10;     // fixed-width output arrays
// camera terms of one Gaussian (the camera adjoint): dL/dviewmatrix[16], dL/dprojmatrix[16], dL/dcampos[3], each in its
// input's element order [4*c + r] (the GB_CAM_POSE pose terms), then dL/dtan_fovx and dL/dtan_fovy (the focal terms)
constexpr int C_VIEW = 0, C_PROJ = 16, C_CAMPOS = 32, GB_CAM_POSE = 35, C_TANX = 35, C_TANY = 36, GB_CAM = 37;

// Shared-memory image of one stage's inputs, indexed by slot (position in the stage's list of visible Gaussians).
// Field-major, so the adjoint's threads (consecutive slots) read consecutive words.
struct GbInputs {
  float4 sh[12][GB_SLOTS];    // SH float j of slot k: word (j & 3) of sh[j >> 2][k]
  float4 acc[4][GB_SLOTS];    // the 16 blend-adjoint sums
  float4 rec[3][GB_SLOTS];    // blend-record floats 4..15 (combined opacity, normal)
  float4 rot[GB_SLOTS];
  float mean[3][GB_SLOTS];
  float scale[3][GB_SLOTS];
  float cov[6][GB_SLOTS];
  unsigned clamped[GB_SLOTS]; // the aligned 4-byte word that holds the Gaussian's clamp bits
};
static_assert(sizeof(float) * ((GB_SH_ROW + GB_FIXED) * GB_SPAN + 40) <= sizeof(GbInputs),
              "a span's staged outputs reuse the stage's inputs");

// A stage is a run of whole consecutive spans whose visible Gaussians fit in GB_SLOTS slots.  Two stages are in flight:
// the one whose adjoint runs and the next one, whose inputs are being gathered.
struct GbShared {
  GbInputs buf[2];
  int gidx[2][GB_SLOTS];                    // Gaussian of each slot
  short slot[2][GB_MAX_SPANS][GB_SPAN];     // slot of each Gaussian of the stage's spans, -1 if culled
  int cnt[GB_THREADS / 32];
};

// The reference's quaternion -> rotation matrix.  Which product of each entry is fused into its sum is written out:
// it is the choice the compiler made for the previous one-block-per-span kernel, and left to the compiler it changes
// with the surrounding code (x*z and r*y are shared by two entries each).  tests/test_gauss_bwd.py holds the
// gradients bit-identical.
__device__ __forceinline__ void rot_from_quat(float r, float x, float y, float z, float R[3][3]) {
  R[0][0] = 1.f - 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z));
  R[0][1] = 2.f * __fmaf_rn(x, y, -__fmul_rn(r, z));
  R[0][2] = 2.f * __fmaf_rn(r, y, __fmul_rn(x, z));
  R[1][0] = 2.f * __fmaf_rn(x, y, __fmul_rn(r, z));
  R[1][1] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(z, z));
  R[1][2] = 2.f * __fmaf_rn(y, z, -__fmul_rn(r, x));
  R[2][0] = 2.f * __fmaf_rn(-r, y, __fmul_rn(x, z));
  R[2][1] = 2.f * __fmaf_rn(y, z, __fmul_rn(r, x));
  R[2][2] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(y, y));
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

// The adjoint chain of one rasterized Gaussian from its blend-adjoint sums A0..A3 and forward record rec1..rec3.
// The expressions and their float/double promotions are the reference's; do not reassociate them.
// NCAM > 0: also the Gaussian's camera terms (cam), the adjoint of the same chain with respect to the camera: the view-space
// point t (dL/dt, with the depth) and W of J(t)·W (dL/dT), the projected centre (the 1/(w + 1e-7) multipliers) and the
// SH view direction (minus the dnormvdv3 result).  Entries the forward does not read (viewmatrix[3,7,11,15],
// projmatrix[2,6,10,14]) stay 0.  NCAM: the number of camera terms formed, 0 (none), GB_CAM_POSE or GB_CAM (the pose
// terms and the focal terms).
template <int NCAM, class SH>
__device__ __forceinline__ void gauss_adjoint(
    int D, float mx, float my, float mz, bool has_scales, float4 q_in, float scx, float scy, float scz,
    float scale_modifier, bool has_sh, unsigned cm, SH sh, const float* cov3D, bool norm_precomp, float4 A0,
    float4 A1, float4 A2, float4 A3, float4 rec1, float4 rec2, float4 rec3, const float* __restrict__ view,
    const float* __restrict__ proj, float h_x, float h_y, float tan_fovx, float tan_fovy, float kernel_size,
    const float* __restrict__ campos, float (&out)[GB_ROW], float (&cam)[GB_CAM]) {
  if constexpr (NCAM > 0) {
#pragma unroll
    for (int j = 0; j < NCAM; j++) cam[j] = 0.f;
  }
  float o_mean2D[3] = {0, 0, 0}, o_conic[4] = {0, 0, 0, 0}, o_opac = 0, o_color[3] = {0, 0, 0}, o_depth = 0;
  float o_mean[3] = {0, 0, 0}, o_cov[6] = {0, 0, 0, 0, 0, 0}, o_norm[3] = {0, 0, 0};
  float o_scale[3] = {0, 0, 0}, o_rot[4] = {0, 0, 0, 0};
  float dsh_scale[16];   // dRGB/dsh_k for k < (D+1)^2, else 0
#pragma unroll
  for (int q = 0; q < 16; q++) dsh_scale[q] = 0.f;
  float dL_dRGB[3] = {0, 0, 0};
  o_color[0] = A0.x; o_color[1] = A0.y; o_color[2] = A0.z; o_depth = A0.w;
  o_norm[0] = A1.x; o_norm[1] = A1.y; o_norm[2] = A1.z;
  o_mean2D[0] = A1.w; o_mean2D[1] = A2.x; o_mean2D[2] = A2.y;
  o_conic[0] = A2.z; o_conic[1] = A2.w; o_conic[3] = A3.x;
  o_opac = A3.y;

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
    if constexpr (NCAM > 0) {
      // t = [m, 1]·view (columns 0..2): dL/dview[4k + r] = m_k dL/dt_r, dL/dview[12 + r] = dL/dt_r.  T = J·W with
      // W[k][r] = view[4r + k] and J = [[a0, 0, a2], [0, b1, b2]]: dL/dW[k][r] = sum_i J[i][k] dL/dT[i][r].
      const float m3[3] = {mx, my, mz};
      const float dt[3] = {dL_dtx, dL_dty, dL_dtz};
      const float dT0[3] = {dL_dT00, dL_dT01, dL_dT02}, dT1[3] = {dL_dT10, dL_dT11, dL_dT12};
#pragma unroll
      for (int r = 0; r < 3; r++) {
#pragma unroll
        for (int k = 0; k < 3; k++) cam[C_VIEW + 4 * k + r] = m3[k] * dt[r];
        cam[C_VIEW + 12 + r] = dt[r];
      }
#pragma unroll
      for (int r = 0; r < 3; r++) {
        cam[C_VIEW + 4 * r + 0] += a0 * dT0[r];
        cam[C_VIEW + 4 * r + 1] += b1 * dT1[r];
        cam[C_VIEW + 4 * r + 2] += a2 * dT0[r] + b2 * dT1[r];
      }
    }
    if constexpr (NCAM > C_TANY) {
      // The focal terms.  h = W / (2 tan) enters J00 = h_x / tz and J02 = -h_x tx / tz^2 (tx the clamped t_x), so
      // dL/dh_x = dL/dJ00 / tz - dL/dJ02 tx / tz^2 and dh_x/dtan_fovx = -h_x / tan_fovx.  A clamped t_x is
      // ±1.3 tan_fovx · tz: J02 then also moves with the bound, by ∓1.3 h_x / tz.  Likewise y with h_y, J11, J12.
      // In double, from the float values the chain already holds: new uses of its float products could change the
      // compiler's fusion of them into the gradient sums.
      const double z = tz, zi = 1.0 / z, hx = h_x, hy = h_y;
      const double dJ02 = dL_dJ02, dJ12 = dL_dJ12;
      double gtx = -(hx / (double)tan_fovx) * (((double)dL_dJ00 - dJ02 * (double)tx * zi) * zi);
      double gty = -(hy / (double)tan_fovy) * (((double)dL_dJ11 - dJ12 * (double)ty * zi) * zi);
      if (txtz < -limx || txtz > limx) gtx += dJ02 * ((txtz > 0.f ? -1.3 : 1.3) * hx * zi);
      if (tytz < -limy || tytz > limy) gty += dJ12 * ((tytz > 0.f ? -1.3 : 1.3) * hy * zi);
      cam[C_TANX] = (float)gtx;
      cam[C_TANY] = (float)gty;
    }
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
    if constexpr (NCAM > 0) {
      // the homogeneous centre [m, 1]·proj and its divide: dL/dhom = (gx w, gy w, ., -(gx mul1 + gy mul2)), w = m_w;
      // the depth is t_z: dL/dview[4k + 2] = m_k dL/ddepth, dL/dview[14] = dL/ddepth
      const float m3[3] = {mx, my, mz};
      const float dhx = gx * m_w, dhy = gy * m_w, dhw = -(gx * mul1 + gy * mul2);
#pragma unroll
      for (int k = 0; k < 3; k++) {
        cam[C_PROJ + 4 * k + 0] = m3[k] * dhx;
        cam[C_PROJ + 4 * k + 1] = m3[k] * dhy;
        cam[C_PROJ + 4 * k + 3] = m3[k] * dhw;
        cam[C_VIEW + 4 * k + 2] += m3[k] * o_depth;
      }
      cam[C_PROJ + 12] = dhx;
      cam[C_PROJ + 13] = dhy;
      cam[C_PROJ + 15] = dhw;
      cam[C_VIEW + 14] += o_depth;
    }
  }

  // ---------------- RGB -> SH and view direction -> mean ----------------
  if (has_sh) {
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
      if constexpr (NCAM > 0) {
        // -dnormvdv3(v, dL_ddir), evaluated again in double: reading dm here would give its final products a second
        // use, and the compiler would then no longer fuse them into the o_mean sums, changing dL_dmean3D's rounding
        const double vx = ox, vy = oy, vz = oz, gx = dL_ddir.x, gy = dL_ddir.y, gz = dL_ddir.z;
        const double s2 = vx * vx + vy * vy + vz * vz, inv = 1.0 / (s2 * sqrt(s2));
        cam[C_CAMPOS + 0] = (float)(-((s2 - vx * vx) * gx - vy * vx * gy - vz * vx * gz) * inv);
        cam[C_CAMPOS + 1] = (float)(-(-vx * vy * gx + (s2 - vy * vy) * gy - vz * vy * gz) * inv);
        cam[C_CAMPOS + 2] = (float)(-(-vx * vz * gx - vy * vz * gy + (s2 - vz * vz) * gz) * inv);
      }
    };
    sh_adjoint(sh);
  }

  // ---------------- cov3D -> scale / rotation, normal -> rotation ----------------
  if (has_scales) {
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

    if (!norm_precomp) {
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

#pragma unroll
  for (int c = 0; c < 3; c++) {
    out[O_MEAN2D + c] = o_mean2D[c]; out[O_COLOR + c] = o_color[c]; out[O_MEAN3D + c] = o_mean[c];
    out[O_NORM + c] = o_norm[c]; out[O_SCALE + c] = o_scale[c]; out[O_RGB + c] = dL_dRGB[c];
  }
#pragma unroll
  for (int c = 0; c < 4; c++) { out[O_CONIC + c] = o_conic[c]; out[O_ROT + c] = o_rot[c]; }
#pragma unroll
  for (int c = 0; c < 6; c++) out[O_COV + c] = o_cov[c];
#pragma unroll
  for (int q = 0; q < 16; q++) out[O_SHF + q] = dsh_scale[q];
  out[O_OPAC] = o_opac;
  out[O_DEPTH] = o_depth;
}

// Writes the span's contiguous range dst[base*w, (base+n)*w) once, with the whole CTA: 16-byte stores for the aligned
// middle, scalar stores for the head and tail that the caller's pointer leaves unaligned (phase-2 ranges start at
// any Gaussian).  val(g, c) is element c of span Gaussian g's row.
template <class F>
__device__ __forceinline__ void emit_rows(float* __restrict__ dst, int base, int n, int w, F val) {
  float* d = dst + (size_t)base * w;
  const int nfl = n * w;
  const int head = min(nfl, (int)(((16u - ((unsigned)reinterpret_cast<uintptr_t>(d) & 15u)) & 15u) >> 2));
  const int nv4 = (nfl - head) >> 2;
  float4* d4 = reinterpret_cast<float4*>(d + head);
  // (g, c) of this thread's first element, advanced by the 4 * GB_THREADS floats of each step without a division
  int g = (head + 4 * (int)threadIdx.x) / w, c = head + 4 * (int)threadIdx.x - g * w;
  const int dg = 4 * GB_THREADS / w, dc = 4 * GB_THREADS - dg * w;
#pragma unroll 4
  for (int q = threadIdx.x; q < nv4; q += GB_THREADS) {
    int gg = g, cc = c;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      v[j] = val(gg, cc);
      if (++cc == w) { cc = 0; ++gg; }
    }
    d4[q] = make_float4(v[0], v[1], v[2], v[3]);
    g += dg;
    c += dc;
    if (c >= w) { c -= w; ++g; }
  }
  const int tail0 = head + 4 * nv4, nscalar = head + (nfl - tail0);
  for (int r = threadIdx.x; r < nscalar; r += GB_THREADS) {
    const int e = r < head ? r : tail0 + (r - head);
    const int g = e / w;
    d[e] = val(g, e - g * w);
  }
}

// Writes dst[0, nfl) from a staged image whose element e sits at src[e] and whose 16-byte units line up with dst's:
// 16-byte copies for the aligned middle, scalar ones for the head and tail.
__device__ __forceinline__ void copy_range(float* __restrict__ dst, const float* src, int nfl) {
  const int head = min(nfl, (int)(((16u - ((unsigned)reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u) >> 2));
  const int nv4 = (nfl - head) >> 2;
  const float4* s4 = reinterpret_cast<const float4*>(src + head);
  float4* d4 = reinterpret_cast<float4*>(dst + head);
  for (int q = threadIdx.x; q < nv4; q += GB_THREADS) d4[q] = s4[q];
  const int tail0 = head + 4 * nv4, nscalar = head + (nfl - tail0);
  for (int r = threadIdx.x; r < nscalar; r += GB_THREADS) {
    const int e = r < head ? r : tail0 + (r - head);
    dst[e] = src[e];
  }
}

// The camera terms of a stage's slots are staged, field-major, after the span's staged outputs in the consumed inputs.
constexpr int GB_CAM_STAGE = (GB_SPAN * (GB_SH_ROW + GB_FIXED) + 4 * GB_NFIXED + 3) & ~3;
static_assert(sizeof(float) * (GB_CAM_STAGE + GB_CAM * GB_SLOTS) <= sizeof(GbInputs),
              "a stage's camera terms fit beside a span's staged outputs");

// The per-Gaussian adjoint over spans [g_begin, g_end).  NCAM > 0: also the first NCAM camera terms; span s (counted
// from g_begin) writes cam_part[j * nspans + s], the float64 sum of its rasterized Gaussians' camera term j in index
// order.
template <int NCAM>
__device__ __forceinline__ void
gauss_bwd_body(int g_begin, int g_end, int spans_per_cta, int acc_row0, int D, int M,
               const float* __restrict__ means3D, const int* __restrict__ radii, const float* __restrict__ shs,
               const unsigned char* __restrict__ clamped, const float* __restrict__ scales,
               const float* __restrict__ rotations, float scale_modifier, const float* __restrict__ cov3Ds,
               const float* __restrict__ rec, const float* __restrict__ norm3D_precomp,
               const float* __restrict__ view, const float* __restrict__ proj, float h_x, float h_y,
               float tan_fovx, float tan_fovy, float kernel_size, const float* __restrict__ campos,
               const float* __restrict__ acc, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic,
               float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor, float* __restrict__ dL_ddepth,
               float* __restrict__ dL_dmean3D, float* __restrict__ dL_dcov3D, float* __restrict__ dL_dnorm3D,
               float* __restrict__ dL_dsh, float* __restrict__ dL_dscale, float* __restrict__ dL_drot,
               double* __restrict__ cam_part) {
  extern __shared__ __align__(16) unsigned char gb_smem[];
  GbShared& S = *reinterpret_cast<GbShared*>(gb_smem);
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int nspans = (g_end - g_begin + GB_SPAN - 1) / GB_SPAN;
  const int span_end = min(nspans, (blockIdx.x + 1) * spans_per_cta);
  int next = blockIdx.x * spans_per_cta;             // first span not yet in a stage
  if (next >= span_end) return;
  const int Dc = min(max(D, 0), 3);
  const int nsh = (Dc + 1) * (Dc + 1) * 3;          // SH floats the adjoint reads per Gaussian
  const int nq = (nsh + 3) >> 2;                    // ... as 16-byte units when the rows allow it
  const bool sh_vec = ((3 * M) & 3) == 0 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0;
  const bool has_sh = shs != nullptr, has_scales = scales != nullptr;
  float* const fixed_out[GB_NFIXED] = {dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_ddepth,
                                       dL_dmean3D, dL_dcov3D, dL_dnorm3D, dL_dscale, dL_drot};
  // their widths, offsets in the adjoint's outputs and offsets of their staged images (a span's range plus up to 3
  // floats of shift, rounded to 16 bytes)
  constexpr int kFixedW[GB_NFIXED] = {3, 4, 1, 3, 1, 3, 6, 3, 3, 4};
  constexpr int kFixedO[GB_NFIXED] = {O_MEAN2D, O_CONIC, O_OPAC, O_COLOR, O_DEPTH, O_MEAN3D, O_COV, O_NORM, O_SCALE, O_ROT};
  constexpr int I = GB_SPAN, kImageOff[GB_NFIXED] = {0,            3 * I + 4,     7 * I + 8,     8 * I + 12,
                                                     11 * I + 16,  12 * I + 20,   15 * I + 24,   21 * I + 28,
                                                     24 * I + 32,  27 * I + 36};
  static_assert(kImageOff[9] + GB_SPAN * kFixedW[9] + 4 == GB_SPAN * GB_FIXED + 4 * GB_NFIXED, "image offsets");

  // radius of this thread's Gaussian in the next four spans, loaded well before the compaction needs it
  auto radius = [&](int s) {
    const int base = g_begin + s * GB_SPAN;
    return s < span_end && t < GB_SPAN && t < g_end - base ? radii[base + t] : 0;
  };
  int rq[4];
#pragma unroll
  for (int j = 0; j < 4; j++) rq[j] = radius(next + j);

  // Fills stage b with whole spans from `next` on and issues the gather of its slots' inputs.  Starts with a
  // barrier, which also publishes the copies of the stage before.  Returns the stage's span count and slot count.
  auto prepare = [&](int b, int& nsp, int& nslots) {
    nsp = 0;
    nslots = 0;
    while (nsp < GB_MAX_SPANS && next < span_end) {
      const bool vis = rq[0] > 0;
      const unsigned bal = __ballot_sync(0xffffffffu, vis);
      if (lane == 0) S.cnt[wid] = __popc(bal);
      __syncthreads();
      int off = 0, nv = 0;
#pragma unroll
      for (int q = 0; q < GB_THREADS / 32; q++) { off += q < wid ? S.cnt[q] : 0; nv += S.cnt[q]; }
      __syncthreads();
      if (nslots + nv > GB_SLOTS) break;
      const int k = vis ? nslots + off + __popc(bal & ((1u << lane) - 1u)) : -1;
      if (t < GB_SPAN) S.slot[b][nsp][t] = (short)k;
      if (vis) S.gidx[b][k] = g_begin + next * GB_SPAN + t;
      nslots += nv;
      ++nsp;
      ++next;
      rq[0] = rq[1]; rq[1] = rq[2]; rq[2] = rq[3]; rq[3] = radius(next + 3);
    }
    __syncthreads();
    const int* gidx = S.gidx[b];
    GbInputs& in = S.buf[b];
    for (int u = t; u < nslots * 4; u += GB_THREADS) {
      const int k = u >> 2, q = u & 3;
      cp_async16(&in.acc[q][k], acc + (size_t)(gidx[k] - acc_row0) * 16 + 4 * q);
    }
    for (int u = t; u < nslots * 3; u += GB_THREADS) {
      const int k = u / 3, q = u - 3 * k;
      const size_t i = (size_t)gidx[k];
      cp_async16(&in.rec[q][k], rec + i * REC_FLOATS + 4 + 4 * q);
      cp_async4(&in.mean[q][k], means3D + 3 * i + q);
      if (has_scales) cp_async4(&in.scale[q][k], scales + 3 * i + q);
    }
    for (int u = t; u < nslots * 6; u += GB_THREADS) {
      const int k = u / 6, q = u - 6 * k;
      cp_async4(&in.cov[q][k], cov3Ds + 6 * (size_t)gidx[k] + q);
    }
    for (int k = t; k < nslots; k += GB_THREADS) {
      const int idx = gidx[k];
      if (has_scales) cp_async16(&in.rot[k], rotations + 4 * (size_t)idx);
      if (has_sh) cp_async4(&in.clamped[k], clamped + (idx & ~3));
    }
    if (has_sh) {
      // 16 (64) lanes per slot: a power of two, so the slot and the unit are a shift and a mask
      if (sh_vec) {
        for (int u = t; u < nslots * 16; u += GB_THREADS) {
          const int k = u >> 4, q = u & 15;
          if (q < nq) cp_async16(&in.sh[q][k], shs + (size_t)gidx[k] * 3 * M + 4 * q);
        }
      } else {
        for (int u = t; u < nslots * 64; u += GB_THREADS) {
          const int k = u >> 6, j = u & 63;
          if (j < nsh) cp_async4(reinterpret_cast<float*>(&in.sh[j >> 2][k]) + (j & 3), shs + (size_t)gidx[k] * 3 * M + j);
        }
      }
    }
    cp_async_commit();
  };

  int first_cur = next, nsp_cur, nslots_cur;
  prepare(0, nsp_cur, nslots_cur);
  for (int b = 0;; b ^= 1) {
    cp_async_wait_all();   // this thread's copies of stage b have landed
    const bool more = next < span_end;
    const int first_next = next;
    int nsp_next = 0, nslots_next = 0;
    if (more) prepare(b ^ 1, nsp_next, nslots_next);
    else __syncthreads();

    // ---------------- adjoint: thread k takes slot k ----------------
    GbInputs& in = S.buf[b];
    float o[GB_ROW];
    float cam[GB_CAM];
    const bool active = t < nslots_cur;
    if (active) {
      const int k = t;
      const float* shk = reinterpret_cast<const float*>(&in.sh[0][k]);   // float j at word (j >> 2) * 4 * SLOTS + (j & 3)
      const float cov3D[6] = {in.cov[0][k], in.cov[1][k], in.cov[2][k], in.cov[3][k], in.cov[4][k], in.cov[5][k]};
      const unsigned cm = has_sh ? (in.clamped[k] >> (8 * (S.gidx[b][k] & 3))) & 0xffu : 0u;
      gauss_adjoint<NCAM>(D, in.mean[0][k], in.mean[1][k], in.mean[2][k], has_scales,
                    has_scales ? in.rot[k] : make_float4(0.f, 0.f, 0.f, 0.f),
                    has_scales ? in.scale[0][k] : 0.f, has_scales ? in.scale[1][k] : 0.f,
                    has_scales ? in.scale[2][k] : 0.f, scale_modifier, has_sh, cm,
                    [&](int j) { return shk[(j >> 2) * (4 * GB_SLOTS) + (j & 3)]; }, cov3D,
                    norm3D_precomp != nullptr, in.acc[0][k], in.acc[1][k], in.acc[2][k], in.acc[3][k],
                    in.rec[0][k], in.rec[1][k], in.rec[2][k], view, proj, h_x, h_y, tan_fovx, tan_fovy,
                    kernel_size, campos, o, cam);
    }
    // ---------------- epilogue, span by span: stage the span's outputs, then write each output's range once ----------
    // Staged over the consumed inputs: the dL_dsh factor rows, then one image per fixed-width array laid out as its
    // range in global memory (shifted by `pre` floats so that its 16-byte units line up with the destination's).
    // The fixed-width arrays are then plain copies; dL_dsh is formed while it is written, for any M.
    float* const sh_rows = reinterpret_cast<float*>(&S.buf[b]);
    float* const images = sh_rows + GB_SPAN * GB_SH_ROW;
    float* const cam_stage = sh_rows + GB_CAM_STAGE;
    const int rel = active ? S.gidx[b][t] - (g_begin + first_cur * GB_SPAN) : -1;   // span * GB_SPAN + position
    for (int sp = 0; sp < nsp_cur; sp++) {
      const int base = g_begin + (first_cur + sp) * GB_SPAN, n = min(GB_SPAN, g_end - base);
      int pre[GB_NFIXED];
#pragma unroll
      for (int x = 0; x < GB_NFIXED; x++)
        pre[x] = (int)((reinterpret_cast<uintptr_t>(fixed_out[x] + (size_t)base * kFixedW[x]) >> 2) & 3u);
      __syncthreads();   // every read of the inputs (sp == 0) or of the previous span's staged outputs is done
      // thread t stages the outputs of its slot's Gaussian if that lies in this span, and zeros for position t of the
      // span if that Gaussian was culled
      auto stage = [&](int g, bool z) {
#pragma unroll
        for (int j = 0; j < GB_SH_ROW; j++) sh_rows[g * GB_SH_ROW + j] = z ? 0.f : o[O_SHF + j];
#pragma unroll
        for (int x = 0; x < GB_NFIXED; x++) {
          float* im = images + kImageOff[x] + pre[x] + g * kFixedW[x];
#pragma unroll
          for (int c = 0; c < kFixedW[x]; c++) im[c] = z ? 0.f : o[kFixedO[x] + c];
        }
      };
      if (active && rel / GB_SPAN == sp) stage(rel % GB_SPAN, false);
      if (t < n && S.slot[b][sp][t] < 0) stage(t, true);
      if constexpr (NCAM > 0) {
        if (sp == 0 && active) {
#pragma unroll
          for (int j = 0; j < NCAM; j++) cam_stage[j * GB_SLOTS + t] = cam[j];
        }
      }
      __syncthreads();
      if constexpr (NCAM > 0) {
        // thread j sums term j over the span's Gaussians in index order
        if (t < NCAM) {
          double s = 0.0;
          for (int p = 0; p < n; p++) {
            const int k = S.slot[b][sp][p];
            if (k >= 0) s += (double)cam_stage[t * GB_SLOTS + k];
          }
          cam_part[(size_t)t * nspans + first_cur + sp] = s;
        }
      }
#pragma unroll
      for (int x = 0; x < GB_NFIXED; x++)
        copy_range(fixed_out[x] + (size_t)base * kFixedW[x], images + kImageOff[x] + pre[x], n * kFixedW[x]);
      if (dL_dsh != nullptr) {
        // dL_dsh[g][k][ch] = dRGB/dsh_k(g) * dL_dRGB[ch](g); coefficients k >= 16 have no factor and give 0 * dL_dRGB
        emit_rows(dL_dsh, base, n, 3 * M, [=](int g, int c) {
          const int kk = c / 3, ch = c - 3 * kk;
          const float* row = sh_rows + g * GB_SH_ROW;
          const float f = row[min(kk, 15)];
          return (kk < 16 ? f : 0.f) * row[16 + ch];
        });
      }
    }
    if (!more) break;
    first_cur = first_next;
    nsp_cur = nsp_next;
    nslots_cur = nslots_next;
  }
}

#define GB_PARAMS                                                                                                    \
  int g_begin, int g_end, int spans_per_cta, int acc_row0, int D, int M, const float* __restrict__ means3D,         \
      const int* __restrict__ radii, const float* __restrict__ shs, const unsigned char* __restrict__ clamped,      \
      const float* __restrict__ scales, const float* __restrict__ rotations, float scale_modifier,                  \
      const float* __restrict__ cov3Ds, const float* __restrict__ rec, const float* __restrict__ norm3D_precomp,    \
      const float* __restrict__ view, const float* __restrict__ proj, float h_x, float h_y, float tan_fovx,         \
      float tan_fovy, float kernel_size, const float* __restrict__ campos, const float* __restrict__ acc,           \
      float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity,               \
      float* __restrict__ dL_dcolor, float* __restrict__ dL_ddepth, float* __restrict__ dL_dmean3D,                 \
      float* __restrict__ dL_dcov3D, float* __restrict__ dL_dnorm3D, float* __restrict__ dL_dsh,                    \
      float* __restrict__ dL_dscale, float* __restrict__ dL_drot
#define GB_ARGS                                                                                                      \
  g_begin, g_end, spans_per_cta, acc_row0, D, M, means3D, radii, shs, clamped, scales, rotations, scale_modifier,   \
      cov3Ds, rec, norm3D_precomp, view, proj, h_x, h_y, tan_fovx, tan_fovy, kernel_size, campos, acc, dL_dmean2D,  \
      dL_dconic, dL_dopacity, dL_dcolor, dL_ddepth, dL_dmean3D, dL_dcov3D, dL_dnorm3D, dL_dsh, dL_dscale, dL_drot

__global__ void __launch_bounds__(GB_THREADS, GB_CTAS_PER_SM) gauss_bwd_kernel(GB_PARAMS) {
  gauss_bwd_body<0>(GB_ARGS, nullptr);
}

__global__ void __launch_bounds__(GB_THREADS, GB_CTAS_PER_SM)
gauss_bwd_camera_kernel(GB_PARAMS, double* __restrict__ cam_part) {
  gauss_bwd_body<GB_CAM_POSE>(GB_ARGS, cam_part);
}

// the pose terms and the focal terms: a kernel of its own, so that the pose-only camera backward keeps its code
__global__ void __launch_bounds__(GB_THREADS, GB_CTAS_PER_SM)
gauss_bwd_intrinsics_kernel(GB_PARAMS, double* __restrict__ cam_part) {
  gauss_bwd_body<GB_CAM>(GB_ARGS, cam_part);
}

#undef GB_PARAMS
#undef GB_ARGS

// dL_dcamera[j] = the sum of the spans' partials of term j, rounded to float once.  The order depends on nspans only:
// thread i adds spans i, i + CR_THREADS, ... in turn, then a fixed tree adds the threads' sums.
constexpr int CR_THREADS = 256;
// the sum of term blockIdx.x over the spans, in that order, valid in thread 0
__device__ __forceinline__ double camera_span_sum(int nspans, const double* __restrict__ cam_part) {
  __shared__ double s[CR_THREADS];
  const int j = blockIdx.x, t = threadIdx.x;
  const double* p = cam_part + (size_t)j * nspans;
  double v = 0.0;
  for (int i = t; i < nspans; i += CR_THREADS) v += p[i];
  s[t] = v;
  __syncthreads();
#pragma unroll
  for (int w = CR_THREADS / 2; w > 0; w >>= 1) {
    if (t < w) s[t] += s[t + w];
    __syncthreads();
  }
  return s[0];
}

__global__ void __launch_bounds__(CR_THREADS)
camera_reduce_kernel(int nspans, const double* __restrict__ cam_part, float* __restrict__ dL_dcamera) {
  const int j = blockIdx.x, t = threadIdx.x;
  const double s = camera_span_sum(nspans, cam_part);
  if (t == 0) dL_dcamera[j] = (float)s;
}

// The same sum over the spans of a phase-2 Gaussian slice, left unrounded: the ranks of a sharded frame add their
// slices' float64 partials and round once.
__global__ void __launch_bounds__(CR_THREADS)
camera_partial_reduce_kernel(int nspans, const double* __restrict__ cam_part, double* __restrict__ dL_dcamera) {
  const int j = blockIdx.x, t = threadIdx.x;
  const double s = camera_span_sum(nspans, cam_part);
  if (t == 0) dL_dcamera[j] = s;
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

// ncam: the number of camera terms, 35 (pose) or 37 (pose and focal)
size_t sfgs_camera_scratch_bytes(int P, int ncam) {
  return sfgs_align_up((size_t)ncam * ((P + GB_SPAN - 1) / GB_SPAN) * sizeof(double));
}

void sfgs_launch_camera_reduce(int P, int ncam, const double* cam_part, float* dL_dcamera, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  camera_reduce_kernel<<<ncam, CR_THREADS, 0, st>>>((P + GB_SPAN - 1) / GB_SPAN, cam_part, dL_dcamera);
}

// n: the length of the Gaussian slice whose span partials cam_part holds (the order of the sum depends on it alone)
void sfgs_launch_camera_partial_reduce(int n, int ncam, const double* cam_part, double* dL_dcamera, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  camera_partial_reduce_kernel<<<ncam, CR_THREADS, 0, st>>>((n + GB_SPAN - 1) / GB_SPAN, cam_part, dL_dcamera);
}

// cam_part: NULL for the adjoint alone; else [ncam][spans] doubles (sfgs_camera_scratch_bytes) that receive every
// span's camera partials, ncam = 35 (pose terms) or 37 (pose and focal terms)
void sfgs_launch_gauss_bwd(const sfgs_backward_args* a, const GeomLayout& g, float focal_x, float focal_y,
                           const float* acc, int g_begin, int g_end, int acc_row0, double* cam_part, int ncam,
                           cudaStream_t st) {
  if (g_end <= g_begin) return;
  static SfgsPerDeviceOnce attr_once;
  if (attr_once.first_use()) {
    cudaFuncSetAttribute(gauss_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GbShared));
    cudaFuncSetAttribute(gauss_bwd_camera_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GbShared));
    cudaFuncSetAttribute(gauss_bwd_intrinsics_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GbShared));
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  { int v = 0; if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) sms = v; }
  // each CTA takes an equal share of consecutive spans, so that a stage can gather whole runs of them
  const int nspans = (g_end - g_begin + GB_SPAN - 1) / GB_SPAN;
  const int ctas = nspans < GB_CTAS_PER_SM * sms ? nspans : GB_CTAS_PER_SM * sms;
  const int spans_per_cta = (nspans + ctas - 1) / ctas;
  const int blocks = (nspans + spans_per_cta - 1) / spans_per_cta;
  const float* cov3D_ptr = a->cov3D_precomp != nullptr ? a->cov3D_precomp : g.cov3D;
  float* dL_dsh = a->M > 0 ? a->dL_dsh : nullptr;
  SFGS_COUNT_LAUNCH();
#define GB_LAUNCH_ARGS                                                                                               \
  g_begin, g_end, spans_per_cta, acc_row0, a->D, a->M, a->means3D, a->radii, a->shs, g.clamped, a->scales,          \
      a->rotations, a->scale_modifier, cov3D_ptr, g.rec, a->norm3D_precomp, a->viewmatrix, a->projmatrix, focal_x,  \
      focal_y, a->tan_fovx, a->tan_fovy, a->kernel_size, a->cam_pos, acc, a->dL_dmean2D, a->dL_dconic,              \
      a->dL_dopacity, a->dL_dcolor, a->dL_ddepth, a->dL_dmean3D, a->dL_dcov3D, a->dL_dnorm3D, dL_dsh, a->dL_dscale, \
      a->dL_drot
  if (cam_part != nullptr && ncam == GB_CAM)
    gauss_bwd_intrinsics_kernel<<<blocks, GB_THREADS, sizeof(GbShared), st>>>(GB_LAUNCH_ARGS, cam_part);
  else if (cam_part != nullptr)
    gauss_bwd_camera_kernel<<<blocks, GB_THREADS, sizeof(GbShared), st>>>(GB_LAUNCH_ARGS, cam_part);
  else
    gauss_bwd_kernel<<<blocks, GB_THREADS, sizeof(GbShared), st>>>(GB_LAUNCH_ARGS);
#undef GB_LAUNCH_ARGS
}
