// sfgs_preprocess.cu — per-Gaussian projection stage (forward).
//
// Replaces FORWARD::preprocess / preprocessCUDA (RAST/cuda_rasterizer/forward.cu:214-328),
// checkFrustum (RAST/cuda_rasterizer/rasterizer_impl.cu:54-66) and the
// tile-instance counting that the reference obtains from its prefix sum
// (rasterizer_impl.cu:283).  One thread per Gaussian; the result is one packed
// 64-byte blend record per Gaussian plus a per-tile instance histogram.
//
// The arithmetic that decides tile/key indexing (view depth, projected centre,
// 2D covariance, radius, tile rectangle) is written with the same operand
// order and the same float/double promotions as the reference so that the
// compiler contracts it into the same FMA sequence: radii, tiles_touched and
// the depth bits of the sort key must be bit-identical.
#include "sfgs_common.cuh"

namespace {

__device__ __forceinline__ float ndc_to_pix(float v, int S) {
  // double arithmetic, as auxiliary.h:42-45 (its literals are doubles)
  return ((v + 1.0) * S - 1.0) * 0.5;
}

struct Sym3 { float c0, c1, c2, c3, c4, c5; };

// 3D covariance from scale * modifier and the (un-normalised) quaternion.
// M = S * R (column-major glm semantics), Sigma = M^T M, upper triangle.
// Mirrors computeCov3D, forward.cu:129-163.
__device__ __forceinline__ void rot_from_quat(float r, float x, float y, float z, float R[3][3]) {
  // R[c][k]: column c, row k, same element order as the glm::mat3 constructor call.
  // The products below are pinned with explicit round-to-nearest intrinsics to the exact
  // mul / fma split the reference's compiled binary uses for this block (read off its SASS:
  // xy, yz and ry are fused into the add, rz, rx and xz are rounded products), because
  // cov3D feeds the radius and therefore the tile/key indexing that must match bit for bit.
  const float yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
  const float rz = __fmul_rn(r, z), rx = __fmul_rn(r, x), xz = __fmul_rn(x, z);
  const float s_yz = __fadd_rn(yy, zz);
  const float s_xz = __fmaf_rn(x, x, zz);
  const float s_xy = __fmaf_rn(x, x, yy);
  const float xy_m_rz = __fmaf_rn(x, y, -rz), xy_p_rz = __fmaf_rn(x, y, rz);
  const float xz_p_ry = __fmaf_rn(r, y, xz), xz_m_ry = __fmaf_rn(-r, y, xz);
  const float yz_m_rx = __fmaf_rn(y, z, -rx), yz_p_rx = __fmaf_rn(y, z, rx);
  R[0][0] = __fsub_rn(1.f, __fadd_rn(s_yz, s_yz)); R[0][1] = __fadd_rn(xy_m_rz, xy_m_rz); R[0][2] = __fadd_rn(xz_p_ry, xz_p_ry);
  R[1][0] = __fadd_rn(xy_p_rz, xy_p_rz); R[1][1] = __fsub_rn(1.f, __fadd_rn(s_xz, s_xz)); R[1][2] = __fadd_rn(yz_m_rx, yz_m_rx);
  R[2][0] = __fadd_rn(xz_m_ry, xz_m_ry); R[2][1] = __fadd_rn(yz_p_rx, yz_p_rx); R[2][2] = __fsub_rn(1.f, __fadd_rn(s_xy, s_xy));
}

__device__ __forceinline__ Sym3 cov3d_from_scale_rot(float sx, float sy, float sz, float mod,
                                                     float qr, float qx, float qy, float qz) {
  float R[3][3];
  rot_from_quat(qr, qx, qy, qz, R);
  const float s0 = mod * sx, s1 = mod * sy, s2 = mod * sz;
  float M[3][3];
#pragma unroll
  for (int c = 0; c < 3; c++) { M[c][0] = s0 * R[c][0]; M[c][1] = s1 * R[c][1]; M[c][2] = s2 * R[c][2]; }
  // Sigma[c][r] = M[r][0]*M[c][0] + M[r][1]*M[c][1] + M[r][2]*M[c][2]
  Sym3 S;
  S.c0 = M[0][0] * M[0][0] + M[0][1] * M[0][1] + M[0][2] * M[0][2];
  S.c1 = M[1][0] * M[0][0] + M[1][1] * M[0][1] + M[1][2] * M[0][2];
  S.c2 = M[2][0] * M[0][0] + M[2][1] * M[0][1] + M[2][2] * M[0][2];
  S.c3 = M[1][0] * M[1][0] + M[1][1] * M[1][1] + M[1][2] * M[1][2];
  S.c4 = M[2][0] * M[1][0] + M[2][1] * M[1][1] + M[2][2] * M[1][2];
  S.c5 = M[2][0] * M[2][0] + M[2][1] * M[2][1] + M[2][2] * M[2][2];
  return S;
}

// Shortest-axis normal, flipped toward the camera.  Mirrors computeNorm3D, forward.cu:167-211.
__device__ __forceinline__ void normal_from_scale_rot(float sx, float sy, float sz,
                                                      float qr, float qx, float qy, float qz,
                                                      float px, float py, float pz,
                                                      float cx, float cy, float cz, float n[3]) {
  float R[3][3];
  rot_from_quat(qr, qx, qy, qz, R);
  float a0, a1, a2;
  if (sx > sz && sy > sz) { a0 = 0.f; a1 = 0.f; a2 = 1.f; }
  else if (sx > sy && sz > sy) { a0 = 0.f; a1 = 1.f; a2 = 0.f; }
  else { a0 = 1.f; a1 = 0.f; a2 = 0.f; }
  // transpose(R) * axis : out[r] = Rt[0][r]*a0 + Rt[1][r]*a1 + Rt[2][r]*a2, Rt[c][r] = R[r][c]
  float n0 = R[0][0] * a0 + R[0][1] * a1 + R[0][2] * a2;
  float n1 = R[1][0] * a0 + R[1][1] * a1 + R[1][2] * a2;
  float n2 = R[2][0] * a0 + R[2][1] * a1 + R[2][2] * a2;
  const float dx = px - cx, dy = py - cy, dz = pz - cz;
  const float d = dx * n0 + dy * n1 + dz * n2;
  if (d > 0) { n0 = -n0; n1 = -n1; n2 = -n2; }
  n[0] = n0; n[1] = n1; n[2] = n2;
}

// EWA projection of the 3D covariance + Mip-Splatting 2D filter.
// Mirrors computeCov2D, forward.cu:74-124. Returns (cov00+k, cov01, cov11+k, coef).
__device__ __forceinline__ float4 cov2d_project(float mx, float my, float mz,
                                                float focal_x, float focal_y,
                                                float tan_fovx, float tan_fovy, float kernel_size,
                                                const Sym3& V, const float* __restrict__ vm) {
  float tx = vm[0] * mx + vm[4] * my + vm[8] * mz + vm[12];
  float ty = vm[1] * mx + vm[5] * my + vm[9] * mz + vm[13];
  const float tz = vm[2] * mx + vm[6] * my + vm[10] * mz + vm[14];
  const float limx = 1.3f * tan_fovx;
  const float limy = 1.3f * tan_fovy;
  const float txtz = tx / tz;
  const float tytz = ty / tz;
  tx = min(limx, max(-limx, txtz)) * tz;
  ty = min(limy, max(-limy, tytz)) * tz;

  // J columns: (a0, 0, a2), (0, b1, b2), 0
  const float a0 = focal_x / tz;
  const float a2 = -(focal_x * tx) / (tz * tz);
  const float b1 = focal_y / tz;
  const float b2 = -(focal_y * ty) / (tz * tz);
  // W columns: (vm0,vm4,vm8), (vm1,vm5,vm9), (vm2,vm6,vm10); T = W * J
  float T0[3], T1[3];
  T0[0] = vm[0] * a0 + vm[1] * 0.0f + vm[2] * a2;
  T0[1] = vm[4] * a0 + vm[5] * 0.0f + vm[6] * a2;
  T0[2] = vm[8] * a0 + vm[9] * 0.0f + vm[10] * a2;
  T1[0] = vm[0] * 0.0f + vm[1] * b1 + vm[2] * b2;
  T1[1] = vm[4] * 0.0f + vm[5] * b1 + vm[6] * b2;
  T1[2] = vm[8] * 0.0f + vm[9] * b1 + vm[10] * b2;
  // X = T^T * V^T : X[c][r] = T[r][0]*V[0][c] + T[r][1]*V[1][c] + T[r][2]*V[2][c]   (r = 0,1)
  const float V0[3] = {V.c0, V.c1, V.c2}, V1[3] = {V.c1, V.c3, V.c4}, V2[3] = {V.c2, V.c4, V.c5};
  float X0[3], X1[3];   // X0[c] = X[c][0], X1[c] = X[c][1]
#pragma unroll
  for (int c = 0; c < 3; c++) {
    X0[c] = T0[0] * V0[c] + T0[1] * V1[c] + T0[2] * V2[c];
    X1[c] = T1[0] * V0[c] + T1[1] * V1[c] + T1[2] * V2[c];
  }
  // cov[c][r] = X[0][r]*T[c][0] + X[1][r]*T[c][1] + X[2][r]*T[c][2]
  float c00 = X0[0] * T0[0] + X0[1] * T0[1] + X0[2] * T0[2];
  float c01 = X1[0] * T0[0] + X1[1] * T0[1] + X1[2] * T0[2];
  float c11 = X1[0] * T1[0] + X1[1] * T1[1] + X1[2] * T1[2];

  const float det_0 = fmax(1e-6, (double)(c00 * c11 - c01 * c01));
  const float det_1 = fmax(1e-6, (double)((c00 + kernel_size) * (c11 + kernel_size) - c01 * c01));
  float coef = sqrt(det_0 / (det_1 + 1e-6) + 1e-6);
  if (det_0 <= 1e-6 || det_1 <= 1e-6) coef = 0.0f;
  c00 += kernel_size;
  c11 += kernel_size;
  return make_float4(c00, c01, c11, coef);
}

// SH -> RGB (+0.5, clamp at 0 with mask).  Follows computeColorFromSH, forward.cu:20-71.
//
// The clamp flag (colour < 0 before the clamp) is CONTROL FLOW of the backward pass: a colour within an ulp of zero
// that lands on the other side flips dL/dSH of that channel between 0 and its full value (seen once in a 5M-Gaussian
// frame while the colour itself only differed by 1e-7).  So this routine is evaluated exactly like the reference's
// binary evaluates it — every multiply / add / fused multiply-add below is the one in the reference's compiled SASS
// (read off oracle/_ref, preprocessCUDA<3>, section after the three IEEE divisions of the view direction), pinned
// with round-to-nearest intrinsics so the compiler cannot contract it differently: colours, and therefore the clamp
// flags, are bit-identical to the reference (tests: rgb compared bit for bit on every visible Gaussian).
template <typename ShGet>
__device__ __forceinline__ void sh_to_rgb(int deg, ShGet sh /* sh(j) = coefficient j/3, channel j%3 */,
                                          float px, float py, float pz, float cx, float cy, float cz,
                                          float rgb[3], unsigned& clamp_mask) {
  const float dx = __fsub_rn(px, cx), dy = __fsub_rn(py, cy), dz = __fsub_rn(pz, cz);
  // glm::length: dot = (x*x + y*y) + z*z, contracted as fma(z, z, fma(x, x, y*y))
  const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
  const float x = __fdiv_rn(dx, len), y = __fdiv_rn(dy, len), z = __fdiv_rn(dz, len);
  float r0 = __fmul_rn(sh(0), SH_C0), r1 = __fmul_rn(sh(1), SH_C0), r2 = __fmul_rn(sh(2), SH_C0);
  // one fused multiply-add per coefficient and channel, coefficients in ascending order (the three channels are
  // independent chains); each basis value is formed in the reference's association order and used at once
#define SH_ACC(k, c) { const float c_ = (c); r0 = __fmaf_rn(c_, sh(3 * (k)), r0); r1 = __fmaf_rn(c_, sh(3 * (k) + 1), r1); r2 = __fmaf_rn(c_, sh(3 * (k) + 2), r2); }
  if (deg > 0) {
    SH_ACC(1, -__fmul_rn(y, SH_C1)); SH_ACC(2, __fmul_rn(z, SH_C1)); SH_ACC(3, -__fmul_rn(x, SH_C1));
    if (deg > 1) {
      const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
      const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
      const float zz2 = __fadd_rn(zz, zz);                                  // 2 zz (exact)
      const float xx_m_yy = __fsub_rn(xx, yy);
      SH_ACC(4, __fmul_rn(xy, SH_C2_0));
      SH_ACC(5, __fmul_rn(yz, SH_C2_1));
      SH_ACC(6, __fmul_rn(__fsub_rn(__fsub_rn(zz2, xx), yy), SH_C2_2));     // (2zz - xx) - yy
      SH_ACC(7, __fmul_rn(xz, SH_C2_3));
      SH_ACC(8, __fmul_rn(xx_m_yy, SH_C2_4));
      if (deg > 2) {
        const float zz4_m_xx_m_yy = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);                       // fma(zz, 4, -xx) - yy
        SH_ACC(9, __fmul_rn(__fmul_rn(y, SH_C3_0), __fmaf_rn(xx, 3.0f, -yy)));                      // fma(xx, 3, -yy)
        SH_ACC(10, __fmul_rn(__fmul_rn(xy, SH_C3_1), z));
        SH_ACC(11, __fmul_rn(__fmul_rn(y, SH_C3_2), zz4_m_xx_m_yy));
        SH_ACC(12, __fmul_rn(__fmul_rn(z, SH_C3_3), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2))));   // (2zz - 3xx) - 3yy
        SH_ACC(13, __fmul_rn(zz4_m_xx_m_yy, __fmul_rn(x, SH_C3_4)));
        SH_ACC(14, __fmul_rn(xx_m_yy, __fmul_rn(z, SH_C3_5)));
        SH_ACC(15, __fmul_rn(__fmul_rn(x, SH_C3_6), __fmaf_rn(yy, -3.0f, xx)));                     // fma(yy, -3, xx)
      }
    }
  }
#undef SH_ACC
  // result += 0.5; clamped = result < 0; result = max(result, 0)   (forward.cu:63-70; the binary tests r < -0.5)
  const float v0 = __fadd_rn(r0, 0.5f), v1 = __fadd_rn(r1, 0.5f), v2 = __fadd_rn(r2, 0.5f);
  clamp_mask = (v0 < 0.0f ? 1u : 0u) | (v1 < 0.0f ? 2u : 0u) | (v2 < 0.0f ? 4u : 0u);
  rgb[0] = (v0 < 0.0f) ? 0.0f : v0; rgb[1] = (v1 < 0.0f) ? 0.0f : v1; rgb[2] = (v2 < 0.0f) ? 0.0f : v2;
}

constexpr int PRE_THREADS = 256;
constexpr int PRE_SPAN = 1024;        // Gaussians per block: four per thread in the cull phase

// Upper bound of the screen-space radius the exact projection can produce (for the conservative pre-cull).
//   radius = ceil(3 sqrt(lambda_max)),  lambda_max <= mid + sqrt(max(0.1, mid^2 - det)) <= 2 mid + 0.32 = trace(cov2D') + 0.32,
//   trace(cov2D') = trace(T Sigma T^T) + 2 k <= |J|_F^2 |W|_F^2 trace(Sigma) + 2 k   (T = W J, kernel_size k on the diagonal)
//   |J|_F^2 = (fx^2 (1 + (tx/tz)^2) + fy^2 (1 + (ty/tz)^2)) / tz^2 with |tx/tz| <= 1.3 tan(fovx/2) after the reference's clamp.
// Every factor is rounded up generously (1 %, +3 px): the bound only has to be safe, not tight — a Gaussian passes the
// pre-cull when the tile rectangle of (centre, bound) is non-empty, and the exact path then decides.
__device__ __forceinline__ float radius_bound(float trace_sigma, float view_z, float jw2 /* (fx^2(1+limx^2) + fy^2(1+limy^2)) |W|_F^2 */,
                                              float kernel_size) {
  const float tr2d = jw2 * trace_sigma / (view_z * view_z) * 1.01f + 2.f * kernel_size + 0.32f;
  return 3.f * sqrtf(tr2d) + 3.f;
}

__global__ void __launch_bounds__(PRE_THREADS, 3)
preprocess_kernel(int P, int D, int M,
                  const float* __restrict__ means3D, const float* __restrict__ scales, float scale_modifier,
                  const float* __restrict__ rotations, const float* __restrict__ opacities,
                  const float* __restrict__ shs, const float* __restrict__ cov3D_precomp,
                  const float* __restrict__ norm3D_precomp, const float* __restrict__ colors_precomp,
                  const float* __restrict__ viewmatrix, const float* __restrict__ projmatrix,
                  const float* __restrict__ cam_pos, int W, int H, float tan_fovx, float tan_fovy,
                  float focal_x, float focal_y, float kernel_size, int gx, int gy, int band0, int band1,
                  int prefiltered,
                  int* __restrict__ radii, float* __restrict__ rec, float* __restrict__ cov3D_out,
                  unsigned char* __restrict__ clamped, uint32_t* __restrict__ tiles_touched,
                  uint32_t* __restrict__ tile_count, uint32_t* __restrict__ hdr, uint4* __restrict__ tmp,
                  unsigned long long capacity) {
  extern __shared__ __align__(16) unsigned char pre_smem[];
  float4* s_sh = reinterpret_cast<float4*>(pre_smem);                                    // [12][PRE_THREADS]
  uint32_t* s_incl = reinterpret_cast<uint32_t*>(pre_smem + 12 * PRE_THREADS * sizeof(float4));
  int4* s_rect = reinterpret_cast<int4*>(s_incl + PRE_THREADS);
  uint32_t* s_gid = reinterpret_cast<uint32_t*>(s_rect + PRE_THREADS);
  unsigned short* s_cand = reinterpret_cast<unsigned short*>(s_gid + PRE_THREADS);        // [PRE_SPAN]
  __shared__ int s_wcnt[4][PRE_THREADS / 32];
  const float* vm = viewmatrix;
  const float* pm = projmatrix;
  const int tid = threadIdx.x;
  const unsigned lane = tid & 31u, wid = tid >> 5;
  const int base = blockIdx.x * PRE_SPAN;

  // ================= phase A: conservative cull, four Gaussians per thread (independent load chains) =================
  // 64 % of the 1M benchmark frame and 93 % of the 5M frame never reach the image.  Running the exact projection
  // thread-per-Gaussian makes every warp pay the full path for its few visible lanes; instead all Gaussians take this
  // cheap test (centre, view depth, a safe radius bound) and only the candidates — compacted in index order — run the
  // exact path in dense warps below.  A non-candidate provably has an empty tile rectangle: radius 0, no tiles.
  const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
  const float wf2 = vm[0] * vm[0] + vm[1] * vm[1] + vm[2] * vm[2] + vm[4] * vm[4] + vm[5] * vm[5] + vm[6] * vm[6] +
                    vm[8] * vm[8] + vm[9] * vm[9] + vm[10] * vm[10];
  const float jw2 = (focal_x * focal_x * (1.f + limx * limx) + focal_y * focal_y * (1.f + limy * limy)) * wf2;
  unsigned cand_bits = 0;          // bit j: Gaussian base + j*256 + tid is a candidate
  // every load of the four Gaussians is issued before anything is computed: one DRAM round trip per thread instead of
  // eight dependent ones (the test is latency-bound; the few bytes fetched for Gaussians behind the camera are cheaper
  // than a second trip)
  float3 pos4[4], scl4[4];
  float4 rot4[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = base + j * PRE_THREADS + tid;
    const size_t ii = (size_t)(i < P ? i : P - 1);
    pos4[j] = make_float3(means3D[3 * ii], means3D[3 * ii + 1], means3D[3 * ii + 2]);
    if (cov3D_precomp != nullptr) {
      const float* c = cov3D_precomp + 6 * ii;
      scl4[j] = make_float3(c[0], c[3], c[5]);
      rot4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      scl4[j] = make_float3(scales[3 * ii], scales[3 * ii + 1], scales[3 * ii + 2]);
      rot4[j] = *reinterpret_cast<const float4*>(rotations + 4 * ii);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int i = base + j * PRE_THREADS + tid;
    bool cand_j = false;
    if (i < P) {
      const float px = pos4[j].x, py = pos4[j].y, pz = pos4[j].z;
      const float view_z = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
      if (prefiltered && !(view_z > 0.2f)) hdr[HDR_PREFILTER] = 1u;     // the reference traps (auxiliary.h:157-161)
      if (view_z > 0.199f) {                                            // 0.2 with a margin: the exact test follows
        const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
        const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
        const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
        const float p_w = 1.0f / (hw + 0.0000001f);
        const float pix_x = ndc_to_pix(hx * p_w, W), pix_y = ndc_to_pix(hy * p_w, H);
        float trace_sigma;
        if (cov3D_precomp != nullptr) {
          trace_sigma = scl4[j].x + scl4[j].y + scl4[j].z;
        } else {
          const float sx = scl4[j].x, sy = scl4[j].y, sz = scl4[j].z;
          const float4 q = rot4[j];
          float R[3][3];
          rot_from_quat(q.x, q.y, q.z, q.w, R);
          // trace(Sigma) = sum_r (mod s_r)^2 sum_c R[c][r]^2
          const float n0 = R[0][0] * R[0][0] + R[1][0] * R[1][0] + R[2][0] * R[2][0];
          const float n1 = R[0][1] * R[0][1] + R[1][1] * R[1][1] + R[2][1] * R[2][1];
          const float n2 = R[0][2] * R[0][2] + R[1][2] * R[1][2] + R[2][2] * R[2][2];
          trace_sigma = scale_modifier * scale_modifier * (sx * sx * n0 + sy * sy * n1 + sz * sz * n2);
        }
        const float rb = radius_bound(fabsf(trace_sigma), view_z, jw2, kernel_size);
        if (!(rb < 1.0e9f) || !(fabsf(pix_x) < 1.0e9f) || !(fabsf(pix_y) < 1.0e9f)) cand_j = true;   // inf / NaN: let the exact path decide
        else {
          const TileRect r = tile_rect(pix_x, pix_y, (int)rb + 1, gx, gy);
          cand_j = (r.x1 - r.x0) * (r.y1 - r.y0) != 0;
        }
      }
      if (!cand_j) { radii[i] = 0; tiles_touched[i] = 0u; }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, cand_j);
    if (lane == 0) s_wcnt[j][wid] = __popc(bal);
    // rank of this lane among the warp's candidates of pass j, parked in the upper bits
    if (cand_j) cand_bits |= (1u << j) | ((unsigned)__popc(bal & ((1u << lane) - 1u)) << (4 + 5 * j));
  }
  __syncthreads();
  int ncand = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    int off = ncand;
#pragma unroll
    for (int w = 0; w < PRE_THREADS / 32; w++) { off += (w < (int)wid) ? s_wcnt[j][w] : 0; ncand += s_wcnt[j][w]; }
    if ((cand_bits >> j) & 1u) s_cand[off + ((cand_bits >> (4 + 5 * j)) & 31u)] = (unsigned short)(j * PRE_THREADS + tid);
  }
  __syncthreads();

  // ================= phase B: exact projection of the candidates, dense warps =================
  const bool need_sr = cov3D_precomp == nullptr || norm3D_precomp == nullptr;
  // 192 contiguous, 16-byte aligned bytes of SH per Gaussian: staged by cp.async into this thread's own
  // shared-memory column while the covariance math runs
  const bool sh_staged = colors_precomp == nullptr && M == 16 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0;
  const int sh_nq = D == 0 ? 1 : (D == 1 ? 3 : (D == 2 ? 7 : 12));   // float4s covering (D+1)^2 coefficients
  const unsigned wbase = tid & ~31u;

  for (int k0 = 0; k0 < ncand; k0 += PRE_THREADS) {     // block-uniform trip count
    const int k = k0 + tid;
    const bool in_range = k < ncand;
    const int idx = base + (int)s_cand[in_range ? k : 0];
    TileRect vis_rect = {0, 0, 0, 0};
    float vis_depth = 0.f;
    int out_radius = 0;
    uint32_t out_tiles = 0;
    // results of the geometry half that the colour half and the record stores need
    bool visible = false;
    float px = 0.f, py = 0.f, pz = 0.f, sx = 0.f, sy = 0.f, sz = 0.f, opac_in = 0.f;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    float g_pix_x = 0.f, g_pix_y = 0.f, g_conx = 0.f, g_cony = 0.f, g_conz = 0.f, g_coef = 0.f;
    Sym3 g_V = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

    if (in_range) {
      if (sh_staged) {
        const float4* s4 = reinterpret_cast<const float4*>(shs + (size_t)idx * 48);
#pragma unroll
        for (int q4 = 0; q4 < 12; q4++)
          if (q4 < sh_nq) {
            const unsigned sa = (unsigned)__cvta_generic_to_shared(&s_sh[q4 * PRE_THREADS + tid]);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(s4 + q4));
          }
        asm volatile("cp.async.commit_group;\n" ::);
      }
      px = means3D[3 * (size_t)idx]; py = means3D[3 * (size_t)idx + 1]; pz = means3D[3 * (size_t)idx + 2];
      if (need_sr) {
        sx = scales[3 * (size_t)idx]; sy = scales[3 * (size_t)idx + 1]; sz = scales[3 * (size_t)idx + 2];
        q = *reinterpret_cast<const float4*>(rotations + 4 * (size_t)idx);
      }
      opac_in = opacities[idx];
      const float view_z = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
      if (view_z > 0.2f) {
        const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
        const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
        const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
        const float p_w = 1.0f / (hw + 0.0000001f);
        const float proj_x = hx * p_w, proj_y = hy * p_w;

        Sym3 V;
        if (cov3D_precomp != nullptr) {
          const float* c = cov3D_precomp + 6 * (size_t)idx;
          V.c0 = c[0]; V.c1 = c[1]; V.c2 = c[2]; V.c3 = c[3]; V.c4 = c[4]; V.c5 = c[5];
        } else {
          V = cov3d_from_scale_rot(sx, sy, sz, scale_modifier, q.x, q.y, q.z, q.w);
        }

        const float4 cov = cov2d_project(px, py, pz, focal_x, focal_y, tan_fovx, tan_fovy, kernel_size, V, vm);
        const float det = (cov.x * cov.z - cov.y * cov.y);
        if (det != 0.0f) {
          const float det_inv = 1.f / det;
          const float conx = cov.z * det_inv, cony = -cov.y * det_inv, conz = cov.x * det_inv;
          const float mid = 0.5f * (cov.x + cov.z);
          const float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
          const float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
          const float my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
          const float pix_x = ndc_to_pix(proj_x, W), pix_y = ndc_to_pix(proj_y, H);
          const int iradius = my_radius;
          const TileRect r = tile_rect(pix_x, pix_y, iradius, gx, gy);
          const uint32_t ntiles_full = (uint32_t)((r.x1 - r.x0) * (r.y1 - r.y0));
          // screen-space shard: this rank only bins the tile rows [band0, band1)
          TileRect rb = r;
          rb.y0 = max(r.y0, band0); rb.y1 = min(r.y1, band1);
          const uint32_t ntiles = rb.y1 > rb.y0 ? (uint32_t)((rb.x1 - rb.x0) * (rb.y1 - rb.y0)) : 0u;
          if (ntiles_full != 0) {
            visible = true;
            g_pix_x = pix_x; g_pix_y = pix_y; g_conx = conx; g_cony = cony; g_conz = conz; g_coef = cov.w;
            g_V = V;
            out_radius = iradius;
            out_tiles = ntiles;
            vis_rect = rb;
            vis_depth = view_z;
          }
        }
      }
    }
    // ---- reserve this warp's slots of the unsorted instance list NOW: the returning atomic travels to L2 and back
    // while the normals and colours below are evaluated (it used to be issued after them and waited for in place)
    uint32_t incl = out_tiles;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl += y; }
    const uint32_t warp_total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t warp_base = 0;
    if (warp_total != 0 && lane == 31) warp_base = atomicAdd(&hdr[HDR_TMP_COUNT], warp_total);

    if (in_range) {
      if (visible) {
        if (cov3D_precomp == nullptr) {
          float* co = cov3D_out + 6 * (size_t)idx;
          co[0] = g_V.c0; co[1] = g_V.c1; co[2] = g_V.c2; co[3] = g_V.c3; co[4] = g_V.c4; co[5] = g_V.c5;
        }
        float n[3];
        if (norm3D_precomp != nullptr) {
          n[0] = norm3D_precomp[3 * (size_t)idx]; n[1] = norm3D_precomp[3 * (size_t)idx + 1]; n[2] = norm3D_precomp[3 * (size_t)idx + 2];
        } else {
          normal_from_scale_rot(sx, sy, sz, q.x, q.y, q.z, q.w, px, py, pz, cam_pos[0], cam_pos[1], cam_pos[2], n);
        }
        float rgb[3];
        unsigned cmask = 0;
        if (colors_precomp == nullptr) {
          if (sh_staged) {
            asm volatile("cp.async.wait_group 0;\n" ::: "memory");
            // coefficient j sits in word (j & 3) of float4 [j >> 2][tid] of this thread's shared-memory column
            const float* col = reinterpret_cast<const float*>(s_sh) + 4 * tid;
            sh_to_rgb(D, [&](int j) { return col[(j >> 2) * (4 * PRE_THREADS) + (j & 3)]; }, px, py, pz, cam_pos[0],
                      cam_pos[1], cam_pos[2], rgb, cmask);
          } else {
            const float* shp = shs + (size_t)idx * M * 3;
            sh_to_rgb(D, [&](int j) { return shp[j]; }, px, py, pz, cam_pos[0], cam_pos[1], cam_pos[2], rgb, cmask);
          }
        } else {
          rgb[0] = colors_precomp[3 * (size_t)idx]; rgb[1] = colors_precomp[3 * (size_t)idx + 1]; rgb[2] = colors_precomp[3 * (size_t)idx + 2];
        }
        clamped[idx] = (unsigned char)cmask;

        float4* o = reinterpret_cast<float4*>(rec + (size_t)idx * REC_FLOATS);
        o[0] = make_float4(g_pix_x, g_pix_y, g_conx, g_cony);
        o[1] = make_float4(g_conz, opac_in * g_coef, vis_depth, 0.f);
        o[2] = make_float4(rgb[0], rgb[1], rgb[2], n[0]);
        o[3] = make_float4(n[1], n[2], 0.f, 0.f);
      }
      radii[idx] = out_radius;
      tiles_touched[idx] = out_tiles;
    }
    // ---- append this warp's tile instances to the unsorted list -----------------------------------
    // The warp's instances are dealt out to the lanes round-robin (instance j -> owner found by a binary search over
    // the inclusive prefix kept in shared memory), so a large splat does not serialise its lane.  The histogram
    // update (it replaces the per-Gaussian prefix sum of the reference) is a fire-and-forget reduction: nothing in
    // this kernel waits for L2 any more — the slot inside the tile bucket is handed out by the key scatter, which
    // counts the same histogram back down (round 2a took the slot from a RETURNING atomic here and stalled on it:
    // 38 % of this kernel's warp-stall samples sat in this loop).
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");   // culled threads may still have copies in flight
    if (warp_total != 0) {
      warp_base = __shfl_sync(0xffffffffu, warp_base, 31);
      s_incl[tid] = incl;
      s_rect[tid] = make_int4(vis_rect.x0, vis_rect.y0, vis_rect.x1 - vis_rect.x0, (int)__float_as_uint(vis_depth));
      s_gid[tid] = (uint32_t)idx;
      __syncwarp();
      for (uint32_t j = lane; j < warp_total; j += 32) {
        // owner = first lane whose inclusive prefix exceeds j
        int lo = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
          if (s_incl[wbase + lo + step - 1] <= j) lo += step;
        const uint32_t excl = lo > 0 ? s_incl[wbase + lo - 1] : 0u;
        const int4 rc = s_rect[wbase + lo];
        const uint32_t kk = j - excl;                      // kk-th tile of the owner's rectangle, row-major
        const uint32_t ty = kk / (uint32_t)rc.z, tx = kk - ty * (uint32_t)rc.z;
        const uint32_t tile = (uint32_t)(rc.y + (int)ty) * (uint32_t)gx + (uint32_t)(rc.x + (int)tx);
        atomicAdd(&tile_count[tile], 1u);                  // result unused: RED
        const unsigned long long slot = (unsigned long long)warp_base + j;
        if (slot < capacity) tmp[slot] = make_uint4(s_gid[wbase + lo], (uint32_t)rc.w, tile, 0u);
      }
      __syncwarp();     // the warp's shared rows are rewritten by its next pass
    }
  }
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D,
                                    const float* __restrict__ vm, unsigned char* __restrict__ present) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const float px = means3D[3 * idx], py = means3D[3 * idx + 1], pz = means3D[3 * idx + 2];
  const float view_z = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
  present[idx] = view_z > 0.2f ? 1 : 0;
}

}  // namespace

void sfgs_launch_preprocess(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, unsigned long long capacity, float focal_x, float focal_y,
                            cudaStream_t st) {
  const int blocks = (a->P + PRE_SPAN - 1) / PRE_SPAN;
  constexpr size_t smem = PRE_THREADS * (12 * sizeof(float4) + sizeof(uint32_t) + sizeof(int4) + sizeof(uint32_t)) +
                          PRE_SPAN * sizeof(unsigned short);
  static SfgsPerDeviceOnce attr_once;   // function attributes are per device
  if (attr_once.first_use()) {
    cudaFuncSetAttribute(preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  const SfgsBand band = sfgs_band(a->tile_row_begin, a->tile_row_end, im.tiles_y);
  const int band0 = band.b0, band1 = band.b1;
  SFGS_COUNT_LAUNCH();
  preprocess_kernel<<<blocks, PRE_THREADS, smem, st>>>(
      a->P, a->D, a->M, a->means3D, a->scales, a->scale_modifier, a->rotations, a->opacities, a->shs,
      a->cov3D_precomp, a->norm3D_precomp, a->colors_precomp, a->viewmatrix, a->projmatrix, a->cam_pos,
      a->width, a->height, a->tan_fovx, a->tan_fovy, focal_x, focal_y, a->kernel_size, im.tiles_x, im.tiles_y,
      band0, band1, a->prefiltered,
      a->radii, g.rec, g.cov3D, g.clamped, g.tiles_touched, im.tile_count, im.hdr, b.tmp, capacity);
}

void sfgs_launch_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present,
                              cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present);
}
