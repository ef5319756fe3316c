// subpixel_adjudicator_f64.cu — the float64 adjudicator (oracle/adjudicator_f64.cu) for a forward with subpixel offsets.
//
// TEST INFRASTRUCTURE, compiled at test time by tests/subpixel_oracle.py.  The per-Gaussian part is the adjudicator's
// own kernel (included below); the per-pixel part is its render adjoint with one change: pixel (px, py) samples at
// ((float)px + off[py][px][0], (float)py + off[py][px][1]), the position the rasterizer blends it at.
#include "../oracle/adjudicator_f64.cu"

namespace {

__global__ void adj_render_backward_subpixel_kernel(
    int W, int H, const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ point_list,
    const float* __restrict__ bg, const float* __restrict__ means2D, const float* __restrict__ conic_opacity,
    const float* __restrict__ colors, const float* __restrict__ depths, const float* __restrict__ norms,
    const float* __restrict__ accum_alphas, const uint32_t* __restrict__ n_contrib,
    const float* __restrict__ dL_dpix, const float* __restrict__ dL_dpix_depth,
    const float* __restrict__ dL_dpix_norm, const float* __restrict__ dL_dpix_alpha,
    double* __restrict__ dL_dmean2D /*[P,3]*/, double* __restrict__ dL_dconic /*[P,4]*/,
    double* __restrict__ dL_dopacity, double* __restrict__ dL_dcolors, double* __restrict__ dL_ddepths,
    double* __restrict__ dL_dnorm3D, const float* __restrict__ off) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= W * H) return;
  const int gx = (W + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
  const int px = pix % W, py = pix / W;
  const int tile = (py / TILE) * gx + (px / TILE);
  const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
  // the sample position of a forward with subpixel offsets, as the product forms it (pixel + offset, in float)
  const float pfx = (float)px + off[2 * (size_t)pix], pfy = (float)py + off[2 * (size_t)pix + 1];
  const double ddelx_dx = 0.5 * W, ddely_dy = 0.5 * H;
  const double T_final = 1.0 - (double)accum_alphas[pix];
  double T = T_final;
  const uint32_t last_contributor = n_contrib[pix];
  double accum_rec[3] = {0, 0, 0}, accum_red = 0, accum_ren[3] = {0, 0, 0}, accum_rea = 0;
  double last_color[3] = {0, 0, 0}, last_depth = 0, last_norm[3] = {0, 0, 0}, last_alpha = 0;
  double dLp[3], dLn[3];
  for (int i = 0; i < 3; i++) { dLp[i] = dL_dpix[i * HW + pix]; dLn[i] = dL_dpix_norm[i * HW + pix]; }
  const double dLd = dL_dpix_depth[pix], dLa = dL_dpix_alpha[pix];
  double bg_dot = 0;
  for (int i = 0; i < 3; i++) bg_dot += (double)bg[i] * dLp[i];
  uint32_t contributor = r1 - r0;
  for (uint32_t k = r1; k-- > r0;) {
    contributor--;
    if (contributor >= last_contributor) continue;
    const uint32_t id = point_list[k];
    const float mxf = means2D[2 * id], myf = means2D[2 * id + 1];
    const float* co = conic_opacity + 4 * (size_t)id;
    // ---- float32 control flow, the reference's expressions (backward.cu:617-628) ----
    {
      const float dxf = mxf - pfx, dyf = myf - pfy;
      const float power_f = -0.5f * (co[0] * dxf * dxf + co[2] * dyf * dyf) - co[1] * dxf * dyf;
      if (power_f > 0.0f) continue;
      const float G_f = exp(power_f);
      const float alpha_f = min(0.99f, co[3] * G_f);
      if (alpha_f < 1.0f / 255.0f) continue;
    }
    // ---- float64 values ----
    const double dx = (double)mxf - (double)pfx, dy = (double)myf - (double)pfy;
    const double c0 = co[0], c1 = co[1], c2 = co[2], op = co[3];
    const double power = -0.5 * (c0 * dx * dx + c2 * dy * dy) - c1 * dx * dy;
    const double G = exp(power);
    const double alpha = fmin((double)0.99f, op * G);
    T = T / (1.0 - alpha);
    const double weight = alpha * T;
    double dL_dalpha = 0.0;
    for (int ch = 0; ch < 3; ch++) {
      const double c = colors[3 * id + ch];
      accum_rec[ch] = last_alpha * last_color[ch] + (1.0 - last_alpha) * accum_rec[ch];
      last_color[ch] = c;
      dL_dalpha += (c - accum_rec[ch]) * dLp[ch];
      atomic_add_d(&dL_dcolors[3 * id + ch], weight * dLp[ch]);
    }
    const double dep = depths[id];
    accum_red = last_alpha * last_depth + (1.0 - last_alpha) * accum_red;
    last_depth = dep;
    dL_dalpha += (dep - accum_red) * dLd;
    atomic_add_d(&dL_ddepths[id], weight * dLd);
    for (int ch = 0; ch < 3; ch++) {
      const double n = norms[3 * id + ch];
      accum_ren[ch] = last_alpha * last_norm[ch] + (1.0 - last_alpha) * accum_ren[ch];
      last_norm[ch] = n;
      dL_dalpha += (n - accum_ren[ch]) * dLn[ch];
      atomic_add_d(&dL_dnorm3D[3 * id + ch], weight * dLn[ch]);
    }
    accum_rea = last_alpha + (1.0 - last_alpha) * accum_rea;
    dL_dalpha += (1.0 - accum_rea) * dLa;
    dL_dalpha *= T;
    last_alpha = alpha;
    dL_dalpha += (-T_final / (1.0 - alpha)) * bg_dot;
    const double dL_dG = op * dL_dalpha;
    const double gdx = G * dx, gdy = G * dy;
    const double dG_ddelx = -gdx * c0 - gdy * c1;
    const double dG_ddely = -gdy * c2 - gdx * c1;
    atomic_add_d(&dL_dmean2D[3 * id], dL_dG * dG_ddelx * ddelx_dx);
    atomic_add_d(&dL_dmean2D[3 * id + 1], dL_dG * dG_ddely * ddely_dy);
    atomic_add_d(&dL_dmean2D[3 * id + 2], fabs(dL_dG * dG_ddelx * ddelx_dx) + fabs(dL_dG * dG_ddely * ddely_dy));
    atomic_add_d(&dL_dconic[4 * id], -0.5 * gdx * dx * dL_dG);
    atomic_add_d(&dL_dconic[4 * id + 1], -0.5 * gdx * dy * dL_dG);
    atomic_add_d(&dL_dconic[4 * id + 3], -0.5 * gdy * dy * dL_dG);
    atomic_add_d(&dL_dopacity[id], G * dL_dalpha);
  }
}

}  // namespace

extern "C" {

// adj_backward_f64 (oracle/adjudicator_f64.cu) with the [H,W,2] device offsets the forward used
int adj_backward_f64_subpixel(int P, int D, int M, int W, int H,
                     const uint32_t* ranges, const uint32_t* point_list, const float* bg, const float* means2D,
                     const float* conic_opacity, const float* colors, const float* depths, const float* norms,
                     const float* accum_alphas, const uint32_t* n_contrib, const float* dL_dpix,
                     const float* dL_dpix_depth, const float* dL_dpix_norm, const float* dL_dpix_alpha,
                     const float* means3D, const int* radii, const float* shs, const unsigned char* clamped,
                     const float* scales, const float* rotations, float scale_modifier, const float* cov3Ds,
                     const float* view, const float* proj, float tan_fovx, float tan_fovy, float kernel_size,
                     const float* campos,
                     double* dL_dmean2D, double* dL_dconic, double* dL_dopacity, double* dL_dcolors,
                     double* dL_ddepths, double* dL_dnorm3D, double* dL_dmean3D, double* dL_dcov3D, double* dL_dsh,
                     double* dL_dscale, double* dL_drot, void* stream, const float* subpixel_offset) {
  cudaStream_t st = (cudaStream_t)stream;
  const int N = W * H;
  if (N > 0 && P > 0) {
    adj_render_backward_subpixel_kernel<<<(N + 127) / 128, 128, 0, st>>>(
        W, H, ranges, point_list, bg, means2D, conic_opacity, colors, depths, norms, accum_alphas, n_contrib, dL_dpix,
        dL_dpix_depth, dL_dpix_norm, dL_dpix_alpha, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors, dL_ddepths,
        dL_dnorm3D, subpixel_offset);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    adj_gauss_backward_kernel<<<(P + 127) / 128, 128, 0, st>>>(
        P, D, M, means3D, radii, shs, clamped, scales, rotations, scale_modifier, cov3Ds, norms, view, proj, W, H,
        tan_fovx, tan_fovy, kernel_size, campos, conic_opacity, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors,
        dL_ddepths, dL_dmean3D, dL_dcov3D, dL_dnorm3D, dL_dsh, dL_dscale, dL_drot);
    e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaStreamSynchronize(st);
}

}  // extern "C"
