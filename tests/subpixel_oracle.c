/* subpixel_oracle.c — the CPU oracle (oracle/sfgs_oracle.c) for a forward with subpixel offsets.
 *
 * TEST INFRASTRUCTURE, compiled at test time by tests/subpixel_oracle.py with the oracle's flags.  Preprocess, binning
 * and the per-Gaussian adjoint are the oracle's own routines (included below); the blend and its adjoint are the
 * oracle's with one change: pixel (px, py) samples at ((float)px + off[py][px][0], (float)py + off[py][px][1]), the
 * position the rasterizer blends it at.  off: [H,W,2] floats.
 */
#include "../oracle/sfgs_oracle.c"

void oracle_render_subpixel(int W, int H, int ED, const uint32_t* ranges, const uint32_t* point_list,
                            const float* means2D, const float* colors, const float* norms, const float* depths,
                            const float* extras, const float* conic_opacity, const float* bg, float* out_color,
                            float* out_depth, float* out_norm, float* out_alpha, float* out_extra, uint32_t* n_contrib,
                            const float* off) {
  const int gx = (W + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 16)
  for (int pix = 0; pix < H * W; pix++) {
    const int px = pix % W, py = pix / W;
    const int tile = (py / TILE) * gx + (px / TILE);
    const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
    const float pfx = (float)px + off[2 * (size_t)pix], pfy = (float)py + off[2 * (size_t)pix + 1];
    float T = 1.0f, C[3] = {0, 0, 0}, Dp = 0, N[3] = {0, 0, 0}, E[MAX_EXTRA];
    for (int i = 0; i < ED; i++) E[i] = 0;
    uint32_t contributor = 0, last = 0;
    for (uint32_t k = r0; k < r1; k++) {
      contributor++;
      const uint32_t id = point_list[k];
      const float dx = means2D[2 * id] - pfx, dy = means2D[2 * id + 1] - pfy;
      const float* co = conic_opacity + 4 * (size_t)id;
      /* GPU: t = fma(co.x*dx, dx, (co.z*dy)*dy) ... keep the reference's expression, contraction-agnostic to 1 ulp */
      const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
      if (power > 0.0f) continue;
      const float alpha = fminf_(0.99f, co[3] * expf(power));
      if (alpha < 1.0f / 255.0f) continue;
      const float test_T = T * (1 - alpha);
      if (test_T < 0.0001f) break;   /* done: this and all later Gaussians are not applied */
      for (int ch = 0; ch < 3; ch++) C[ch] += colors[3 * id + ch] * alpha * T;
      Dp += depths[id] * alpha * T;
      for (int ch = 0; ch < 3; ch++) N[ch] += norms[3 * id + ch] * alpha * T;
      for (int ch = 0; ch < ED; ch++) E[ch] += extras[(size_t)id * ED + ch] * alpha * T;
      T = test_T;
      last = contributor;
    }
    out_alpha[pix] = 1 - T;
    n_contrib[pix] = last;
    for (int ch = 0; ch < 3; ch++) out_color[ch * HW + pix] = C[ch] + T * bg[ch];
    out_depth[pix] = Dp;
    for (int ch = 0; ch < 3; ch++) out_norm[ch * HW + pix] = N[ch];
    for (int ch = 0; ch < ED; ch++) out_extra[ch * HW + pix] = E[ch];
  }
}

void oracle_render_backward_subpixel(int W, int H, int ED, const uint32_t* ranges, const uint32_t* point_list,
                                     const float* bg, const float* means2D, const float* conic_opacity,
                                     const float* colors, const float* depths, const float* norms, const float* extras,
                                     const float* accum_alphas, const uint32_t* n_contrib, const float* dL_dpix,
                                     const float* dL_dpix_depth, const float* dL_dpix_norm,
                                     const float* dL_dpix_alpha, const float* dL_dpix_extra,
                                     float* dL_dmean2D /*[P,3]*/, float* dL_dconic /*[P,4]*/, float* dL_dopacity,
                                     float* dL_dcolors, float* dL_ddepths, float* dL_dnorm3D, float* dL_dextras,
                                     const float* off) {
  const int gx = (W + TILE - 1) / TILE;
  const size_t HW = (size_t)H * W;
  const float ddelx_dx = 0.5 * W, ddely_dy = 0.5 * H;
#pragma omp parallel for schedule(dynamic, 16)
  for (int pix = 0; pix < H * W; pix++) {
    const int px = pix % W, py = pix / W;
    const int tile = (py / TILE) * gx + (px / TILE);
    const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
    const float pfx = (float)px + off[2 * (size_t)pix], pfy = (float)py + off[2 * (size_t)pix + 1];
    const float T_final = 1 - accum_alphas[pix];
    float T = T_final;
    const uint32_t last_contributor = n_contrib[pix];
    float accum_rec[3] = {0, 0, 0}, accum_red = 0, accum_ren[3] = {0, 0, 0}, accum_rea = 0, accum_ree[MAX_EXTRA];
    float last_color[3] = {0, 0, 0}, last_depth = 0, last_norm[3] = {0, 0, 0}, last_alpha = 0, last_extra[MAX_EXTRA];
    float dLp[3], dLn[3], dLe[MAX_EXTRA];
    for (int i = 0; i < 3; i++) { dLp[i] = dL_dpix[i * HW + pix]; dLn[i] = dL_dpix_norm[i * HW + pix]; }
    const float dLd = dL_dpix_depth[pix], dLa = dL_dpix_alpha[pix];
    for (int i = 0; i < ED; i++) { dLe[i] = dL_dpix_extra[i * HW + pix]; accum_ree[i] = 0; last_extra[i] = 0; }
    uint32_t contributor = r1 - r0;
    for (uint32_t k = r1; k-- > r0;) {
      contributor--;
      if (contributor >= last_contributor) continue;
      const uint32_t id = point_list[k];
      const float dx = means2D[2 * id] - pfx, dy = means2D[2 * id + 1] - pfy;
      const float* co = conic_opacity + 4 * (size_t)id;
      const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
      if (power > 0.0f) continue;
      const float G = expf(power);
      const float alpha = fminf_(0.99f, co[3] * G);
      if (alpha < 1.0f / 255.0f) continue;
      T = T / (1.f - alpha);
      const float weight = alpha * T;
      float dL_dalpha = 0.0f;
      for (int ch = 0; ch < 3; ch++) {
        const float c = colors[3 * id + ch];
        accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
        last_color[ch] = c;
        dL_dalpha += (c - accum_rec[ch]) * dLp[ch];
        atomic_addf(&dL_dcolors[3 * id + ch], weight * dLp[ch]);
      }
      const float dep = depths[id];
      accum_red = last_alpha * last_depth + (1.f - last_alpha) * accum_red;
      last_depth = dep;
      dL_dalpha += (dep - accum_red) * dLd;
      atomic_addf(&dL_ddepths[id], weight * dLd);
      for (int ch = 0; ch < 3; ch++) {
        const float n = norms[3 * id + ch];
        accum_ren[ch] = last_alpha * last_norm[ch] + (1.f - last_alpha) * accum_ren[ch];
        last_norm[ch] = n;
        dL_dalpha += (n - accum_ren[ch]) * dLn[ch];
        atomic_addf(&dL_dnorm3D[3 * id + ch], weight * dLn[ch]);
      }
      for (int ch = 0; ch < ED; ch++) {
        const float e = extras[(size_t)id * ED + ch];
        accum_ree[ch] = last_alpha * last_extra[ch] + (1.f - last_alpha) * accum_ree[ch];
        last_extra[ch] = e;
        dL_dalpha += (e - accum_ree[ch]) * dLe[ch];
        atomic_addf(&dL_dextras[(size_t)id * ED + ch], weight * dLe[ch]);
      }
      accum_rea = last_alpha + (1.f - last_alpha) * accum_rea;
      dL_dalpha += (1 - accum_rea) * dLa;
      dL_dalpha *= T;
      last_alpha = alpha;
      float bg_dot = 0;
      for (int i = 0; i < 3; i++) bg_dot += bg[i] * dLp[i];
      dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
      const float dL_dG = co[3] * dL_dalpha;
      const float gdx = G * dx, gdy = G * dy;
      const float dG_ddelx = -gdx * co[0] - gdy * co[1];
      const float dG_ddely = -gdy * co[2] - gdx * co[1];
      atomic_addf(&dL_dmean2D[3 * id], dL_dG * dG_ddelx * ddelx_dx);
      atomic_addf(&dL_dmean2D[3 * id + 1], dL_dG * dG_ddely * ddely_dy);
      atomic_addf(&dL_dmean2D[3 * id + 2], fabsf(dL_dG * dG_ddelx * ddelx_dx) + fabsf(dL_dG * dG_ddely * ddely_dy));
      atomic_addf(&dL_dconic[4 * id], -0.5f * gdx * dx * dL_dG);
      atomic_addf(&dL_dconic[4 * id + 1], -0.5f * gdx * dy * dL_dG);
      atomic_addf(&dL_dconic[4 * id + 3], -0.5f * gdy * dy * dL_dG);
      atomic_addf(&dL_dopacity[id], G * dL_dalpha);
    }
  }
}
