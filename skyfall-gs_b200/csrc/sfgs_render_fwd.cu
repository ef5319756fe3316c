// sfgs_render_fwd.cu — front-to-back alpha compositing, one CTA per 16x16 tile.
//
// Replaces FORWARD::render / renderCUDA (RAST/cuda_rasterizer/forward.cu:333-468).
// Semantics kept exactly: pixel centres at integer coordinates, `power > 0`
// skip, alpha = min(0.99, o*exp(power)), alpha < 1/255 skip, stop when
// T*(1-alpha) < 1e-4 (that Gaussian is not applied), `contributor` counts every
// tested entry, n_contrib = index of the last applied entry, colour gets
// T*background, depth/normal/alpha/extras have zero background.
//
// The tile / block / pixel mapping, the reach-list walk (front to back) and the double-buffered chunk loop are those
// of sfgs_blend_walk.cuh; this file holds the slot body and the epilogue.  The inner loop touches shared memory only
// (the reference gathers colour/depth/normal from global memory per pixel), and a warp whose 32 pixels are saturated
// stops on its own.
#include "sfgs_blend_walk.cuh"
#include <algorithm>
#include <type_traits>

namespace {

// peer-mapped [8,H,W] frame blocks of the ranks of one node (sfgs_forward_args.out_peers); n == 0: local outputs
struct OutPeers {
  float* p[8];
  int n;
};

// HAS_EXTRA: also blend the ED channels of `extras` [P,ED] into out_extra [ED,H,W] (extra_attrs; Skyfall-GS never
// passes them).  The channels are read from global memory per applied pair, so this instantiation is a slow path.
// How the body takes the peer table: the form that leaves the code generated for the two default kernels what it was
// before the body moved out of them (by value with extra_attrs, by reference otherwise; the semantics are the same).
template <bool HAS_EXTRA>
using PeersArg = std::conditional_t<HAS_EXTRA, const OutPeers, const OutPeers&>;

// JITTER: subpixel offsets — pixel (x, y) samples the splats at (x, y) + off[W y + x] ([H,W,2] floats); the tile's
// list, the walk and the slot body are unchanged (the reach masks were dilated by the offsets' bound).
template <bool HAS_EXTRA, bool JITTER>
__device__ __forceinline__ void
render_fwd_warp(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H,
                int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_norm,
                float* __restrict__ out_norm_raw, float* __restrict__ out_alpha, uint32_t* __restrict__ n_contrib,
                PeersArg<HAS_EXTRA> peers, const float* __restrict__ extras, int ED, float* __restrict__ out_extra,
                const float2* __restrict__ off) {
  if (hdr[HDR_OVERFLOW]) return;
  __shared__ BlendStage<HAS_EXTRA> s_warp[BLEND_WARPS];   // extra_attrs: the slot's gid word is the Gaussian id
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  BlendStage<HAS_EXTRA>& S = s_warp[wid];
  const BlendPixel pix(band0, W, H, wid, lane);
  const bool inside = pix.inside;
  const uint32_t pix_id = pix.id;
  const float2 o = JITTER && inside ? off[pix_id] : make_float2(0.f, 0.f);
  const float pixfx = JITTER ? pix.x + o.x : pix.x, pixfy = JITTER ? pix.y + o.y : pix.y;

  const uint2 range = ranges[pix.tile];
  const int total = (int)(range.y - range.x);

  // Transmittance of a live pixel.  A pixel that is finished (outside the image, or its next T would drop below
  // 1e-4) parks its transmittance in T_done and continues with T = 0: every later record then fails the same
  // `T*(1-alpha) < 1e-4` test on its own, so the blend loop needs no separate per-lane "done" flag (a live T is
  // never 0: it starts at 1, shrinks by factors >= 0.01 and stops before it reaches 1e-4).
  float T = inside ? 1.0f : 0.0f;
  float T_done = 0.0f;
  uint32_t last_contributor = 0;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f, Dp = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
  float E[HAS_EXTRA ? SFGS_MAX_EXTRA : 1];
  if constexpr (HAS_EXTRA)
    for (int ch = 0; ch < ED; ch++) E[ch] = 0.f;
  const SfgsExpConsts ek = sfgs_exp_consts(hdr[HDR_ZERO]);

  BlendWalk<false, HAS_EXTRA ? GID_GAUSSIAN : GID_NONE> walk(S, inst_mask, point_list, rec, range, total, wid, lane);
  // branch-free slot body (a pair that is not applied multiplies every accumulator update by an exact 0)
  auto slot = [&](const int buf, const int k, const float4 a /* mx, my, con.x, con.y */,
                  const float4 c /* con.z, opac, depth, 1-based list position */) {
    const float dx = a.x - pixfx, dy = a.y - pixfy;
    const float power = -0.5f * (a.z * dx * dx + c.x * dy * dy) - a.w * dx * dy;
    const float4 f = S.rec[buf][k][2];        // r, g, b, nx
    const float4 g = S.rec[buf][k][3];        // ny, nz
    const float alpha = min(0.99f, c.y * sfgs_expf(power, ek));
    const bool ok = !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
    const float test_T = T * (1 - alpha);
    const bool stop = ok && (test_T < 0.0001f);
    const bool apply = ok && !stop;
    const float Ta = apply ? T : 0.0f;
    // colour and normal (|values| <= 1) take the pair's weight alpha*T as one factor, and so do the extras; the depth
    // image reaches hundreds of units, where 1e-5 absolute is below one ulp, so it keeps the reference's exact
    // association (depth * alpha) * T and stays bit-identical
    const float w = alpha * Ta;
    C0 = fmaf(f.x, w, C0); C1 = fmaf(f.y, w, C1); C2 = fmaf(f.z, w, C2);
    Dp = fmaf(c.z * alpha, Ta, Dp);
    N0 = fmaf(f.w, w, N0); N1 = fmaf(g.x, w, N1); N2 = fmaf(g.y, w, N2);
    if constexpr (HAS_EXTRA) {
      const float* ex = extras + (size_t)S.gid[buf][k] * ED;
      for (int ch = 0; ch < ED; ch++) E[ch] = fmaf(ex[ch], w, E[ch]);
    }
    T_done = stop ? fmaxf(T_done, T) : T_done;
    T = apply ? test_T : (stop ? 0.0f : T);
    last_contributor = apply ? __float_as_uint(c.w) : last_contributor;
  };
  blend_chunks<true>(
      walk, [&] { return __all_sync(0xffffffffu, T == 0.0f); },   // every pixel is saturated or outside the image
      [&](const int buf, const int n) {
        if (n == BLEND_CH) {                        // every chunk of a warp but its last: no per-slot bound test
#pragma unroll
          for (int k = 0; k < BLEND_CH; k++) slot(buf, k, S.rec[buf][k][0], S.rec[buf][k][1]);
        } else {
#pragma unroll 1
          for (int k = 0; k < n; k++) slot(buf, k, S.rec[buf][k][0], S.rec[buf][k][1]);
        }
      });
  if (T == 0.0f) T = T_done;         // finished early: the transmittance it finished with

  if (inside) {
    const size_t HW = (size_t)H * W;
    n_contrib[pix_id] = last_contributor;
    const float c0 = C0 + T * bg_color[0], c1 = C1 + T * bg_color[1], c2 = C2 + T * bg_color[2];
    if (out_norm_raw != nullptr) {
      // fused post-op: F.normalize(norm, p=2, dim=0, eps=1e-12) (RAST/diff_gauss/__init__.py:48); the raw blend is
      // kept for the adjoint
      out_norm_raw[0 * HW + pix_id] = N0;
      out_norm_raw[1 * HW + pix_id] = N1;
      out_norm_raw[2 * HW + pix_id] = N2;
      const float d = fmaxf(sqrtf(N0 * N0 + N1 * N1 + N2 * N2), 1e-12f);
      N0 = N0 / d; N1 = N1 / d; N2 = N2 / d;
    }
    if (peers.n > 0) {
      // the all-gather of the band: this pixel goes to every rank's frame (plane order colour, depth, alpha, normal)
      for (int r = 0; r < peers.n; r++) {
        float* f = peers.p[r];
        f[0 * HW + pix_id] = c0; f[1 * HW + pix_id] = c1; f[2 * HW + pix_id] = c2;
        f[3 * HW + pix_id] = Dp;
        f[4 * HW + pix_id] = 1 - T;
        f[5 * HW + pix_id] = N0; f[6 * HW + pix_id] = N1; f[7 * HW + pix_id] = N2;
      }
    } else {
      out_alpha[pix_id] = 1 - T;
      out_color[0 * HW + pix_id] = c0;
      out_color[1 * HW + pix_id] = c1;
      out_color[2 * HW + pix_id] = c2;
      out_depth[pix_id] = Dp;
      out_norm[0 * HW + pix_id] = N0;
      out_norm[1 * HW + pix_id] = N1;
      out_norm[2 * HW + pix_id] = N2;
    }
    if constexpr (HAS_EXTRA)
      for (int ch = 0; ch < ED; ch++) out_extra[ch * HW + pix_id] = E[ch];
  }
}

template <bool HAS_EXTRA>
__global__ void __launch_bounds__(BLEND_THREADS)
render_fwd_warp_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                       const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H,
                       int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                       float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_norm,
                       float* __restrict__ out_norm_raw, float* __restrict__ out_alpha, uint32_t* __restrict__ n_contrib,
                       const OutPeers peers, const float* __restrict__ extras, int ED, float* __restrict__ out_extra) {
  render_fwd_warp<HAS_EXTRA, false>(ranges, point_list, inst_mask, hdr, W, H, band0, rec, bg_color, out_color, out_depth,
                                    out_norm, out_norm_raw, out_alpha, n_contrib, peers, extras, ED, out_extra, nullptr);
}

// subpixel offsets into local outputs; no extra_attrs (sfgs_rasterize_forward_subpixel rejects them)
__global__ void __launch_bounds__(BLEND_THREADS)
render_fwd_jitter_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                         const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H,
                         int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                         float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_norm,
                         float* __restrict__ out_norm_raw, float* __restrict__ out_alpha,
                         uint32_t* __restrict__ n_contrib, const float2* __restrict__ off) {
  render_fwd_warp<false, true>(ranges, point_list, inst_mask, hdr, W, H, band0, rec, bg_color, out_color, out_depth,
                               out_norm, out_norm_raw, out_alpha, n_contrib, OutPeers{}, nullptr, 0, nullptr, off);
}

// subpixel offsets with the fused image all-gather of the tile-row sharded mode: the band goes to every rank's
// [8,H,W] frame block (a kernel of its own, so that the local-output kernel above keeps its code)
__global__ void __launch_bounds__(BLEND_THREADS)
render_fwd_jitter_peers_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                               const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W,
                               int H, int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                               float* __restrict__ out_norm_raw, uint32_t* __restrict__ n_contrib,
                               const OutPeers peers, const float2* __restrict__ off) {
  render_fwd_warp<false, true>(ranges, point_list, inst_mask, hdr, W, H, band0, rec, bg_color, nullptr, nullptr,
                               nullptr, out_norm_raw, nullptr, n_contrib, peers, nullptr, 0, nullptr, off);
}

// max |off_x|, max |off_y| over the frame into HDR_OFF_EX / HDR_OFF_EY (non-negative floats order as their bits), and
// HDR_OFF_BAD if any offset is NaN or Inf (those are left out of the bound; the forward then fails)
__global__ void __launch_bounds__(256)
offset_bound_kernel(size_t n, const float2* __restrict__ off, uint32_t* __restrict__ hdr) {
  float ex = 0.f, ey = 0.f;
  bool bad = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float2 o = off[i];
    const bool fx = isfinite(o.x), fy = isfinite(o.y);
    bad |= !fx || !fy;
    ex = fmaxf(ex, fx ? fabsf(o.x) : 0.f);
    ey = fmaxf(ey, fy ? fabsf(o.y) : 0.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ex = fmaxf(ex, __shfl_xor_sync(0xffffffffu, ex, o));
    ey = fmaxf(ey, __shfl_xor_sync(0xffffffffu, ey, o));
  }
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&hdr[HDR_OFF_EX], __float_as_uint(ex));
    atomicMax(&hdr[HDR_OFF_EY], __float_as_uint(ey));
    if (bad) hdr[HDR_OFF_BAD] = 1u;
  }
}

}  // namespace

void sfgs_launch_offset_bound(const ImageLayout& im, int W, int H, const float* off, cudaStream_t st) {
  const size_t n = (size_t)W * H;
  const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, 132 * 8);
  SFGS_COUNT_LAUNCH();
  offset_bound_kernel<<<blocks, 256, 0, st>>>(n, reinterpret_cast<const float2*>(off), im.hdr);
}

void sfgs_launch_render_fwd(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, const float* off, cudaStream_t st) {
  dim3 grid;
  int band0;
  if (!blend_grid(a->tile_row_begin, a->tile_row_end, im, grid, band0)) return;
  OutPeers op = {};
  if (a->out_peers != nullptr && a->n_out_peers > 0)
    for (op.n = 0; op.n < a->n_out_peers && op.n < 8; op.n++) op.p[op.n] = a->out_peers[op.n];
  if (off != nullptr && op.n > 0) {
    SFGS_COUNT_LAUNCH();
    render_fwd_jitter_peers_kernel<<<grid, BLEND_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr,
                                                                   a->width, a->height, band0, g.rec, a->background,
                                                                   a->out_norm_raw, im.n_contrib, op,
                                                                   reinterpret_cast<const float2*>(off));
    return;
  }
  if (off != nullptr) {
    SFGS_COUNT_LAUNCH();
    render_fwd_jitter_kernel<<<grid, BLEND_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr, a->width,
                                                             a->height, band0, g.rec, a->background, a->out_color,
                                                             a->out_depth, a->out_norm, a->out_norm_raw, a->out_alpha,
                                                             im.n_contrib, reinterpret_cast<const float2*>(off));
    return;
  }
  SFGS_COUNT_LAUNCH();
  const auto kernel = a->ED > 0 ? render_fwd_warp_kernel<true> : render_fwd_warp_kernel<false>;
  kernel<<<grid, BLEND_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr, a->width, a->height, band0,
                                         g.rec, a->background, a->out_color, a->out_depth, a->out_norm, a->out_norm_raw,
                                         a->out_alpha, im.n_contrib, op, a->extra_attrs, a->ED, a->out_extra);
}
