// sfgs_render_fwd.cu — front-to-back alpha compositing, one CTA per 16x16 tile.
//
// Replaces FORWARD::render / renderCUDA (RAST/cuda_rasterizer/forward.cu:333-468).
// Semantics kept exactly: pixel centres at integer coordinates, `power > 0`
// skip, alpha = min(0.99, o*exp(power)), alpha < 1/255 skip, stop when
// T*(1-alpha) < 1e-4 (that Gaussian is not applied), `contributor` counts every
// tested entry, n_contrib = index of the last applied entry, colour gets
// T*background, depth/normal/alpha/extras have zero background.
//
// Mapping: each warp owns an 8x4 pixel block and runs its own pipeline; nothing in the kernel is block-wide.  The warp
// walks the tile's sorted list front to back 32 positions at a time and keeps the positions whose reach mask (computed
// by the sort stage, sfgs_common.cuh) has its block's bit: that removes ~80% of the (pixel, Gaussian) evaluations
// without changing any result.  It gathers the kept records 16 at a time into a private double-buffered slot of packed
// 64-byte blend records (two lanes per record, cp.async, overlapping the previous chunk's math) and blends the chunk in
// slot order.  The inner loop touches shared memory only (the reference gathers colour/depth/normal from global memory
// per pixel), record parameters sit at immediate offsets, and a warp whose 32 pixels are saturated stops on its own.
#include "sfgs_common.cuh"
#include <type_traits>

namespace {

constexpr int FWD_THREADS = 256;

// peer-mapped [8,H,W] frame blocks of the ranks of one node (sfgs_forward_args.out_peers); n == 0: local outputs
struct OutPeers {
  float* p[8];
  int n;
};

constexpr int F4_CH = 16;
struct alignas(16) FwdWarpSmem {
  float4 rec[2][F4_CH][4];      // 2 KB   the chunk's blend records, double buffered; the free word [1].w of a staged
                                //        record carries its 1-based list position (bits of a uint32)
  uint32_t list[64];            // ring of collected list positions
};
// extra_attrs only: the Gaussian id of each slot, behind the fields above so that their offsets do not move
struct FwdWarpSmemExtra : FwdWarpSmem {
  uint32_t gid[2][F4_CH];
};

// HAS_EXTRA: also blend the ED channels of `extras` [P,ED] into out_extra [ED,H,W] (extra_attrs; Skyfall-GS never
// passes them).  The channels are read from global memory per applied pair, so this instantiation is a slow path.
template <bool HAS_EXTRA>
__global__ void __launch_bounds__(FWD_THREADS)
render_fwd_warp_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                       const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H,
                       int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                       float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_norm,
                       float* __restrict__ out_norm_raw, float* __restrict__ out_alpha, uint32_t* __restrict__ n_contrib,
                       const OutPeers peers, const float* __restrict__ extras, int ED, float* __restrict__ out_extra) {
  if (hdr[HDR_OVERFLOW]) return;
  using Smem = std::conditional_t<HAS_EXTRA, FwdWarpSmemExtra, FwdWarpSmem>;
  __shared__ Smem s_warp[FWD_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  Smem& S = s_warp[wid];
  const int tiles_x = (W + SFGS_TILE - 1) / SFGS_TILE;
  const int tile_y = blockIdx.y + band0;
  const int tile = tile_y * tiles_x + blockIdx.x;
  // warp w covers the 8x4 block (w%2, w/2) of the tile, lane -> (lane%8, lane/8)
  const int px = blockIdx.x * SFGS_TILE + (wid & 1) * 8 + (lane & 7);
  const int py = tile_y * SFGS_TILE + (wid >> 1) * 4 + (lane >> 3);
  const bool inside = px < W && py < H;
  const uint32_t pix_id = (uint32_t)W * py + px;
  const float pixfx = (float)px, pixfy = (float)py;

  const uint2 range = ranges[tile];
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
  const unsigned lt_mask = (1u << lane) - 1u;

  int p = 0;                       // positions [p, total) are still unscanned
  int head = 0, have = 0;          // ring of collected positions: [head, head + have)
  auto scan_gather = [&](int buf) -> int {
    while (have < F4_CH && p < total) {
      const int pos = p + lane;
      unsigned m = 0;
      if (pos < total) m = inst_mask[range.x + pos];
      const bool bit = (m >> wid) & 1u;
      const unsigned b = __ballot_sync(0xffffffffu, bit);
      if (bit) S.list[(head + have + __popc(b & lt_mask)) & 63] = (uint32_t)pos;
      have += __popc(b);
      p += 32;
    }
    __syncwarp();
    const int n = min(have, F4_CH);
    if (lane < 2 * n) {              // two lanes per 64-byte record
      const int r = lane >> 1, hf = lane & 1;
      const uint32_t pos = S.list[(head + r) & 63];
      const uint32_t id = point_list[range.x + pos];
      const float* src = rec + (size_t)id * REC_FLOATS;
      // the record's second quad is (con.z, opacity, depth, free): copied as 8 + 4 bytes, the free word takes the
      // 1-based list position (the value n_contrib records), so the blend loop reads it with the quad it loads anyway
      if (hf == 0) {
        cp_async16(&S.rec[buf][r][0], src);
        cp_async16(&S.rec[buf][r][2], src + 8);
        if constexpr (HAS_EXTRA) S.gid[buf][r] = id;
      } else {
        cp_async16(&S.rec[buf][r][3], src + 12);
        cp_async8(&S.rec[buf][r][1], src + 4);
        cp_async4(&S.rec[buf][r][1].z, src + 6);
        S.rec[buf][r][1].w = __uint_as_float(pos + 1u);
      }
    }
    cp_async_commit();
    head = (head + n) & 63;
    have -= n;
    return n;
  };

  int buf = 0;
  int n_cur = scan_gather(0);
  while (n_cur > 0) {
    cp_async_wait_all();
    __syncwarp();                                   // chunk `buf` has landed and is visible to the whole warp
    if (__all_sync(0xffffffffu, T == 0.0f)) break;  // every pixel of the block is saturated (or outside the image)
    const int n_next = scan_gather(buf ^ 1);        // the next chunk's gather overlaps the math below
    // branch-free slot body (one basic block per chunk: slot k+1's load -> exp chain overlaps slot k's accumulation).
    // A pair that is not applied multiplies every accumulator update by an exact 0.
    auto slot_body = [&](const int k, const float4 a, const float4 c) {
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
    auto slot = [&](const int k) {
      slot_body(k, S.rec[buf][k][0] /* mx, my, con.x, con.y */, S.rec[buf][k][1] /* con.z, opac, depth, 1-based list position */);
    };
    if (n_cur == F4_CH) {                           // every chunk of a warp but its last: no per-slot bound test
#pragma unroll
      for (int k = 0; k < F4_CH; k++) slot(k);
    } else {
#pragma unroll 1
      for (int k = 0; k < n_cur; k++) slot(k);
    }
    buf ^= 1;
    n_cur = n_next;
  }
  cp_async_wait_all();               // nothing may still be landing in this CTA's shared memory when it exits
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

}  // namespace

void sfgs_launch_render_fwd(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, cudaStream_t st) {
  const SfgsBand band = sfgs_band(a->tile_row_begin, a->tile_row_end, im.tiles_y);
  const int band0 = band.b0, band1 = band.b1;
  if (band1 <= band0) return;
  dim3 grid(im.tiles_x, band1 - band0, 1);
  OutPeers op = {};
  if (a->out_peers != nullptr && a->n_out_peers > 0)
    for (op.n = 0; op.n < a->n_out_peers && op.n < 8; op.n++) op.p[op.n] = a->out_peers[op.n];
  SFGS_COUNT_LAUNCH();
  const auto kernel = a->ED > 0 ? render_fwd_warp_kernel<true> : render_fwd_warp_kernel<false>;
  kernel<<<grid, FWD_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr, a->width, a->height, band0, g.rec,
                                       a->background, a->out_color, a->out_depth, a->out_norm, a->out_norm_raw,
                                       a->out_alpha, im.n_contrib, op, a->extra_attrs, a->ED, a->out_extra);
}
