// sfgs_render_bwd.cu — adjoint of the alpha compositing, one CTA per 16x16 tile.
//
// Replaces BACKWARD::render / renderCUDA (RAST/cuda_rasterizer/backward.cu:509-754), which issues >= 14
// global float atomicAdd per (pixel, Gaussian) pair.
//
// The tile / block / pixel mapping, the reach-list walk (back to front, from the block's last contributor) and the
// double-buffered chunk loop are those of sfgs_blend_walk.cuh.  Per 16-record chunk:
//
//   phase 1  pixel-parallel (lane = pixel): the per-pixel recursion over the chunk's records in slot order.  The
//            reference's eight per-channel accumulators collapse into the scalar form
//                dL/dalpha_j = T_j (g_j - A_j),  g_j = <dL/dpix, attr_j>,  A_j = a_{j+1} g_{j+1} + (1 - a_{j+1}) A_{j+1}
//            (the channel-sum of accum_rec/accum_red/accum_ren/accum_rea, backward.cu:660-711), carried as one
//            register C = A of the next active record.  Per pair only two numbers leave the lane:  w = alpha*T  and
//            h = G * dL/dalpha ; they are parked in a per-warp shared-memory tile [pixel][slot].  Slot k is a
//            compile-time constant after unrolling, so record parameters, list position and the (w, h) hand-over all
//            sit at immediate offsets;
//   phase 2  record-parallel (lane = slot of the chunk x half of the block's pixels): all 14 per-Gaussian sums are
//            linear in (w, h):
//                sum w*dL/dpix_c (7 channels),  sum h*{1, dx, dy, dx^2, dx dy, dy^2},  sum |..| for the abs-gradient,
//            so each lane streams down its record's column of the tile accumulating in registers — no cross-lane
//            reduction except one 16-lane exchange between the two pixel halves.  The loop is fully unrolled and
//            sums h against the pixels' compile-time offsets from the centre of their 8x2 half; the moments about
//            the record's centre follow once per chunk by binomial expansion;
//   combine  each (block, record) pair ends in four red.global.add.v4.f32 (tools/red_bench.cu times such traffic on
//            its own; the ~16 M issued per frame hide behind the math): ~200x fewer global atomics than the reference.
//            The ORDERED instantiation (the deterministic backward, sfgs_bwd_order.cu) stores the pair's 16 words with
//            plain 16-byte stores to its own row of a partial table instead, row (sorted instance) * 8 + block, and
//            sets that row's written flag; a later pass adds the rows of each Gaussian in a fixed order.
//
// A record that none of the warp's 32 pixels blends (0.6 % on the benchmark frame: the reach mask is conservative)
// occupies a slot with zeros.
// (T is recovered back to front as T_j = T_{j+1} * rcp.approx(1 - alpha_{j+1}).  Refining the reciprocal with a Newton step
// costs time and does NOT change the error statistics against the float64 adjudicator — the worst elements are
// summation-order noise of ill-conditioned sums, which vary by 5x between runs of either implementation, not T drift.)
// (Numerics of the expansion in phase 2: for a record whose centre is (DX, DY) from the half's centre, sum h dx^2
// formed as DX^2 sum h - 2 DX sum h x + sum h x^2 carries rounding error of about eps (|DX| + |x|)^2 sum|h|, where the
// direct sum over the pixels carries eps (DX - x)^2 sum|h|.  With the origin at the half's first pixel (offsets 0..7)
// the expansion's error was several times the direct sum's for the many small records centred inside the block, and
// the float64-adjudicated conic gradients (cov3D, scales, rotations) exceeded the reference build's error.  Centred
// offsets (+-3.5 .. +-0.5, rows +-0.5) bring it back within the reference's error.)
#include "sfgs_blend_walk.cuh"
#include <type_traits>

namespace {

constexpr int PIXF = 8;           // floats per pixel-table row: dLc[3], dLd, dLn[3], half centre (see below)

// PEER: the target may be another GPU's memory reached over NVLink and every GPU of the node adds into it, so the
// reduction must be system-scope; otherwise the default (device) scope
template <bool PEER>
__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
  if (PEER)
    asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
  else
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

// peer-mapped accumulator slices of the ranks of one node (sfgs_backward_args.acc_peers)
struct PeerTable {
  float* p[8];
  int per;      // Gaussians per slice
};

struct WarpSmem {
  BlendStage<true> st;          // 2.4 KB the walk's records, ring and gid words
  float2 wh[32][BLEND_CH + 1];  // 4.25 KB phase-1 -> phase-2 hand-over, [pixel][slot], padded
  float pix[32][PIXF];          // 1 KB    per-pixel cotangents
};
struct WarpSmemJitter : WarpSmem {
  float2 pos[32];               // 256 B   per-pixel sample positions (JITTER)
};
// DIST: the pixel rows widened by the depth distortion's per-pixel constants
template <class Base>
struct WarpSmemDist : Base {
  float2 dist[32];              // 256 B   (2 c A, mu) per pixel
};

// HAS_EXTRA: also the adjoint of the ED channels of `extras` [P,ED] (extra_attrs; Skyfall-GS never passes them):
// phase 1 keeps the reference's per-pixel recursion of the extras and adds one global atomicAdd per (pixel, Gaussian,
// channel) into dL_dextras, so this instantiation is a slow path.
// ORDERED: no reduction at all.  The 16 words of a (block, record) pair go to row (range.x + list position) * 8 + wid
// of `part` [R*8,16] and written[row] is set; exactly one warp owns each row.  `acc` is not touched.  The slot's gid
// word carries the sorted instance range.x + list position instead of the Gaussian id (nothing else reads it here).
// JITTER: subpixel offsets — pixel (x, y) samples the splats at (x, y) + off[W y + x] ([H,W,2] floats, the buffer the
// forward used).  Phase 1 only moves the pixel; phase 2 sums h against each pixel's sample position about the half's
// centre (read from the warp's table `pos`), with the same centred origin.
// DIST: the depth distortion's adjoint (sfgs_rasterize_backward_distortion).  With c = dL/dR, A = the pixel's alpha and
// the forward's state (mu, M2): dR/dw_i = A (m_i - mu)^2 + M2 joins g, the record's dL/dw, so the recursion carries
// it to every alpha -- the M2 term is the same for every record and joins the alpha cotangent, the other is formed per
// slot from (2 c A, mu) in the warp's table `dist`; dR/dm_i = 2 A w_i (m_i - mu) joins the depth word (3) of phase 2,
// formed per (pixel, slot) as the difference m_i - mu.  With c = 0 every sum is what it is without the option.
// RAYD: ray depth (sfgs_rasterize_backward_ray_depth).  Phase 1 takes the record's depth at the pixel's sample
// position, d(p) = z + g . (p - mu) (g: the slope words, staged in quad [3].zw), as the depth attribute of g; phase 2
// adds the sums of w c (p - mu) over the record's pixels (c the pixel's depth cotangent), formed against the pixels'
// offsets from the half's centre and shifted to the record's centre by the expansion of the h-moments, into the free
// words 14-15.  Word 3 still sums w c.  With c = 0 every sum is what it is without the option.
template <bool PEER, bool HAS_EXTRA, bool ORDERED, bool JITTER, bool DIST, bool RAYD>
__device__ __forceinline__ void
render_bwd_warp(const uint2* __restrict__ ranges, const char* __restrict__ binning_base,
                const uint32_t* __restrict__ hdr, int W, int H, int band0,
                const float* __restrict__ bg_color, const float* __restrict__ rec,
                const float* __restrict__ accum_alphas, const uint32_t* __restrict__ n_contrib,
                const float* __restrict__ dL_dpixels, const float* __restrict__ dL_dpixel_depths,
                const float* __restrict__ dL_dpixel_norms, const float* __restrict__ dL_dpixel_alphas,
                const float* __restrict__ norm_raw, float* __restrict__ acc /* [P,16] zero-initialised */,
                const PeerTable peers, const float* __restrict__ extras,
                const float* __restrict__ dL_dpixel_extras, float* __restrict__ dL_dextras, int ED,
                float* __restrict__ part, unsigned char* __restrict__ written, const float2* __restrict__ off,
                const float* __restrict__ dist_state, const float* __restrict__ dL_dpix_dist) {
  using SmemBase = std::conditional_t<JITTER, WarpSmemJitter, WarpSmem>;
  using Smem = std::conditional_t<DIST, WarpSmemDist<SmemBase>, SmemBase>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  Smem& S = reinterpret_cast<Smem*>(smem_raw)[wid];

  // the binning buffer layout depends on the capacity the forward used; it is recorded in the image header
  const unsigned long long cap = ((unsigned long long)hdr[HDR_CAP_HI] << 32) | hdr[HDR_CAP_LO];
  const BinningLayout bl(const_cast<char*>(binning_base), (size_t)cap);
  const uint32_t* __restrict__ point_list = bl.point_list;
  const unsigned char* __restrict__ inst_mask = bl.inst_mask;

  const BlendPixel px(band0, W, H, wid, lane);
  const bool inside = px.inside;
  const uint32_t pix_id = px.id;
  float pixfx = px.x, pixfy = px.y;          // the sample position (the pixel centre without offsets)
  const size_t HW = (size_t)H * W;

  const uint2 range = ranges[px.tile];
  const int total = (int)(range.y - range.x);
  if (total == 0) return;

  const float T_final = inside ? (1 - accum_alphas[pix_id]) : 0;
  float T = T_final;
  const uint32_t last_contributor = inside ? n_contrib[pix_id] : 0;
  // records at 1-based list position > max(last_contributor) over the warp's block are never used by it
  uint32_t wmax = last_contributor;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  const int used = min((int)wmax, total);
  if (used == 0) return;            // warp-uniform; nothing below is block-wide

  float dLc0 = 0, dLc1 = 0, dLc2 = 0, dLd = 0, dLn0 = 0, dLn1 = 0, dLn2 = 0, dLa = 0;
  if (inside) {
    dLc0 = dL_dpixels[0 * HW + pix_id]; dLc1 = dL_dpixels[1 * HW + pix_id]; dLc2 = dL_dpixels[2 * HW + pix_id];
    dLd = dL_dpixel_depths[pix_id];
    dLn0 = dL_dpixel_norms[0 * HW + pix_id]; dLn1 = dL_dpixel_norms[1 * HW + pix_id]; dLn2 = dL_dpixel_norms[2 * HW + pix_id];
    dLa = dL_dpixel_alphas[pix_id];
    if (norm_raw != nullptr) {
      // dL_dpixel_norms is w.r.t. the unit normal y = x / max(|x|, eps): apply the adjoint of F.normalize here
      // (torch: g/d - [|x| >= eps] (g.x)/d^2 * x/|x|, d = max(|x|, eps))
      const float x0 = norm_raw[0 * HW + pix_id], x1 = norm_raw[1 * HW + pix_id], x2 = norm_raw[2 * HW + pix_id];
      const float n = sqrtf(x0 * x0 + x1 * x1 + x2 * x2);
      const float d = fmaxf(n, 1e-12f);
      const float gx = dLn0 * x0 + dLn1 * x1 + dLn2 * x2;
      float r0 = dLn0 / d, r1 = dLn1 / d, r2 = dLn2 / d;
      if (n >= 1e-12f) {
        const float s = gx / (d * d) / n;
        r0 -= s * x0; r1 -= s * x1; r2 -= s * x2;
      }
      dLn0 = r0; dLn1 = r1; dLn2 = r2;
    }
  }
  if constexpr (DIST) {
    float2 q = make_float2(0.f, 0.f);
    if (inside) {
      const float c = dL_dpix_dist[pix_id];
      dLa = fmaf(c, dist_state[HW + pix_id], dLa);
      q = make_float2(2.f * c * accum_alphas[pix_id], dist_state[pix_id]);
    }
    S.dist[lane] = q;
  }
  // background term of dL/dalpha: (-T_final / (1 - alpha)) * <bg, dL/dcolour>
  const float tb = -T_final * (bg_color[0] * dLc0 + bg_color[1] * dLc1 + bg_color[2] * dLc2);
  {
    float4* pt = reinterpret_cast<float4*>(&S.pix[lane][0]);
    pt[0] = make_float4(dLc0, dLc1, dLc2, dLd);
    // the free word: the centre of the lane's 8x2 half of the block, its x in even lanes and its y in odd ones;
    // phase 2 reads it from the half's pixels 0 and 1
    pt[1] = make_float4(dLn0, dLn1, dLn2, (lane & 1) ? pixfy - (float)((lane >> 3) & 1) + 0.5f
                                                     : pixfx - (float)(lane & 7) + 3.5f);
  }
  if constexpr (JITTER) {
    // the sample position goes to the warp's table: phase 2 reads every pixel's, phase 1 its own at each chunk (so it
    // is not held in registers across phase 2)
    const float2 o = inside ? off[pix_id] : make_float2(0.f, 0.f);
    S.pos[lane] = make_float2(px.x + o.x, px.y + o.y);
  }
  __syncwarp();

  // extras: the pixel's cotangents and the reference's recursion state (accum_ree = the extras' A, last_extra = g_last)
  float dL_dpixel_extra[HAS_EXTRA ? SFGS_MAX_EXTRA : 1];
  float accum_ree[HAS_EXTRA ? SFGS_MAX_EXTRA : 1];
  float last_extra[HAS_EXTRA ? SFGS_MAX_EXTRA : 1];
  if constexpr (HAS_EXTRA)
    for (int ch = 0; ch < ED; ch++) {
      dL_dpixel_extra[ch] = inside ? dL_dpixel_extras[ch * HW + pix_id] : 0.f;
      accum_ree[ch] = 0.f;
      last_extra[ch] = 0.f;
    }

  // C = the A of the next active record, advanced at each active record as C' = alpha g + (1 - alpha) C (the
  // reference keeps A, g_last and last_alpha and forms this only at the next record); last_alpha is kept for the
  // extras' recursion only
  float C = 0.f, last_alpha = 0.f;
  float dcA = 0.f, dmu = 0.f;                  // DIST: c A and mu, read from the warp's table at each chunk
  const SfgsExpConsts ek = sfgs_exp_consts(hdr[HDR_ZERO]);
  BlendWalk<true, ORDERED ? GID_INSTANCE : GID_GAUSSIAN> walk(S.st, inst_mask, point_list, rec, range, used, wid,
                                                               lane);

  // ---- phase 2: lane (k = lane & 15, half = lane >> 4) sums slot k of the chunk over pixels half*16 .. +15.  The
  // half is 8 x 2 pixels; in coordinates centred on it, its pixel i sits at the compile-time offset
  // (x, y) = ((i & 7) - 3.5, (i >> 3) - 0.5).  The loop sums h against those constants, and the moments about the
  // record's centre (dx = DX - x, dy = DY - y, where (DX, DY) = record centre - half centre) follow once per chunk
  // (see the numerics note at the top).
  const int ck = lane & (BLEND_CH - 1), chalf = lane >> 4;
  auto phase2 = [&](int buf, int n) {
    __syncwarp();
    const bool have_rec = ck < n;
    const int slot = have_rec ? ck : 0;          // idle lanes shadow slot 0 (always valid, n >= 1)
    const float4 ra = S.st.rec[buf][slot][0];   // mx, my, con.x, con.y
    const float4 rb = S.st.rec[buf][slot][1];   // con.z, opac, depth
    const uint32_t gid = S.st.gid[buf][slot];
    const float2* whp = &S.wh[chalf * 16][ck];
    const float4* pix = reinterpret_cast<const float4*>(&S.pix[chalf * 16][0]);
    // DIST: each pixel's depth cotangent for this record, dL/d depth + 2 c A (m - mu)
    const auto dLd_of = [&](const int i, const float dLd_i) {
      if constexpr (DIST) {
        const float2 q = S.dist[chalf * 16 + i];
        return fmaf(q.x, rb.z - q.y, dLd_i);
      } else {
        return dLd_i;
      }
    };
    const float DX = ra.x - pix[1].w, DY = ra.y - pix[3].w;
    // abs-gradient term |h| (|u| + |v|), u = (W/2)(con.x dx + con.y dy), v = (H/2)(con.y dx + con.z dy): affine in
    // the pixel offset, so each is one FFMA from its row's base.  au .. bv are the conic scaled by d(ndc)/d(pixel)
    // (W/2 or H/2; 0.5 con is exact)
    const float au = 0.5f * ra.z * W, bu = 0.5f * ra.w * W, av = 0.5f * ra.w * H, bv = 0.5f * rb.x * H;
    const float u0 = fmaf(au, DX, bu * DY), v0 = fmaf(av, DX, bv * DY);
    const float urow[2] = {fmaf(bu, 0.5f, u0), fmaf(bu, -0.5f, u0)}, vrow[2] = {fmaf(bv, 0.5f, v0), fmaf(bv, -0.5f, v0)};
    float s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0;      // sum w * dL/dpix_c
    float sab = 0;
    float sh, shx, shy, shxx, shxy, shyy;     // sums of h * {1, dx, dy, dx^2, dx dy, dy^2} over the half
    float sdx = 0, sdy = 0;                   // RAYD: sums of w c * {x, y} over the half (c: the depth cotangent)
    if constexpr (JITTER) {
      // pixel i samples at (x, y) = its sample position - the half's centre (exact: the two are close), i.e. its
      // compile-time offset plus its own subpixel offset: the sums of h * {1, x, y, x^2, x y, y^2} run over those, the
      // moments about the record's centre follow by the same expansion, and |u| + |v| is evaluated per pixel
      const float2* posp = &S.pos[chalf * 16];
      const float hcx = pix[1].w, hcy = pix[3].w;
      float sx = 0, sy = 0, sxx = 0, sxy = 0, syy = 0;
      sh = 0;
#pragma unroll 4                            // fully unrolled, the ORDERED instantiation spills
      for (int i = 0; i < 16; i++) {
        const float2 q = posp[i];
        const float x = q.x - hcx, y = q.y - hcy;
        const float2 wh = whp[i * (BLEND_CH + 1)];
        const float4 p0 = pix[2 * i], p1 = pix[2 * i + 1];
        s0 = fmaf(wh.x, p0.x, s0); s1 = fmaf(wh.x, p0.y, s1); s2 = fmaf(wh.x, p0.z, s2);
        s3 = fmaf(wh.x, dLd_of(i, p0.w), s3);
        s4 = fmaf(wh.x, p1.x, s4); s5 = fmaf(wh.x, p1.y, s5); s6 = fmaf(wh.x, p1.z, s6);
        if constexpr (RAYD) {
          const float wc = wh.x * p0.w;
          sdx = fmaf(wc, x, sdx); sdy = fmaf(wc, y, sdy);
        }
        const float hx = wh.y * x, hy = wh.y * y;
        sh += wh.y;
        sx += hx; sy += hy;
        sxx = fmaf(hx, x, sxx); sxy = fmaf(hx, y, sxy); syy = fmaf(hy, y, syy);
        const float u = fmaf(-au, x, fmaf(-bu, y, u0)), v = fmaf(-av, x, fmaf(-bv, y, v0));
        sab = fmaf(fabsf(wh.y), fabsf(u) + fabsf(v), sab);
      }
      shx = fmaf(DX, sh, -sx); shy = fmaf(DY, sh, -sy);
      shxx = fmaf(DX, shx, -fmaf(DX, sx, -sxx));
      shxy = fmaf(DX, shy, -fmaf(DY, sx, -sxy));
      shyy = fmaf(DY, shy, -fmaf(DY, sy, -syy));
    } else {
      float h1[2] = {0, 0}, hx[2] = {0, 0}, sxx = 0;                  // per row: sum h * {1, x}; sum h x^2
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const float x = (float)(i & 7) - 3.5f;
        const int r = i >> 3;
        const float2 wh = whp[i * (BLEND_CH + 1)];
        const float4 p0 = pix[2 * i], p1 = pix[2 * i + 1];
        s0 = fmaf(wh.x, p0.x, s0); s1 = fmaf(wh.x, p0.y, s1); s2 = fmaf(wh.x, p0.z, s2);
        s3 = fmaf(wh.x, dLd_of(i, p0.w), s3);
        s4 = fmaf(wh.x, p1.x, s4); s5 = fmaf(wh.x, p1.y, s5); s6 = fmaf(wh.x, p1.z, s6);
        if constexpr (RAYD) {
          const float wc = wh.x * p0.w;
          sdx = fmaf(wc, x, sdx); sdy = fmaf(wc, r ? 0.5f : -0.5f, sdy);
        }
        h1[r] += wh.y;
        hx[r] = fmaf(wh.y, x, hx[r]);
        sxx = fmaf(wh.y, x * x, sxx);
        const float u = fmaf(-au, x, urow[r]), v = fmaf(-av, x, vrow[r]);
        sab = fmaf(fabsf(wh.y), fabsf(u) + fabsf(v), sab);
      }
      // sums of h * {1, x, y, x^2, x y, y^2} over the half (y = -0.5 in row 0, +0.5 in row 1) ...
      sh = h1[0] + h1[1];
      const float sx = hx[0] + hx[1], sy = 0.5f * (h1[1] - h1[0]);
      const float sxy = 0.5f * (hx[1] - hx[0]), syy = 0.25f * sh;
      // ... and about the centre: sum h dx = DX sum h - sum h x, sum h dx^2 = DX sum h dx - (DX sum h x - sum h x^2), ...
      shx = fmaf(DX, sh, -sx); shy = fmaf(DY, sh, -sy);
      shxx = fmaf(DX, shx, -fmaf(DX, sx, -sxx));
      shxy = fmaf(DX, shy, -fmaf(DY, sx, -sxy));
      shyy = fmaf(DY, shy, -fmaf(DY, sy, -syy));
    }
    // RAYD: sum w c (p - mu) = sum w c (x - DX, y - DY) over the half, before the halves are added (DX, DY differ)
    float e14 = 0.f, e15 = 0.f;
    if constexpr (RAYD) {
      e14 = fmaf(-DX, s3, sdx);
      e15 = fmaf(-DY, s3, sdy);
    }
#define XH(v) v += __shfl_xor_sync(0xffffffffu, v, 16)
    XH(s0); XH(s1); XH(s2); XH(s3); XH(s4); XH(s5); XH(s6);
    XH(sh); XH(shx); XH(shy); XH(shxx); XH(shxy); XH(shyy); XH(sab);
    if constexpr (RAYD) { XH(e14); XH(e15); }
#undef XH
    if (ORDERED && have_rec) {
      const float o = rb.y;
      const size_t row = (size_t)gid * BLEND_WARPS + wid;
      float4* dst = reinterpret_cast<float4*>(part + row * 16);
      if (lane < 16) {
        dst[0] = make_float4(s0, s1, s2, s3);
        dst[1] = make_float4(s4, s5, s6, -o * fmaf(au, shx, bu * shy));
        written[row] = 1;
      } else {
        dst[2] = make_float4(-o * fmaf(bv, shy, av * shx), fabsf(o) * sab, -0.5f * o * shxx, -0.5f * o * shxy);
        dst[3] = make_float4(-0.5f * o * shyy, sh, e14, e15);
      }
    } else if (have_rec) {
      const float o = rb.y;
      float* dst;
      if (PEER) {   // the sums of Gaussian gid live on rank gid / per: the reduction itself is the reduce-scatter
        const uint32_t r = gid / (uint32_t)peers.per;
        dst = peers.p[r] + (size_t)(gid - r * (uint32_t)peers.per) * 16;
      } else {
        dst = acc + (size_t)gid * 16;
      }
      if (lane < 16) {
        red_add_v4<PEER>(dst, make_float4(s0, s1, s2, s3));
        red_add_v4<PEER>(dst + 4, make_float4(s4, s5, s6, -o * fmaf(au, shx, bu * shy)));
      } else {
        red_add_v4<PEER>(dst + 8, make_float4(-o * fmaf(bv, shy, av * shx), fabsf(o) * sab,
                                              -0.5f * o * shxx, -0.5f * o * shxy));
        red_add_v4<PEER>(dst + 12, make_float4(-0.5f * o * shyy, sh, e14, e15));
      }
    }
    __syncwarp();
  };

  // ---- phase 1: pixel-parallel recursion over the chunk's records, slot order = back to front.  Branch-free: a
  // chunk is one basic block, so the scheduler can overlap slot k+1's load -> exp chain with slot k's recursion (a
  // (block, record) pair that no pixel blends is 0.6 % of the pairs: the work a branch would skip is negligible, the
  // selects cost what the branch bookkeeping did)
  auto slot = [&](const int buf, const int k, const float4 ra /* mx, my, con.x, con.y */,
                  const float4 rb /* con.z, opac, depth, 1-based list position */) {
    const float dx = ra.x - pixfx, dy = ra.y - pixfy;
    const float power = -0.5f * (ra.z * dx * dx + rb.x * dy * dy) - ra.w * dx * dy;
    const float G = sfgs_expf(power, ek);
    const float alpha = min(0.99f, rb.y * G);
    const bool active = (__float_as_uint(rb.w) <= last_contributor) && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
    const float4 rc = S.st.rec[buf][k][2];    // r, g, b, nx
    const float4 rd = S.st.rec[buf][k][3];    // ny, nz
    // 1 - alpha is in [0.01, 1]: the approximate reciprocal (1 ulp, one MUFU) needs no range fix-up; it is shared
    // by the T recovery and the background term
    const float one_m_alpha = 1.f - alpha;
    float inv_1ma;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv_1ma) : "f"(one_m_alpha));
    const float Tn = T * inv_1ma;
    // two independent chains: halves the dependent-FMA latency of the dot product
    float g = rc.x * dLc0, g2 = rc.w * dLn0;
    g += rc.y * dLc1; g2 += rd.x * dLn1;
    g += rc.z * dLc2; g2 += rd.y * dLn2;
    g += (RAYD ? fmaf(-rd.z, dx, fmaf(-rd.w, dy, rb.z)) : rb.z) * dLd;  g2 += dLa;
    g += g2;
    if constexpr (DIST) {
      const float dm = rb.z - dmu;
      g = fmaf(dcA * dm, dm, g);
    }
    float dL_dalpha_T = g - C;                  // dL/dalpha / T
    if constexpr (HAS_EXTRA) {
      const uint32_t gid = S.st.gid[buf][k];
      for (int ch = 0; ch < ED; ch++) {
        const float ex = extras[(size_t)gid * ED + ch];
        const float ree = last_alpha * last_extra[ch] + (1.f - last_alpha) * accum_ree[ch];
        dL_dalpha_T += (ex - ree) * dL_dpixel_extra[ch];
        accum_ree[ch] = active ? ree : accum_ree[ch];
        last_extra[ch] = active ? ex : last_extra[ch];
        if (active) atomicAdd(&dL_dextras[(size_t)gid * ED + ch], alpha * Tn * dL_dpixel_extra[ch]);
      }
      last_alpha = active ? alpha : last_alpha;
    }
    const float dL_dalpha = fmaf(tb, inv_1ma, Tn * dL_dalpha_T);
    const float w_out = active ? alpha * Tn : 0.f;
    const float h_out = active ? G * dL_dalpha : 0.f;
    T = active ? Tn : T;
    // the roundings of forming A from (A, g_last, last_alpha) at the next record: (1 - alpha) * C, then one FMA
    C = active ? fmaf(alpha, g, __fmul_rn(one_m_alpha, C)) : C;
    S.wh[lane][k] = make_float2(w_out, h_out);
  };
  blend_chunks<ORDERED>(walk, [] { return false; }, [&](const int buf, const int n) {
    if constexpr (JITTER) {
      const float2 q = S.pos[lane];
      pixfx = q.x;
      pixfy = q.y;
    }
    if constexpr (DIST) {
      const float2 q = S.dist[lane];
      dcA = 0.5f * q.x;
      dmu = q.y;
    }
    if (n == BLEND_CH) {                            // every chunk of a warp but its last: no per-slot bound test
      // slot k+1's parameters are read before slot k's hand-over store (the compiler cannot move a shared-memory
      // load above that store on its own), so their latency overlaps slot k's arithmetic
      float4 ra_n = S.st.rec[buf][0][0], rb_n = S.st.rec[buf][0][1];
#pragma unroll
      for (int k = 0; k < BLEND_CH; k++) {
        const float4 ra = ra_n, rb = rb_n;
        if (k + 1 < BLEND_CH) { ra_n = S.st.rec[buf][k + 1][0]; rb_n = S.st.rec[buf][k + 1][1]; }
        slot(buf, k, ra, rb);
      }
    } else {
#pragma unroll 1
      for (int k = 0; k < n; k++) slot(buf, k, S.st.rec[buf][k][0], S.st.rec[buf][k][1]);
    }
    phase2(buf, n);
  });
}

// The one blend adjoint.  Each option is a template argument; a trailing parameter an instantiation does not read costs
// nothing, and new parameters go at the end of the list.  GUARDED (the graph backward, sfgs_rasterize_backward_graph):
// launched whatever the frame's instance count, so it first checks the forward's overflow flag -- after an overflow the
// ranges run past the binning capacity and nothing may read point_list or write partial rows.
// DIST (the depth distortion) is instantiated only without peers, extras and GUARDED, at two CTAs per SM: at the 80
// registers of three its instantiations spilled (8 to 20 bytes).  RAYD (ray depth) likewise without peers, extras,
// GUARDED and DIST: at three CTAs per SM without jitter (80 registers, no spills) and at two with it (the two jitter
// instantiations spilled 4 bytes at 80 registers).
template <bool PEER, bool HAS_EXTRA, bool ORDERED, bool JITTER, bool GUARDED, bool DIST, bool RAYD = false>
__global__ void __launch_bounds__(BLEND_THREADS, DIST || (RAYD && JITTER) ? 2 : 3)
render_bwd_kernel(const uint2* __restrict__ ranges, const char* __restrict__ binning_base,
                  const uint32_t* __restrict__ hdr, int W, int H, int band0,
                  const float* __restrict__ bg_color, const float* __restrict__ rec,
                  const float* __restrict__ accum_alphas, const uint32_t* __restrict__ n_contrib,
                  const float* __restrict__ dL_dpixels, const float* __restrict__ dL_dpixel_depths,
                  const float* __restrict__ dL_dpixel_norms, const float* __restrict__ dL_dpixel_alphas,
                  const float* __restrict__ norm_raw, float* __restrict__ acc /* [P,16] zero-initialised */,
                  const PeerTable peers, const float* __restrict__ extras,
                  const float* __restrict__ dL_dpixel_extras, float* __restrict__ dL_dextras, int ED,
                  float* __restrict__ part, unsigned char* __restrict__ written, const float2* __restrict__ off,
                  const float* __restrict__ dist_state, const float* __restrict__ dL_dpix_dist) {
  if (GUARDED && hdr[HDR_OVERFLOW]) return;
  render_bwd_warp<PEER, HAS_EXTRA, ORDERED, JITTER, DIST, RAYD>(ranges, binning_base, hdr, W, H, band0, bg_color, rec,
                                                          accum_alphas, n_contrib, dL_dpixels, dL_dpixel_depths,
                                                          dL_dpixel_norms, dL_dpixel_alphas, norm_raw, acc, peers,
                                                          extras, dL_dpixel_extras, dL_dextras, ED, part, written, off,
                                                          dist_state, dL_dpix_dist);
}

template <bool JITTER, bool DIST>
constexpr size_t render_bwd_smem() {
  using Base = std::conditional_t<JITTER, WarpSmemJitter, WarpSmem>;
  return BLEND_WARPS * sizeof(std::conditional_t<DIST, WarpSmemDist<Base>, Base>);
}

template <bool PEER, bool HAS_EXTRA, bool ORDERED, bool JITTER, bool GUARDED, bool DIST = false, bool RAYD = false>
auto render_bwd_instance() {
  return sfgs_smem_kernel<render_bwd_kernel<PEER, HAS_EXTRA, ORDERED, JITTER, GUARDED, DIST, RAYD>>(
      render_bwd_smem<JITTER, DIST>());
}

// The adjoint of the depth quantile (sfgs_rasterize_backward_depth_quantile): dL/d depth_j += dL/d depth_q[p] for the
// record j each pixel p selected, into the depth word (3) of the per-Gaussian sums.  It runs after the blend adjoint,
// with that kernel's grid and pixel mapping: warp w of a CTA is the 8x4 block w of the tile (point_list sits at the head
// of the binning layout, so its address does not depend on the capacity).  Lanes that selected the
// same list position are grouped, and the group's first lane adds their cotangents in increasing lane order and
// makes one update:
//   default  one red.global.add.f32 into acc[gid * 16 + 3], gid = point_list[range.x + pos - 1];
//   ORDERED  a plain read-modify-write of word 3 of the partial row (range.x + pos - 1) * 8 + w that the ORDERED blend
//            adjoint wrote.  That row exists: the selected record was applied at one of the block's pixels, so the
//            block's bit of its reach mask is set and its position is <= the block's largest n_contrib.  Exactly one
//            warp owns a row, so the sums stay bit-reproducible.
// Kept out of render_bwd_kernel, which is bound by instruction issue at its register budget: this costs one launch and
// 8 bytes read per pixel.
// RAYD: ray depth, where depth_q = d_j(p) = z_j + g_j . (p - mu_j): each lane also forms c (p - mu_j) at its sample
// position p (off: the forward's offsets, or NULL), and the group's first lane adds those in the same order into words
// 14-15 (dL/dg) beside word 3; the dL/dmu = -g dL/dz part follows in the per-Gaussian adjoint.
template <bool ORDERED, bool RAYD = false>
__global__ void __launch_bounds__(BLEND_THREADS)
depth_q_adjoint_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H,
                       int band0,
                       const uint32_t* __restrict__ depth_q_pos, const float* __restrict__ dL_dpix_depth_q,
                       float* __restrict__ acc, float* __restrict__ part, const float* __restrict__ rec,
                       const float2* __restrict__ off) {
  __shared__ float s_g[BLEND_WARPS][32];
  __shared__ float2 s_gp[RAYD ? BLEND_WARPS : 1][32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const BlendPixel px(band0, W, H, wid, lane);
  const uint32_t pos = px.inside ? depth_q_pos[px.id] : 0u;
  s_g[wid][lane] = px.inside ? dL_dpix_depth_q[px.id] : 0.f;
  if constexpr (RAYD) {
    float2 v = make_float2(0.f, 0.f);
    if (pos != 0) {
      const float* r = rec + (size_t)point_list[ranges[px.tile].x + pos - 1] * REC_FLOATS;
      const float2 o = off != nullptr ? off[px.id] : make_float2(0.f, 0.f);
      const float c = s_g[wid][lane];
      v = make_float2(c * ((px.x + o.x) - r[0]), c * ((px.y + o.y) - r[1]));
    }
    s_gp[wid][lane] = v;
  }
  const unsigned group = __match_any_sync(0xffffffffu, pos);
  __syncwarp();
  if (pos == 0 || lane != __ffs(group) - 1) return;
  float s = 0.f, sx = 0.f, sy = 0.f;
  for (unsigned m = group; m != 0; m &= m - 1) {
    s += s_g[wid][__ffs(m) - 1];
    if constexpr (RAYD) { sx += s_gp[wid][__ffs(m) - 1].x; sy += s_gp[wid][__ffs(m) - 1].y; }
  }
  const uint32_t inst = ranges[px.tile].x + pos - 1;
  if (ORDERED) {
    part[((size_t)inst * BLEND_WARPS + wid) * 16 + 3] += s;
    if constexpr (RAYD) {
      part[((size_t)inst * BLEND_WARPS + wid) * 16 + 14] += sx;
      part[((size_t)inst * BLEND_WARPS + wid) * 16 + 15] += sy;
    }
  } else {
    float* dst = acc + (size_t)point_list[inst] * 16 + 3;
    asm volatile("red.global.add.f32 [%0], %1;\n" ::"l"(dst), "f"(s) : "memory");
    if constexpr (RAYD) {
      asm volatile("red.global.add.f32 [%0], %1;\n" ::"l"(dst + 11), "f"(sx) : "memory");
      asm volatile("red.global.add.f32 [%0], %1;\n" ::"l"(dst + 12), "f"(sy) : "memory");
    }
  }
}

}  // namespace

// After the blend adjoint: part != NULL for the ORDERED (deterministic) backward, whose partial rows it updates;
// ray_depth: the ray-depth form, which reads the records and the offsets (off, or NULL)
void sfgs_launch_depth_q_adjoint(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                                 const BinningLayout& b, const uint32_t* depth_q_pos, const float* dL_dpix_depth_q,
                                 float* acc, float* part, bool ray_depth, const float* off, cudaStream_t st) {
  dim3 grid;
  int band0;
  if (!blend_grid(a->tile_row_begin, a->tile_row_end, im, grid, band0)) return;
  const auto kernel = ray_depth ? (part != nullptr ? depth_q_adjoint_kernel<true, true>
                                                   : depth_q_adjoint_kernel<false, true>)
                      : part != nullptr ? depth_q_adjoint_kernel<true> : depth_q_adjoint_kernel<false>;
  SFGS_COUNT_LAUNCH();
  kernel<<<grid, BLEND_THREADS, 0, st>>>(im.ranges, b.point_list, a->width, a->height, band0, depth_q_pos,
                                         dL_dpix_depth_q, acc, part, g.rec, reinterpret_cast<const float2*>(off));
}

// guarded: the graph backward's blend adjoint.  The entry points' checks leave these combinations: peers only in the
// eager non-deterministic backward; extra_attrs only without offsets and without the ordered form (part != nullptr);
// the depth distortion (dist_state != nullptr) and ray depth (ray_depth) only eager, without peers and extra_attrs,
// and not together.
void sfgs_launch_render_bwd(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, float* acc, float* part, unsigned char* written, const float* off,
                            bool guarded, const float* dist_state, const float* dL_dpix_dist, bool ray_depth,
                            cudaStream_t st) {
  dim3 grid;
  int band0;
  if (!blend_grid(a->tile_row_begin, a->tile_row_end, im, grid, band0)) return;
  PeerTable pt = {};
  const bool peer = a->acc_peers != nullptr && a->n_peers > 0;
  if (peer) {
    for (int r = 0; r < a->n_peers && r < 8; r++) pt.p[r] = a->acc_peers[r];
    pt.per = a->peer_slice;
  }
  const bool ordered = part != nullptr, extra = a->ED > 0, dist = dist_state != nullptr;
  // render_bwd_instance<PEER, HAS_EXTRA, ORDERED, JITTER, GUARDED[, DIST]>
  const auto kernel =
      ray_depth ? (off != nullptr ? (ordered ? render_bwd_instance<false, false, true, true, false, false, true>()
                                             : render_bwd_instance<false, false, false, true, false, false, true>())
                   : ordered      ? render_bwd_instance<false, false, true, false, false, false, true>()
                                  : render_bwd_instance<false, false, false, false, false, false, true>())
      : dist ? (off != nullptr ? (ordered ? render_bwd_instance<false, false, true, true, false, true>()
                                        : render_bwd_instance<false, false, false, true, false, true>())
              : ordered      ? render_bwd_instance<false, false, true, false, false, true>()
                             : render_bwd_instance<false, false, false, false, false, true>())
      : guarded ? (off != nullptr ? (ordered ? render_bwd_instance<false, false, true, true, true>()
                                           : render_bwd_instance<false, false, false, true, true>())
                 : ordered      ? render_bwd_instance<false, false, true, false, true>()
                 : extra        ? render_bwd_instance<false, true, false, false, true>()
                                : render_bwd_instance<false, false, false, false, true>())
      : off != nullptr ? (peer      ? render_bwd_instance<true, false, false, true, false>()
                          : ordered ? render_bwd_instance<false, false, true, true, false>()
                                    : render_bwd_instance<false, false, false, true, false>())
      : ordered ? render_bwd_instance<false, false, true, false, false>()
      : extra   ? render_bwd_instance<false, true, false, false, false>()
      : peer    ? render_bwd_instance<true, false, false, false, false>()
                : render_bwd_instance<false, false, false, false, false>();
  const size_t smem = off != nullptr ? (dist ? render_bwd_smem<true, true>() : render_bwd_smem<true, false>())
                                      : (dist ? render_bwd_smem<false, true>() : render_bwd_smem<false, false>());
  SFGS_COUNT_LAUNCH();
  kernel<<<grid, BLEND_THREADS, smem, st>>>(im.ranges, (const char*)b.point_list, im.hdr, a->width, a->height, band0,
                                          a->background, g.rec, a->accum_alphas, im.n_contrib, a->dL_dpix,
                                          a->dL_dpix_depth, a->dL_dpix_norm, a->dL_dpix_alpha, a->norm_raw, acc, pt,
                                          a->extra_attrs, a->dL_dpix_extra, a->dL_dextra, a->ED, part, written,
                                          reinterpret_cast<const float2*>(off), dist_state, dL_dpix_dist);
}
