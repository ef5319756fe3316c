// sfgs_render_bwd.cu — adjoint of the alpha compositing, one CTA per 16x16 tile.
//
// Replaces BACKWARD::render / renderCUDA (RAST/cuda_rasterizer/backward.cu:509-754), which issues >= 14
// global float atomicAdd per (pixel, Gaussian) pair.
//
// Each warp owns an 8x4 pixel block and runs its own pipeline; nothing in the kernel is block-wide:
//
//   scan     the warp walks the tile's sorted list back to front 32 positions at a time (one coalesced read of the
//            reach masks, see sfgs_common.cuh), keeps the positions whose mask has ITS block's bit (ballot + prefix
//            popcount into a small ring), and as soon as 16 are collected gathers exactly those 16 records (two lanes
//            per 64-byte record, cp.async) into its private double-buffered chunk slot — while the previous chunk is
//            being processed;
//   phase 1  pixel-parallel (lane = pixel): the per-pixel recursion over the chunk's records in slot order.  The
//            reference's eight per-channel accumulators collapse into the scalar form
//                dL/dalpha_j = T_j (g_j - A_j),  g_j = <dL/dpix, attr_j>,  A_j = a_{j+1} g_{j+1} + (1 - a_{j+1}) A_{j+1}
//            (the channel-sum of accum_rec/accum_red/accum_ren/accum_rea, backward.cu:660-711).  Per pair only two
//            numbers leave the lane:  w = alpha*T  and  h = G * dL/dalpha ; they are parked in a per-warp
//            shared-memory tile [pixel][slot].  Slot k is a compile-time constant after unrolling, so record
//            parameters, list position and the (w, h) hand-over all sit at immediate offsets;
//   phase 2  record-parallel (lane = slot of the chunk x half of the block's pixels): all 14 per-Gaussian sums are
//            linear in (w, h):
//                sum w*dL/dpix_c (7 channels),  sum h*{1, dx, dy, dx^2, dx dy, dy^2},  sum |..| for the abs-gradient,
//            so each lane streams down its record's column of the tile accumulating in registers — no cross-lane
//            reduction except one 16-lane exchange between the two pixel halves;
//   combine  each (block, record) pair ends in four red.global.add.v4.f32 (tools/red_bench.cu times such traffic on
//            its own; the ~16 M issued per frame hide behind the math): ~200x fewer global atomics than the reference.
//
// Chunks are always full except the last one of a warp.  A record that none of the warp's 32 pixels blends (0.6 % on
// the benchmark frame: the reach mask is conservative) occupies a slot with zeros.
// (T is recovered back to front as T_j = T_{j+1} * rcp.approx(1 - alpha_{j+1}).  Refining the reciprocal with a Newton step
// costs time and does NOT change the error statistics against the float64 adjudicator — the worst elements are
// summation-order noise of ill-conditioned sums, which vary by 5x between runs of either implementation, not T drift.)
#include "sfgs_common.cuh"

namespace {

constexpr int BWD_THREADS = 256;
constexpr int BWD_WARPS = BWD_THREADS / 32;
constexpr int PIXF = 12;          // floats per pixel-table row: dLc[3], dLd, dLn[3], px, py, pad[3]

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

constexpr int W4_CH = 16;
struct alignas(16) WarpSmem {
  float4 rec[2][W4_CH][4];      // 2 KB   the chunk's blend records, double buffered; the free word [1].w of a staged
                                //        record carries its list position (bits of a uint32)
  uint32_t gid[2][W4_CH];       // Gaussian id of each slot
  float2 wh[32][W4_CH + 1];     // 4.25 KB phase-1 -> phase-2 hand-over, [pixel][slot], padded
  float pix[32][PIXF];          // 1.5 KB  per-pixel cotangents and coordinates
  uint32_t list[64];            // ring of collected list positions
};

// HAS_EXTRA: also the adjoint of the ED channels of `extras` [P,ED] (extra_attrs; Skyfall-GS never passes them):
// phase 1 keeps the reference's per-pixel recursion of the extras and adds one global atomicAdd per (pixel, Gaussian,
// channel) into dL_dextras, so this instantiation is a slow path.
template <bool PEER, bool HAS_EXTRA>
__global__ void __launch_bounds__(BWD_THREADS, 3)
render_bwd_warp_kernel(const uint2* __restrict__ ranges, const char* __restrict__ binning_base,
                       const uint32_t* __restrict__ hdr, int W, int H, int band0,
                       const float* __restrict__ bg_color, const float* __restrict__ rec,
                       const float* __restrict__ accum_alphas, const uint32_t* __restrict__ n_contrib,
                       const float* __restrict__ dL_dpixels, const float* __restrict__ dL_dpixel_depths,
                       const float* __restrict__ dL_dpixel_norms, const float* __restrict__ dL_dpixel_alphas,
                       const float* __restrict__ norm_raw, float* __restrict__ acc /* [P,16] zero-initialised */,
                       const PeerTable peers, const float* __restrict__ extras,
                       const float* __restrict__ dL_dpixel_extras, float* __restrict__ dL_dextras, int ED) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  WarpSmem& S = reinterpret_cast<WarpSmem*>(smem_raw)[wid];

  // the binning buffer layout depends on the capacity the forward used; it is recorded in the image header
  const unsigned long long cap = ((unsigned long long)hdr[HDR_CAP_HI] << 32) | hdr[HDR_CAP_LO];
  const BinningLayout bl(const_cast<char*>(binning_base), (size_t)cap);
  const uint32_t* __restrict__ point_list = bl.point_list;
  const unsigned char* __restrict__ inst_mask = bl.inst_mask;

  const int tiles_x = (W + SFGS_TILE - 1) / SFGS_TILE;
  const int tile_y = blockIdx.y + band0;
  const int tile = tile_y * tiles_x + blockIdx.x;
  const int px = blockIdx.x * SFGS_TILE + (wid & 1) * 8 + (lane & 7);
  const int py = tile_y * SFGS_TILE + (wid >> 1) * 4 + (lane >> 3);
  const bool inside = px < W && py < H;
  const uint32_t pix_id = (uint32_t)W * py + px;
  const float pixfx = (float)px, pixfy = (float)py;
  const size_t HW = (size_t)H * W;

  const uint2 range = ranges[tile];
  const int total = (int)(range.y - range.x);
  if (total == 0) return;

  const float T_final = inside ? (1 - accum_alphas[pix_id]) : 0;
  float T = T_final;
  const uint32_t last_contributor = inside ? n_contrib[pix_id] : 0;
  // records at list position >= max(last_contributor) over the warp's block are never used by it
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
  // background term of dL/dalpha: (-T_final / (1 - alpha)) * <bg, dL/dcolour>
  const float tb = -T_final * (bg_color[0] * dLc0 + bg_color[1] * dLc1 + bg_color[2] * dLc2);
  {
    float4* pt = reinterpret_cast<float4*>(&S.pix[lane][0]);
    pt[0] = make_float4(dLc0, dLc1, dLc2, dLd);
    pt[1] = make_float4(dLn0, dLn1, dLn2, pixfx);
    pt[2] = make_float4(pixfy, 0.f, 0.f, 0.f);
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

  float A = 0.f, g_last = 0.f, last_alpha = 0.f;
  const float ddelx_dx = 0.5 * W;
  const float ddely_dy = 0.5 * H;
  const SfgsExpConsts ek = sfgs_exp_consts(hdr[HDR_ZERO]);
  const unsigned lt_mask = (1u << lane) - 1u;

  // ---- scan + gather of the next chunk into buffer `buf`; returns the number of records in it (0 = list exhausted)
  int p = used;                    // positions [0, p) are still unscanned; the next window is p-1 ... p-32
  int head = 0, have = 0;          // ring of collected positions: [head, head + have)
  auto scan_gather = [&](int buf) -> int {
    while (have < W4_CH && p > 0) {
      const int pos = p - 1 - lane;
      unsigned m = 0;
      if (pos >= 0) m = inst_mask[range.x + pos];
      const bool bit = (m >> wid) & 1u;
      const unsigned b = __ballot_sync(0xffffffffu, bit);
      if (bit) S.list[(head + have + __popc(b & lt_mask)) & 63] = (uint32_t)pos;   // lane 0 = highest position first
      have += __popc(b);
      p -= 32;
    }
    __syncwarp();
    const int n = min(have, W4_CH);
    if (lane < 2 * n) {              // two lanes per 64-byte record
      const int r = lane >> 1, hf = lane & 1;
      const uint32_t pos = S.list[(head + r) & 63];
      const uint32_t id = point_list[range.x + pos];
      const float* src = rec + (size_t)id * REC_FLOATS;
      // the record's second quad is (con.z, opacity, depth, free): it is copied as 8 + 4 bytes and the free word takes
      // the list position, so phase 1 finds every per-record value it needs at an immediate offset of one base
      if (hf == 0) {
        cp_async16(&S.rec[buf][r][0], src);
        cp_async16(&S.rec[buf][r][2], src + 8);
        S.gid[buf][r] = id;
      } else {
        cp_async16(&S.rec[buf][r][3], src + 12);
        cp_async8(&S.rec[buf][r][1], src + 4);
        cp_async4(&S.rec[buf][r][1].z, src + 6);
        S.rec[buf][r][1].w = __uint_as_float(pos);
      }
    }
    cp_async_commit();
    head = (head + n) & 63;
    have -= n;
    return n;
  };

  // ---- phase 2: lane (k = lane & 15, half = lane >> 4) sums slot k of the chunk over pixels half*16 .. +15
  const int ck = lane & (W4_CH - 1), chalf = lane >> 4;
  auto phase2 = [&](int n, int buf) {
    __syncwarp();
    const bool have_rec = ck < n;
    const int slot = have_rec ? ck : 0;          // idle lanes shadow slot 0 (always valid, n >= 1)
    const float4 ra = S.rec[buf][slot][0];      // mx, my, con.x, con.y
    const float4 rb = S.rec[buf][slot][1];      // con.z, opac, depth
    const uint32_t gid = S.gid[buf][slot];
    float s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0;      // sum w * dL/dpix_c
    float sh = 0, shx = 0, shy = 0, shxx = 0, shxy = 0, shyy = 0, sab = 0;
    const int pbase = chalf * 16;
#pragma unroll 4
    for (int i = 0; i < 16; i++) {
      const float2 wh = S.wh[pbase + i][ck];
      const float4 p0 = *reinterpret_cast<const float4*>(&S.pix[pbase + i][0]);
      const float4 p1 = *reinterpret_cast<const float4*>(&S.pix[pbase + i][4]);
      const float pyv = S.pix[pbase + i][8];
      s0 = fmaf(wh.x, p0.x, s0); s1 = fmaf(wh.x, p0.y, s1); s2 = fmaf(wh.x, p0.z, s2); s3 = fmaf(wh.x, p0.w, s3);
      s4 = fmaf(wh.x, p1.x, s4); s5 = fmaf(wh.x, p1.y, s5); s6 = fmaf(wh.x, p1.z, s6);
      const float dx = ra.x - p1.w, dy = ra.y - pyv;
      const float hx = wh.y * dx, hy = wh.y * dy;
      sh += wh.y; shx += hx; shy += hy;
      shxx = fmaf(hx, dx, shxx); shxy = fmaf(hx, dy, shxy); shyy = fmaf(hy, dy, shyy);
      const float t7 = fmaf(ra.z, hx, ra.w * hy), t8 = fmaf(rb.x, hy, ra.w * hx);
      sab = fmaf(fabsf(t7), ddelx_dx, sab); sab = fmaf(fabsf(t8), ddely_dy, sab);
    }
#define XH(v) v += __shfl_xor_sync(0xffffffffu, v, 16)
    XH(s0); XH(s1); XH(s2); XH(s3); XH(s4); XH(s5); XH(s6);
    XH(sh); XH(shx); XH(shy); XH(shxx); XH(shxy); XH(shyy); XH(sab);
#undef XH
    if (have_rec) {
      const float o = rb.y;
      float* dst;
      if (PEER) {   // the sums of Gaussian gid live on rank gid / per: the reduction itself is the reduce-scatter
        const uint32_t r = gid / (uint32_t)peers.per;
        dst = peers.p[r] + (size_t)(gid - r * (uint32_t)peers.per) * 16;
      } else {
        dst = acc + (size_t)gid * 16;
      }
      if (chalf == 0) {
        red_add_v4<PEER>(dst, make_float4(s0, s1, s2, s3));
        red_add_v4<PEER>(dst + 4, make_float4(s4, s5, s6, -ddelx_dx * o * fmaf(ra.z, shx, ra.w * shy)));
      } else {
        red_add_v4<PEER>(dst + 8, make_float4(-ddely_dy * o * fmaf(rb.x, shy, ra.w * shx), fabsf(o) * sab,
                                              -0.5f * o * shxx, -0.5f * o * shxy));
        red_add_v4<PEER>(dst + 12, make_float4(-0.5f * o * shyy, sh, 0.f, 0.f));
      }
    }
    __syncwarp();
  };

  int buf = 0;
  int n_cur = scan_gather(0);
  while (n_cur > 0) {
    cp_async_wait_all();
    __syncwarp();                                   // chunk `buf` has landed and is visible to the whole warp
    const int n_next = scan_gather(buf ^ 1);        // the next chunk's gather overlaps the math below
    // ---- phase 1: pixel-parallel recursion over the chunk's records, slot order = back to front.  Branch-free: a
    // chunk is one basic block, so the scheduler can overlap slot k+1's load -> exp chain with slot k's recursion (a
    // (block, record) pair that no pixel blends is 0.6 % of the pairs: the work a branch would skip is negligible, the
    // selects cost what the branch bookkeeping did)
    auto slot_body = [&](const int k, const float4 ra, const float4 rb) {
      const float dx = ra.x - pixfx, dy = ra.y - pixfy;
      const float power = -0.5f * (ra.z * dx * dx + rb.x * dy * dy) - ra.w * dx * dy;
      const float G = sfgs_expf(power, ek);
      const float alpha = min(0.99f, rb.y * G);
      const bool active = (__float_as_uint(rb.w) < last_contributor) && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
      const float4 rc = S.rec[buf][k][2];       // r, g, b, nx
      const float4 rd = S.rec[buf][k][3];       // ny, nz
      // 1 - alpha is in [0.01, 1]: the approximate reciprocal (1 ulp, one MUFU) needs no range fix-up; it is shared
      // by the T recovery and the background term
      float inv_1ma;
      asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv_1ma) : "f"(1.f - alpha));
      const float Tn = T * inv_1ma;
      // two independent chains: halves the dependent-FMA latency of the dot product
      float g = rc.x * dLc0, g2 = rc.w * dLn0;
      g += rc.y * dLc1; g2 += rd.x * dLn1;
      g += rc.z * dLc2; g2 += rd.y * dLn2;
      g += rb.z * dLd;  g2 += dLa;
      g += g2;
      const float An = last_alpha * g_last + (1.f - last_alpha) * A;
      float dL_dalpha_T = g - An;                 // dL/dalpha / T
      if constexpr (HAS_EXTRA) {
        const uint32_t gid = S.gid[buf][k];
        for (int ch = 0; ch < ED; ch++) {
          const float ex = extras[(size_t)gid * ED + ch];
          const float ree = last_alpha * last_extra[ch] + (1.f - last_alpha) * accum_ree[ch];
          dL_dalpha_T += (ex - ree) * dL_dpixel_extra[ch];
          accum_ree[ch] = active ? ree : accum_ree[ch];
          last_extra[ch] = active ? ex : last_extra[ch];
          if (active) atomicAdd(&dL_dextras[(size_t)gid * ED + ch], alpha * Tn * dL_dpixel_extra[ch]);
        }
      }
      const float dL_dalpha = fmaf(tb, inv_1ma, Tn * dL_dalpha_T);
      const float w_out = active ? alpha * Tn : 0.f;
      const float h_out = active ? G * dL_dalpha : 0.f;
      T = active ? Tn : T;
      A = active ? An : A;
      g_last = active ? g : g_last;
      last_alpha = active ? alpha : last_alpha;
      S.wh[lane][k] = make_float2(w_out, h_out);
    };
    auto slot = [&](const int k) {
      slot_body(k, S.rec[buf][k][0] /* mx, my, con.x, con.y */, S.rec[buf][k][1] /* con.z, opac, depth, list position */);
    };
    if (n_cur == W4_CH) {                           // every chunk of a warp but its last: no per-slot bound test
      // slot k+1's parameters are read before slot k's hand-over store (the compiler cannot move a shared-memory
      // load above that store on its own), so their latency overlaps slot k's arithmetic
      float4 ra_n = S.rec[buf][0][0], rb_n = S.rec[buf][0][1];
#pragma unroll
      for (int k = 0; k < W4_CH; k++) {
        const float4 ra = ra_n, rb = rb_n;
        if (k + 1 < W4_CH) { ra_n = S.rec[buf][k + 1][0]; rb_n = S.rec[buf][k + 1][1]; }
        slot_body(k, ra, rb);
      }
    } else {
#pragma unroll 1
      for (int k = 0; k < n_cur; k++) slot(k);
    }
    phase2(n_cur, buf);
    buf ^= 1;
    n_cur = n_next;
  }
}

}  // namespace

void sfgs_launch_render_bwd(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, float* acc, cudaStream_t st) {
  const SfgsBand band = sfgs_band(a->tile_row_begin, a->tile_row_end, im.tiles_y);
  const int band0 = band.b0, band1 = band.b1;
  if (band1 <= band0) return;
  dim3 grid(im.tiles_x, band1 - band0, 1);
  const size_t smem = sizeof(WarpSmem) * BWD_WARPS;
  static SfgsPerDeviceOnce attr_once;   // function attributes are per device
  if (attr_once.first_use()) {
    cudaFuncSetAttribute(render_bwd_warp_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(render_bwd_warp_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(render_bwd_warp_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  PeerTable pt = {};
  const bool peer = a->acc_peers != nullptr && a->n_peers > 0;
  if (peer) {
    for (int r = 0; r < a->n_peers && r < 8; r++) pt.p[r] = a->acc_peers[r];
    pt.per = a->peer_slice;
  }
  // peer reductions belong to the two-phase backward, which rejects extra_attrs (sfgs_rasterize_backward)
  const auto kernel = a->ED > 0 ? render_bwd_warp_kernel<false, true>
                      : peer    ? render_bwd_warp_kernel<true, false>
                                : render_bwd_warp_kernel<false, false>;
  SFGS_COUNT_LAUNCH();
  kernel<<<grid, BWD_THREADS, smem, st>>>(im.ranges, (const char*)b.point_list, im.hdr, a->width, a->height, band0,
                                          a->background, g.rec, a->accum_alphas, im.n_contrib, a->dL_dpix,
                                          a->dL_dpix_depth, a->dL_dpix_norm, a->dL_dpix_alpha, a->norm_raw, acc, pt,
                                          a->extra_attrs, a->dL_dpix_extra, a->dL_dextra, a->ED);
}
