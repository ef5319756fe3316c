// sfgs_render_fwd.cu — front-to-back alpha compositing, one CTA per 16x16 tile.
//
// Replaces FORWARD::render / renderCUDA (RAST/cuda_rasterizer/forward.cu:333-468).
// Semantics kept exactly: pixel centres at integer coordinates, `power > 0`
// skip, alpha = min(0.99, o*exp(power)), alpha < 1/255 skip, stop when
// T*(1-alpha) < 1e-4 (that Gaussian is not applied), `contributor` counts every
// tested entry, n_contrib = index of the last applied entry, colour gets
// T*background, depth/normal/alpha have zero background.
//
// Mapping: each warp owns an 8x4 pixel block; the tile's sorted Gaussian
// list is streamed through a 2-stage cp.async ring of packed 64-byte blend
// records, so the inner loop touches shared memory only (the reference gathers
// colour/depth/normal from global memory per pixel).  Each record carries the
// reach mask computed by the sort stage; a warp walks only the records whose
// alpha >= 1/255 ellipse can touch its block (bit lists built with ballots), which
// removes ~80% of the (pixel, Gaussian) evaluations without changing any result.
#include "sfgs_common.cuh"
#include <cstdlib>

namespace {

constexpr int FWD_THREADS = 256;
constexpr int FWD_BATCH = 256;   // records per stage (one staging thread per record)
constexpr int FWD_STAGES = 2;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// ---- optional TMA staging: one bulk copy (cp.async.bulk, SASS UBLKCP) per 64-byte blend record, completion by
// mbarrier (each staging warp posts its byte count with one arrive.expect_tx; the phase completes when all eight
// warps have arrived and all announced bytes have landed).  Parity-green, but a uniform-datapath bulk copy per record
// means a warp whose 32 lanes gather 32 scattered records issues 32 serialised bulk copies where LDGSTS issues 4
// vector instructions.  TMA pays for
// tiles, not for 64-byte gathers — the default stays cp.async; build with -DSFGS_TMA_STAGING=1 to reproduce.
#ifndef SFGS_TMA_STAGING
#define SFGS_TMA_STAGING 0
#endif
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(a), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(a) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_64(void* smem, const void* gmem, unsigned long long* bar) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem), b = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 64, [%2];\n"
               ::"r"(d), "l"(gmem), "r"(b) : "memory");
}

// peer-mapped [8,H,W] frame blocks of the ranks of one node (sfgs_forward_args.out_peers); n == 0: local outputs
struct OutPeers {
  float* p[8];
  int n;
};

template <bool HAS_EXTRA>
__global__ void __launch_bounds__(FWD_THREADS)
render_fwd_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                  const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H, int ED,
                  int band0,
                  const float* __restrict__ rec, const float* __restrict__ extras,
                  const float* __restrict__ bg_color, float* __restrict__ out_color,
                  float* __restrict__ out_depth, float* __restrict__ out_norm, float* __restrict__ out_norm_raw,
                  float* __restrict__ out_alpha, float* __restrict__ out_extra, uint32_t* __restrict__ n_contrib,
                  const OutPeers peers) {
  if (hdr[HDR_OVERFLOW]) return;
  __shared__ __align__(16) float4 s_rec[FWD_STAGES][FWD_BATCH][4];   // 32 KB
  __shared__ uint32_t s_id[FWD_STAGES][FWD_BATCH];
  // s_bits[stage][block][word]: bit j of word k set <=> record 32k+j can reach that 8x4 pixel block
  __shared__ uint32_t s_bits[FWD_STAGES][FWD_THREADS / 32][FWD_BATCH / 32];

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
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
  const int nbatches = (total + FWD_BATCH - 1) / FWD_BATCH;

  // Transmittance of a live pixel.  A pixel that is finished (outside the image, or its next T would drop below
  // 1e-4) parks its transmittance in T_done and continues with T = 0: every later record then fails the same
  // `T*(1-alpha) < 1e-4` test on its own, so the inner loop needs no separate per-lane "done" flag (a live T is
  // never 0: it starts at 1, shrinks by factors >= 0.01 and stops before it reaches 1e-4).
  float T = inside ? 1.0f : 0.0f;
  float T_done = 0.0f;
  uint32_t last_contributor = 0;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f, Dp = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
  float E[HAS_EXTRA ? SFGS_MAX_EXTRA : 1];
  if (HAS_EXTRA) {
#pragma unroll
    for (int i = 0; i < SFGS_MAX_EXTRA; i++) E[i] = 0.f;
  }

#if SFGS_TMA_STAGING
  __shared__ __align__(8) unsigned long long s_mbar[FWD_STAGES];
  if (tid == 0) {
    mbar_init(&s_mbar[0], FWD_THREADS / 32);
    mbar_init(&s_mbar[1], FWD_THREADS / 32);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
  }
  __syncthreads();
#endif

  // stage loader: thread t copies record t of the batch (skipped when no block of the tile can be reached) and
  // the warp publishes, per pixel block, the ballot of "this record reaches the block" — bit-REVERSED, so that the
  // walk below finds the next record with one count-leading-zeros (FLO) instead of a bit reversal + FLO per record.
  auto issue = [&](int batch, int stage) {
    const int e = batch * FWD_BATCH + tid;
    unsigned m = 0;
    if (e < total) {
      m = inst_mask[range.x + e];
      if (m) {
        const uint32_t id = point_list[range.x + e];
        const float* src = rec + (size_t)id * REC_FLOATS;
#if SFGS_TMA_STAGING
        tma_load_64(&s_rec[stage][tid][0], src, &s_mbar[stage]);
#else
#pragma unroll
        for (int q = 0; q < 4; q++) cp_async16(&s_rec[stage][tid][q], src + q * 4);
#endif
        if (HAS_EXTRA) s_id[stage][tid] = id;
      }
    }
#if SFGS_TMA_STAGING
    {
      const unsigned nrec = __popc(__ballot_sync(0xffffffffu, m != 0));
      if (lane == 0) {
        if (nrec) mbar_arrive_expect_tx(&s_mbar[stage], nrec * 64u);
        else mbar_arrive(&s_mbar[stage]);
      }
    }
#else
    cp_async_commit();
#endif
#pragma unroll
    for (int blk = 0; blk < FWD_THREADS / 32; blk++) {
      const unsigned word = __ballot_sync(0xffffffffu, (m >> blk) & 1u);
      if (lane == 0) s_bits[stage][blk][wid] = __brev(word);
    }
  };

  const SfgsExpConsts ek = sfgs_exp_consts(hdr[HDR_ZERO]);
  if (nbatches > 0) issue(0, 0);
  for (int b = 0; b < nbatches; b++) {
    const int stage = b & 1;
#if SFGS_TMA_STAGING
    mbar_wait(&s_mbar[stage], (unsigned)(b >> 1) & 1u);
#else
    cp_async_wait<0>();
#endif
    // barrier: stage `b` visible to all, stage `b^1` no longer read by anyone
    const int num_done = __syncthreads_count(T == 0.0f);
    if (num_done == FWD_THREADS) break;
    if (b + 1 < nbatches) issue(b + 1, stage ^ 1);
    for (int word = 0; word < FWD_BATCH / 32; word++) {
      unsigned m = s_bits[stage][wid][word];
      if (m == 0u) continue;
      if (__all_sync(0xffffffffu, T == 0.0f)) break;
      // bit 31 = first record of the word: record 32*word + 31 - kk sits kk records BELOW this pointer / position
      const float4* rec_hi = &s_rec[stage][word * 32 + 31][0];
      const uint32_t pos_hi = (uint32_t)(b * FWD_BATCH + word * 32 + 32);   // 1-based list position of that record
      while (m) {
        unsigned kk;
        asm("bfind.u32 %0, %1;" : "=r"(kk) : "r"(m));   // FLO: highest set bit = next record front to back
        m ^= ek.one << kk;
        const float4* rp = rec_hi - 4 * kk;
        const float4 a = rp[0];   // mx, my, con.x, con.y
        const float4 c = rp[1];   // con.z, opac, depth, -
        const float dx = a.x - pixfx, dy = a.y - pixfy;
        const float power = -0.5f * (a.z * dx * dx + c.x * dy * dy) - a.w * dx * dy;
        if (power > 0.0f) continue;
        const float alpha = min(0.99f, c.y * sfgs_expf(power, ek));
        if (alpha < 1.0f / 255.0f) continue;
        const float test_T = T * (1 - alpha);
        if (test_T < 0.0001f) { T_done = fmaxf(T_done, T); T = 0.0f; continue; }
        const float4 f = rp[2];   // r, g, b, nx
        const float4 g = rp[3];   // ny, nz
        // colour and normal (|values| <= 1) take the pair's weight alpha*T as one factor; the depth image reaches
        // hundreds of units, where 1e-5 absolute is below one ulp, so it keeps the reference's exact association
        // (depth * alpha) * T and stays bit-identical
        const float w = alpha * T;
        C0 = fmaf(f.x, w, C0); C1 = fmaf(f.y, w, C1); C2 = fmaf(f.z, w, C2);
        Dp += c.z * alpha * T;
        N0 = fmaf(f.w, w, N0); N1 = fmaf(g.x, w, N1); N2 = fmaf(g.y, w, N2);
        if (HAS_EXTRA) {
          const float* ex = extras + (size_t)s_id[stage][word * 32 + 31 - (int)kk] * ED;
          for (int ch = 0; ch < ED; ch++) E[ch] += ex[ch] * alpha * T;
        }
        T = test_T;
        last_contributor = pos_hi - kk;
      }
    }
  }
  if (T == 0.0f) T = T_done;   // finished early: the transmittance it finished with

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
    if (HAS_EXTRA)
      for (int ch = 0; ch < ED; ch++) out_extra[ch * HW + pix_id] = E[ch];
  }
}


// =====================================================================================================================
// Warp-private variant (the default path; the kernel above remains for extra_attrs and the TMA-staging experiment).
// Same idea as render_bwd_warp_kernel (sfgs_render_bwd.cu): every warp walks the tile's sorted list itself, front to
// back, keeps the positions whose reach mask has its block's bit, gathers them 16 at a time into a private
// double-buffered slot (two lanes per 64-byte record, cp.async, overlapping the previous chunk's math) and blends the
// chunk in slot order.  Nothing is block-wide: no __syncthreads, no per-record bit scanning, record parameters at
// immediate offsets, and a warp whose 32 pixels are saturated stops scanning on its own.
constexpr int F4_CH = 16;
struct alignas(16) FwdWarpSmem {
  float4 rec[2][F4_CH][4];      // 2 KB   the chunk's blend records, double buffered; the free word [1].w of a staged
                                //        record carries its 1-based list position (bits of a uint32)
  uint32_t list[64];            // ring of collected list positions
};

template <bool FLAT>
__global__ void __launch_bounds__(FWD_THREADS)
render_fwd_warp_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                       const unsigned char* __restrict__ inst_mask, const uint32_t* __restrict__ hdr, int W, int H,
                       int band0, const float* __restrict__ rec, const float* __restrict__ bg_color,
                       float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_norm,
                       float* __restrict__ out_norm_raw, float* __restrict__ out_alpha, uint32_t* __restrict__ n_contrib,
                       const OutPeers peers) {
  if (hdr[HDR_OVERFLOW]) return;
  __shared__ FwdWarpSmem s_warp[FWD_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  FwdWarpSmem& S = s_warp[wid];
  const int tiles_x = (W + SFGS_TILE - 1) / SFGS_TILE;
  const int tile_y = blockIdx.y + band0;
  const int tile = tile_y * tiles_x + blockIdx.x;
  const int px = blockIdx.x * SFGS_TILE + (wid & 1) * 8 + (lane & 7);
  const int py = tile_y * SFGS_TILE + (wid >> 1) * 4 + (lane >> 3);
  const bool inside = px < W && py < H;
  const uint32_t pix_id = (uint32_t)W * py + px;
  const float pixfx = (float)px, pixfy = (float)py;

  const uint2 range = ranges[tile];
  const int total = (int)(range.y - range.x);

  // see render_fwd_kernel: a finished pixel parks its transmittance in T_done and continues with T = 0
  float T = inside ? 1.0f : 0.0f;
  float T_done = 0.0f;
  uint32_t last_contributor = 0;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f, Dp = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
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
    cp_async_wait<0>();
    __syncwarp();                                   // chunk `buf` has landed and is visible to the whole warp
    if (__all_sync(0xffffffffu, T == 0.0f)) break;  // every pixel of the block is saturated (or outside the image)
    const int n_next = scan_gather(buf ^ 1);        // the next chunk's gather overlaps the math below
    auto slot_body = [&](const int k, const float4 a, const float4 c) {
      const float dx = a.x - pixfx, dy = a.y - pixfy;
      const float power = -0.5f * (a.z * dx * dx + c.x * dy * dy) - a.w * dx * dy;
      if (FLAT) {
        // branch-free form (one basic block per chunk: slot k+1's load -> exp chain overlaps slot k's accumulation).
        // A pair that is not applied multiplies every accumulator update by an exact 0.
        const float4 f = S.rec[buf][k][2];      // r, g, b, nx
        const float4 g = S.rec[buf][k][3];      // ny, nz
        const float alpha = min(0.99f, c.y * sfgs_expf(power, ek));
        const bool ok = !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
        const float test_T = T * (1 - alpha);
        const bool stop = ok && (test_T < 0.0001f);
        const bool apply = ok && !stop;
        const float Ta = apply ? T : 0.0f;
        const float w = alpha * Ta;
        C0 = fmaf(f.x, w, C0); C1 = fmaf(f.y, w, C1); C2 = fmaf(f.z, w, C2);
        Dp = fmaf(c.z * alpha, Ta, Dp);           // (depth * alpha) * T, the reference's association
        N0 = fmaf(f.w, w, N0); N1 = fmaf(g.x, w, N1); N2 = fmaf(g.y, w, N2);
        T_done = stop ? fmaxf(T_done, T) : T_done;
        T = apply ? test_T : (stop ? 0.0f : T);
        last_contributor = apply ? __float_as_uint(c.w) : last_contributor;
      } else if (!(power > 0.0f)) {
        const float alpha = min(0.99f, c.y * sfgs_expf(power, ek));
        if (!(alpha < 1.0f / 255.0f)) {
          const float test_T = T * (1 - alpha);
          if (test_T < 0.0001f) { T_done = fmaxf(T_done, T); T = 0.0f; }
          else {
            const float4 f = S.rec[buf][k][2];    // r, g, b, nx
            const float4 g = S.rec[buf][k][3];    // ny, nz
            const float w = alpha * T;            // see render_fwd_kernel for the association of each output
            C0 = fmaf(f.x, w, C0); C1 = fmaf(f.y, w, C1); C2 = fmaf(f.z, w, C2);
            Dp += c.z * alpha * T;
            N0 = fmaf(f.w, w, N0); N1 = fmaf(g.x, w, N1); N2 = fmaf(g.y, w, N2);
            T = test_T;
            last_contributor = __float_as_uint(c.w);
          }
        }
      }
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
  cp_async_wait<0>();                // nothing may still be landing in this CTA's shared memory when it exits
  if (T == 0.0f) T = T_done;

  if (inside) {
    const size_t HW = (size_t)H * W;
    n_contrib[pix_id] = last_contributor;
    const float c0 = C0 + T * bg_color[0], c1 = C1 + T * bg_color[1], c2 = C2 + T * bg_color[2];
    if (out_norm_raw != nullptr) {
      out_norm_raw[0 * HW + pix_id] = N0;
      out_norm_raw[1 * HW + pix_id] = N1;
      out_norm_raw[2 * HW + pix_id] = N2;
      const float d = fmaxf(sqrtf(N0 * N0 + N1 * N1 + N2 * N2), 1e-12f);
      N0 = N0 / d; N1 = N1 / d; N2 = N2 / d;
    }
    if (peers.n > 0) {
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
#if !SFGS_TMA_STAGING
  if (a->ED == 0) {   // default path: warp-private pipelines (render_fwd_warp_kernel)
    // the branch-free form is the default; SFGS_FWD_FLAT=0 selects the branching one (A/B measurements)  — branch-free blend loop
    static const bool flat = [] { const char* e = getenv("SFGS_FWD_FLAT"); return !(e && e[0] == '0'); }();
#define RFW_ARGS im.ranges, b.point_list, b.inst_mask, im.hdr, a->width, a->height, band0, g.rec, a->background, a->out_color,   \
      a->out_depth, a->out_norm, a->out_norm_raw, a->out_alpha, im.n_contrib, op
    if (flat) render_fwd_warp_kernel<true><<<grid, FWD_THREADS, 0, st>>>(RFW_ARGS);
    else render_fwd_warp_kernel<false><<<grid, FWD_THREADS, 0, st>>>(RFW_ARGS);
#undef RFW_ARGS
    return;
  }
#endif
  if (a->ED > 0)
    render_fwd_kernel<true><<<grid, FWD_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr, a->width, a->height, a->ED, band0,
                                                         g.rec, a->extra_attrs, a->background, a->out_color,
                                                         a->out_depth, a->out_norm, a->out_norm_raw, a->out_alpha,
                                                         a->out_extra, im.n_contrib, op);
  else
    render_fwd_kernel<false><<<grid, FWD_THREADS, 0, st>>>(im.ranges, b.point_list, b.inst_mask, im.hdr, a->width, a->height, 0, band0,
                                                          g.rec, nullptr, a->background, a->out_color, a->out_depth,
                                                          a->out_norm, a->out_norm_raw, a->out_alpha, nullptr,
                                                          im.n_contrib, op);
}
