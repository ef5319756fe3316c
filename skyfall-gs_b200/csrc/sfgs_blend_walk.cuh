// sfgs_blend_walk.cuh — the reach-list walk of the blend kernels.  The forward blend (sfgs_render_fwd.cu) and the
// blend adjoint (sfgs_render_bwd.cu) take everything but their own math from here.
//
// One CTA of 256 threads per 16x16 tile.  Warp w owns the 8x4 pixel block (w%2, w/2) of the tile, lane l the pixel
// (l%8, l/8) of the block, and each warp runs its own pipeline: nothing in a blend kernel is block-wide.
//
//   scan     the warp walks the tile's sorted list 32 positions at a time — the forward front to back, from 0 up to
//            the list's length; the adjoint back to front, from its block's last contributor down to 0 — reads the 32
//            reach masks (computed by the sort stage, sfgs_common.cuh) in one coalesced load and keeps the positions
//            whose mask has its block's bit (ballot + prefix popcount into a 64-entry ring).  That removes ~80 % of
//            the (pixel, Gaussian) evaluations without changing any result;
//   gather   as soon as 16 positions are collected (or the list is exhausted) it copies exactly those records, two
//            lanes per 64-byte record, with cp.async into its private double-buffered chunk slot;
//   chunks   blend_chunks overlaps each chunk's gather with the previous chunk's math.  Every chunk of a warp but its
//            last is full, and a kernel runs a full chunk fully unrolled: one branch-free basic block with record
//            parameters at immediate offsets, in which slot k+1's load -> exp chain overlaps slot k's accumulation.
//
// The free word.  A record's second quad is (con.z, opacity, depth, free).  It is copied as 8 + 4 bytes, and the free
// word takes the record's 1-based list position (the bits of a uint32), so the slot body finds it in the quad it loads
// anyway.  That is the value n_contrib holds: the forward stores the position of a pixel's last applied record, and in
// the adjoint a record can be active for a pixel only if its position is <= the pixel's n_contrib.
#pragma once
#include "sfgs_common.cuh"

constexpr int BLEND_THREADS = 256;
constexpr int BLEND_WARPS = BLEND_THREADS / 32;   // = the eight 8x4 blocks of a tile
constexpr int BLEND_CH = 16;                      // records per chunk

// The CTA's tile and the lane's pixel
struct BlendPixel {
  int tile;
  bool inside;          // the pixel lies in the image
  uint32_t id;          // W * y + x
  float x, y;           // pixel centre (integer coordinates)
  __device__ __forceinline__ BlendPixel(int band0, int W, int H, int wid, int lane) {
    const int tiles_x = (W + SFGS_TILE - 1) / SFGS_TILE;
    const int tile_y = blockIdx.y + band0;
    tile = tile_y * tiles_x + blockIdx.x;
    const int px = blockIdx.x * SFGS_TILE + (wid & 1) * 8 + (lane & 7);
    const int py = tile_y * SFGS_TILE + (wid >> 1) * 4 + (lane >> 3);
    inside = px < W && py < H;
    id = (uint32_t)W * py + px;
    x = (float)px;
    y = (float)py;
  }
};

// What a slot's gid word holds: nothing (no gid words), the Gaussian id, or the sorted instance range.x + position
enum BlendGid { GID_NONE, GID_GAUSSIAN, GID_INSTANCE };

// A warp's staging area
struct alignas(16) BlendStageBase {
  float4 rec[2][BLEND_CH][4];   // 2 KB   the chunk's blend records, double buffered
  uint32_t list[64];            // ring of collected list positions
};
template <bool HAS_GID>
struct BlendStage : BlendStageBase {
  uint32_t gid[2][BLEND_CH];
};
template <>
struct BlendStage<false> : BlendStageBase {};

// The walk of one warp over the list of its tile.  gather(buf) scans on until 16 positions are collected or the list
// is exhausted, issues the cp.async copies of up to 16 records into buffer `buf` and returns their number (0: the
// walk is over).
template <bool BACKWARD, int GID>
struct BlendWalk {
  BlendStage<GID != GID_NONE>& S;
  const unsigned char* inst_mask;
  const uint32_t* point_list;
  const float* rec;
  const uint2 range;
  const int n;                      // forward: the list's length; adjoint: the first position it does not walk
  const int wid, lane;
  const unsigned lt_mask;
  int p;                            // forward: positions [p, n) are unscanned; adjoint: positions [0, p)
  int head = 0, have = 0;           // ring of collected positions: [head, head + have)

  __device__ __forceinline__ BlendWalk(BlendStage<GID != GID_NONE>& S, const unsigned char* inst_mask,
                                       const uint32_t* point_list, const float* rec, uint2 range, int n, int wid,
                                       int lane)
      : S(S), inst_mask(inst_mask), point_list(point_list), rec(rec), range(range), n(n), wid(wid), lane(lane),
        lt_mask((1u << lane) - 1u), p(BACKWARD ? n : 0) {}

  __device__ __forceinline__ int gather(int buf) {
    while (have < BLEND_CH && (BACKWARD ? p > 0 : p < n)) {
      const int pos = BACKWARD ? p - 1 - lane : p + lane;   // adjoint: lane 0 takes the highest position
      unsigned m = 0;
      if (BACKWARD ? pos >= 0 : pos < n) m = inst_mask[range.x + pos];
      const bool bit = (m >> wid) & 1u;
      const unsigned b = __ballot_sync(0xffffffffu, bit);
      if (bit) S.list[(head + have + __popc(b & lt_mask)) & 63] = (uint32_t)pos;
      have += __popc(b);
      p += BACKWARD ? -32 : 32;
    }
    __syncwarp();
    const int c = min(have, BLEND_CH);
    if (lane < 2 * c) {               // two lanes per 64-byte record
      const int r = lane >> 1, hf = lane & 1;
      const uint32_t pos = S.list[(head + r) & 63];
      const uint32_t id = point_list[range.x + pos];
      const float* src = rec + (size_t)id * REC_FLOATS;
      if (hf == 0) {
        cp_async16(&S.rec[buf][r][0], src);
        cp_async16(&S.rec[buf][r][2], src + 8);
        if constexpr (GID != GID_NONE) S.gid[buf][r] = GID == GID_INSTANCE ? range.x + pos : id;
      } else {
        cp_async16(&S.rec[buf][r][3], src + 12);
        cp_async8(&S.rec[buf][r][1], src + 4);
        cp_async4(&S.rec[buf][r][1].z, src + 6);
        S.rec[buf][r][1].w = __uint_as_float(pos + 1u);   // the free word: the 1-based list position
      }
    }
    cp_async_commit();
    head = (head + c) & 63;
    have -= c;
    return c;
  }
};

// The double-buffered chunk loop: once a chunk has landed, stop() may end the walk (no copy is then in flight);
// otherwise the next chunk's gather is issued and body(buf, n) processes the n records in buffer `buf`.  XOR_FLIP only
// picks the form of the buffer flip, which steers ptxas's register allocation: in the adjoint, buf ^ 1 spills in two
// of the three default instantiations and 1 - buf spills one word in the ORDERED one.
template <bool XOR_FLIP, class Walk, class Stop, class Body>
__device__ __forceinline__ void blend_chunks(Walk& walk, Stop stop, Body body) {
  int buf = 0;
  int n_cur = walk.gather(0);
  while (n_cur > 0) {
    cp_async_wait_all();
    __syncwarp();                                   // chunk `buf` has landed and is visible to the whole warp
    if (stop()) break;
    const int n_next = walk.gather(buf ^ 1);        // the next chunk's gather overlaps the body
    body(buf, n_cur);
    buf = XOR_FLIP ? buf ^ 1 : 1 - buf;
    n_cur = n_next;
  }
}

// The grid of a blend launch: one CTA per tile of the call's band of tile rows; false if the band is empty
static inline bool blend_grid(int tile_row_begin, int tile_row_end, const ImageLayout& im, dim3& grid, int& band0) {
  const SfgsBand band = sfgs_band(tile_row_begin, tile_row_end, im.tiles_y);
  band0 = band.b0;
  grid = dim3(im.tiles_x, band.b1 - band.b0, 1);
  return band.b1 > band.b0;
}
