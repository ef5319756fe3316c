// sfgs_bwd_order.cu — the fixed-order reduction of the deterministic backward (sfgs_rasterize_backward_deterministic).
//
// The ORDERED blend adjoint (sfgs_render_bwd.cu) leaves one 16-word partial per visited (tile instance, 8x4 block)
// pair in `part`, row = sorted instance * 8 + block, and sets written[row].  This file turns those rows into acc[P,16]
// with every sum in an order fixed by the inputs alone:
//
//   off      exclusive scan of tiles_touched over P (integers: any order gives the same bits).  Gaussian g owns the
//            slots off[g] .. off[g] + tiles_touched[g] - 1, one per tile of its band-clipped rectangle in row-major
//            order — the order the preprocess emits its instances in (sfgs_preprocess.cu, `kk`);
//   inv      inv[off[g] + rank] = sorted instance of (g, tile), rank = the tile's row-major index in the rectangle.
//            One CTA per tile walks its list; (g, tile) -> slot is a bijection, so every store has its own address;
//   reduce   16 lanes per Gaussian, lane c = word c: the Gaussian's slots in increasing rank, inside each slot its
//            written blocks in increasing block index, summed in float64 and stored once as float32.  A Gaussian
//            without a written row gets zeros.
#include "sfgs_common.cuh"

namespace {

constexpr int SCAN_SPAN = 4096;     // Gaussians per block of the offset scan (256 threads x 16)

// per-block totals of tiles_touched
__global__ void __launch_bounds__(256) off_block_sum_kernel(int P, const uint32_t* __restrict__ tt, uint32_t* __restrict__ bsum) {
  __shared__ uint32_t s_w[8];
  const int base = blockIdx.x * SCAN_SPAN;
  uint32_t v = 0;
  for (int i = threadIdx.x; i < SCAN_SPAN; i += 256)
    if (base + i < P) v += tt[base + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < 8; w++) t += s_w[w];
    bsum[blockIdx.x] = t;
  }
}

// exclusive scan of the block totals, in place.  One block; chunks of 1024 with a carry.
__global__ void __launch_bounds__(1024) off_block_scan_kernel(int nb, uint32_t* __restrict__ bsum) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  if (t == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int b = base + t;
    const uint32_t v = b < nb ? bsum[b] : 0u;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
      uint32_t x = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += u; }
      s_warp[lane] = x;
    }
    __syncthreads();
    const uint32_t carry = s_carry;
    if (b < nb) bsum[b] = carry + (w ? s_warp[w - 1] : 0u) + inc - v;
    __syncthreads();
    if (t == 1023) s_carry = carry + s_warp[31];
    __syncthreads();
  }
}

// off[g] = block base + exclusive scan inside the block (16 consecutive Gaussians per thread)
__global__ void __launch_bounds__(256) off_apply_kernel(int P, const uint32_t* __restrict__ tt,
                                                        const uint32_t* __restrict__ bsum, uint32_t* __restrict__ off) {
  __shared__ uint32_t s_warp[8];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int first = blockIdx.x * SCAN_SPAN + t * 16;
  uint32_t v[16], sum = 0;
#pragma unroll
  for (int k = 0; k < 16; k++) { v[k] = first + k < P ? tt[first + k] : 0u; sum += v[k]; }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  uint32_t run = bsum[blockIdx.x] + inc - sum;
  for (int k = 0; k < w; k++) run += s_warp[k];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    if (first + k < P) off[first + k] = run;
    run += v[k];
  }
}

// inv[off[g] + rank(g, tile)] = sorted instance, one CTA per tile of the band.
// GUARD (the graph backward, sfgs_rasterize_backward_graph): nothing is done when the forward overflowed its binning
// capacity (image header `hdr`), because the ranges then run past point_list and inv; without it `hdr` is not read.
template <bool GUARD>
__global__ void __launch_bounds__(256) inv_map_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                                                      const float* __restrict__ rec, const int* __restrict__ radii,
                                                      const uint32_t* __restrict__ off, int gx, int gy, int band0,
                                                      uint32_t* __restrict__ inv, const uint32_t* __restrict__ hdr) {
  if (GUARD && hdr[HDR_OVERFLOW]) return;
  const int tx = blockIdx.x, ty = blockIdx.y + band0;
  const uint2 range = ranges[ty * gx + tx];
  for (uint32_t i = range.x + threadIdx.x; i < range.y; i += blockDim.x) {
    const uint32_t g = point_list[i];
    const float2 m = *reinterpret_cast<const float2*>(rec + (size_t)g * REC_FLOATS);
    // the rectangle and band clip of the preprocess, from the same floats (record words 0-1) and radius
    TileRect r = tile_rect(m.x, m.y, radii[g], gx, gy);
    r.y0 = max(r.y0, band0);
    const uint32_t rank = (uint32_t)(ty - r.y0) * (uint32_t)(r.x1 - r.x0) + (uint32_t)(tx - r.x0);
    inv[off[g] + rank] = i;
  }
}

// acc[g] = sum of Gaussian g's written rows, in (rank, block) order, in float64.  16 lanes per Gaussian, lane c = word
// c.  The slots of a Gaussian are taken 16 at a time (lane k reads slot k's instance and flags); the rows of four
// slots are loaded before they are added, so their latencies overlap.
// GUARD: after an overflowed forward every Gaussian is taken to have no slots (inv was not written), so acc gets zeros.
template <bool GUARD>
__global__ void __launch_bounds__(256) ordered_reduce_kernel(int P, const uint32_t* __restrict__ tt,
                                                             const uint32_t* __restrict__ off,
                                                             const uint32_t* __restrict__ inv,
                                                             const uint2* __restrict__ written,
                                                             const float* __restrict__ part,
                                                             const int* __restrict__ radii, int all_rows,
                                                             float* __restrict__ acc, const uint32_t* __restrict__ hdr) {
  const int g = blockIdx.x * 16 + (threadIdx.x >> 4);
  if (g >= P) return;
  if (!all_rows && radii[g] <= 0) return;          // rows the per-Gaussian adjoint never reads
  const int c = threadIdx.x & 15;
  const unsigned hmask = 0xFFFFu << (threadIdx.x & 16);
  const uint32_t n = (GUARD && hdr[HDR_OVERFLOW]) ? 0u : tt[g];
  const uint32_t base = n ? off[g] : 0u;
  double s = 0.0;
  for (uint32_t k0 = 0; k0 < n; k0 += 16) {
    const uint32_t m = min(16u, n - k0);
    uint32_t my_inst = 0;
    uint2 my_f = make_uint2(0u, 0u);             // one byte per block: 1 = written
    if ((uint32_t)c < m) {
      my_inst = inv[base + k0 + c];
      my_f = written[my_inst];
    }
    for (uint32_t j = 0; j < m; j += 4) {
      float v[4][8];
      uint2 f[4];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const uint32_t inst = __shfl_sync(hmask, my_inst, j + q, 16);
        f[q].x = __shfl_sync(hmask, my_f.x, j + q, 16);
        f[q].y = __shfl_sync(hmask, my_f.y, j + q, 16);   // slots past m come from lanes that loaded nothing: 0
        const float* row = part + (size_t)inst * (BWD_BLOCKS * 16) + c;
#pragma unroll
        for (int b = 0; b < 8; b++) {
          const bool w = (((b < 4 ? f[q].x : f[q].y) >> (8 * (b & 3))) & 0xFFu) != 0u;
          v[q][b] = w ? __ldg(row + b * 16) : 0.f;
        }
      }
#pragma unroll
      for (int q = 0; q < 4; q++)
#pragma unroll
        for (int b = 0; b < 8; b++)
          if ((((b < 4 ? f[q].x : f[q].y) >> (8 * (b & 3))) & 0xFFu) != 0u) s += (double)v[q][b];
    }
  }
  acc[(size_t)g * 16 + c] = (float)s;
}

}  // namespace

size_t sfgs_order_scratch_bytes(int P, long long R) {
  const size_t nb = ((size_t)P + SCAN_SPAN - 1) / SCAN_SPAN;
  return sfgs_align_up(nb * 4) + sfgs_align_up((size_t)P * 4) + sfgs_align_up((size_t)R * 4) +
         sfgs_align_up((size_t)R * BWD_BLOCKS) + sfgs_align_up((size_t)R * BWD_BLOCKS * 16 * sizeof(float));
}

SfgsOrderScratch sfgs_order_scratch(char* base, int P, long long R) {
  SfgsOrderScratch o;
  const size_t nb = ((size_t)P + SCAN_SPAN - 1) / SCAN_SPAN;
  size_t x = 0;
  o.bsum = (uint32_t*)(base + x); x += sfgs_align_up(nb * 4);
  o.off = (uint32_t*)(base + x); x += sfgs_align_up((size_t)P * 4);
  o.inv = (uint32_t*)(base + x); x += sfgs_align_up((size_t)R * 4);
  o.written = (unsigned char*)(base + x); x += sfgs_align_up((size_t)R * BWD_BLOCKS);
  o.part = (float*)(base + x);
  return o;
}

void sfgs_launch_order_prepare(int P, const GeomLayout& g, const ImageLayout& im, const BinningLayout& b,
                               const int* radii, int band0, int band1, const SfgsOrderScratch& o, bool guarded,
                               cudaStream_t st) {
  const int nb = (P + SCAN_SPAN - 1) / SCAN_SPAN;
  SFGS_COUNT_LAUNCH(); off_block_sum_kernel<<<nb, 256, 0, st>>>(P, g.tiles_touched, o.bsum);
  SFGS_COUNT_LAUNCH(); off_block_scan_kernel<<<1, 1024, 0, st>>>(nb, o.bsum);
  SFGS_COUNT_LAUNCH(); off_apply_kernel<<<nb, 256, 0, st>>>(P, g.tiles_touched, o.bsum, o.off);
  if (band1 > band0) {
    SFGS_COUNT_LAUNCH();
    const auto kernel = guarded ? inv_map_kernel<true> : inv_map_kernel<false>;
    kernel<<<dim3(im.tiles_x, band1 - band0), 256, 0, st>>>(im.ranges, b.point_list, g.rec, radii, o.off, im.tiles_x,
                                                            im.tiles_y, band0, o.inv, im.hdr);
  }
}

// hdr_guard: NULL, or the image header whose overflow flag the graph backward's kernel checks first
void sfgs_launch_order_reduce(int P, const GeomLayout& g, const int* radii, bool all_rows, const SfgsOrderScratch& o,
                              float* acc, const uint32_t* hdr_guard, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  const auto kernel = hdr_guard != nullptr ? ordered_reduce_kernel<true> : ordered_reduce_kernel<false>;
  kernel<<<(P + 15) / 16, 256, 0, st>>>(P, g.tiles_touched, o.off, o.inv, reinterpret_cast<const uint2*>(o.written),
                                        o.part, radii, all_rows ? 1 : 0, acc, hdr_guard);
}
