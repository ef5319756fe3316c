// sfgs_binning.cu — tile binning: histogram scan, key emission, per-tile sort.
//
// Replaces cub::DeviceScan::InclusiveSum + duplicateWithKeys +
// cub::DeviceRadixSort::SortPairs + identifyTileRanges
// (RAST/cuda_rasterizer/rasterizer_impl.cu:70-138, 283-324).
//
// The reference sorts all R (tile|depth) 64-bit keys globally with a stable
// LSD radix sort, so inside a tile equal depths keep emission order = ascending
// Gaussian id.  Here the tile part of the key is resolved by a counting sort
// (per-tile histogram from the preprocess stage -> exclusive scan -> bucket
// cursors) and each tile bucket is then sorted on (depth_bits << 32 | id) in
// shared memory.  The resulting (tile, depth, id) order — and therefore
// point_list and ranges — is identical to the reference's, bit for bit.
#include "sfgs_common.cuh"
#include <cstdlib>

namespace {

// ---- exclusive scan of the tile histogram (single CTA, 8 tiles per thread per pass) ----------
constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_ITEMS = 8;
__global__ void __launch_bounds__(SCAN_THREADS)
tile_scan_kernel(int tiles, const uint32_t* __restrict__ tile_count, uint2* __restrict__ ranges,
                 uint32_t* __restrict__ hdr, unsigned long long capacity) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry_s;
  __shared__ uint32_t maxlen_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { carry_s = 0; maxlen_s = 0; }
  __syncthreads();
  uint32_t local_max = 0;
  for (int base = 0; base < tiles; base += SCAN_THREADS * SCAN_ITEMS) {
    const int i0 = base + tid * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint32_t x = 0;
    const bool full = i0 + SCAN_ITEMS <= tiles;   // whole 8-item group in range: two 16-byte loads, four 16-byte stores
    if (full) {
      const uint4 a = reinterpret_cast<const uint4*>(tile_count + i0)[0], b = reinterpret_cast<const uint4*>(tile_count + i0)[1];
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int k = 0; k < SCAN_ITEMS; k++) v[k] = (i0 + k < tiles) ? tile_count[i0 + k] : 0u;
    }
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) {
      local_max = max(local_max, v[k]);
      x += v[k];
    }
    const uint32_t mine = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
      uint32_t s = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
      warp_sums[lane] = s;
    }
    __syncthreads();
    const uint32_t carry = carry_s;
    const uint32_t incl = carry + x + (wid > 0 ? warp_sums[wid - 1] : 0u);
    uint32_t run = incl - mine;   // exclusive prefix of this thread's first tile
    // empty tiles read (0,0) exactly like the reference's memset + identifyTileRanges
    uint2 rg[SCAN_ITEMS];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) {
      rg[k] = v[k] ? make_uint2(run, run + v[k]) : make_uint2(0u, 0u);
      run += v[k];
    }
    if (full) {
#pragma unroll
      for (int k = 0; k < SCAN_ITEMS; k += 2)
        reinterpret_cast<uint4*>(ranges + i0)[k >> 1] = make_uint4(rg[k].x, rg[k].y, rg[k + 1].x, rg[k + 1].y);
    } else {
#pragma unroll
      for (int k = 0; k < SCAN_ITEMS; k++)
        if (i0 + k < tiles) ranges[i0 + k] = rg[k];
    }
    __syncthreads();
    if (tid == SCAN_THREADS - 1) carry_s = incl;
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local_max = max(local_max, __shfl_xor_sync(0xffffffffu, local_max, o));
  if (lane == 0) atomicMax(&maxlen_s, local_max);
  __syncthreads();
  if (tid == 0) {
    const uint32_t R = carry_s;
    hdr[HDR_R] = R;
    hdr[HDR_OVERFLOW] = ((unsigned long long)R > capacity) ? 1u : 0u;
    hdr[HDR_MAXTILE] = maxlen_s;
    hdr[HDR_CAP_LO] = (uint32_t)(capacity & 0xffffffffull);
    hdr[HDR_CAP_HI] = (uint32_t)(capacity >> 32);
  }
}

// ---- key scatter ---------------------------------------------------------------
// One thread per unsorted instance {gaussian, depth bits, tile}: perfectly balanced.
//
// The kernel is latency-bound (four independent instances in flight per thread, ~10 % of the issue slots used), so it
// also computes the instance's REACH MASK (which of the tile's eight 8x4-pixel blocks the splat's alpha >= 1/255
// ellipse can touch, sfgs_common.cuh) from the Gaussian's blend record — the instances of one Gaussian are neighbours
// in the unsorted list, so the 24 record bytes come from L1/L2 — and, when every Gaussian id fits 24 bits (PACK), carries
// it through the sort in the low byte of the key:
//     key = depth_bits << 32 | id << 8 | mask
// (depth, id) is unique inside a tile, so the order is the order of depth_bits << 32 | id.  The sort kernels then touch
// no Gaussian data at all; round 1/2a gathered 56 MB of records inside the sort CTAs to form the masks there.
// With P >= 2^24 the key stays depth_bits << 32 | id and the sort kernels compute the masks as before.
// ITEMS: instances per thread (independent loads in flight).  With the mask the kernel needs ~36 live floats per
// instance in flight, so the packed path runs two per thread; the unpacked path forms no mask and runs four.
template <bool PACK, int ITEMS>
__global__ void __launch_bounds__(256)
scatter_keys_kernel(const uint4* __restrict__ tmp, const uint2* __restrict__ ranges, uint32_t* __restrict__ tile_count,
                    const uint32_t* __restrict__ hdr, const float* __restrict__ rec, int gx, uint64_t* __restrict__ keys) {
  if (hdr[HDR_OVERFLOW]) return;
  const uint32_t R = hdr[HDR_R];
  const uint32_t i0 = blockIdx.x * (256u * ITEMS) + threadIdx.x;
  uint4 t[ITEMS];
  uint32_t start[ITEMS], slot[ITEMS];
  float4 r0[ITEMS];
  float2 r1[ITEMS];
#pragma unroll
  for (int u = 0; u < ITEMS; u++)
    if (i0 + 256u * u < R) t[u] = tmp[i0 + 256u * u];
#pragma unroll
  for (int u = 0; u < ITEMS; u++)
    if (i0 + 256u * u < R) {
      // the slot inside the tile bucket: the histogram the preprocess built is counted back down (any order will do,
      // the bucket is sorted next); the returning atomic is in flight while the reach mask is formed
      slot[u] = atomicSub(&tile_count[t[u].z], 1u) - 1u;
      start[u] = ranges[t[u].z].x;
      if (PACK) {
        r0[u] = *reinterpret_cast<const float4*>(rec + (size_t)t[u].x * REC_FLOATS);
        r1[u] = *reinterpret_cast<const float2*>(rec + (size_t)t[u].x * REC_FLOATS + 4);
      }
    }
#pragma unroll
  for (int u = 0; u < ITEMS; u++)
    if (i0 + 256u * u < R) {
      uint32_t lo = t[u].x;
      if (PACK) {
        const int tile_px = (int)(t[u].z % (uint32_t)gx) * SFGS_TILE, tile_py = (int)(t[u].z / (uint32_t)gx) * SFGS_TILE;
        lo = (t[u].x << 8) | reach_mask(r0[u].x, r0[u].y, r0[u].z, r0[u].w, r1[u].x, r1[u].y, tile_px, tile_py);
      }
      keys[start[u] + slot[u]] = ((uint64_t)t[u].y << 32) | lo;
    }
}

// ---- per-tile sort -------------------------------------------------------------
// One CTA per tile, two launches over the same grid: a light variant (128 threads x 8 keys, 1024-key window) for
// the common short lists and a heavy one (256 threads x 16 keys, 4096-key window, global radix fallback beyond
// that); a CTA whose tile belongs to the other class exits at once.  Lists inside the window are sorted by the
// shared-memory merge sort below.

// Shared-memory sort buffers hold key i at PADIDX(i): one pad word per 16 keys.  A thread owns VT consecutive keys, so
// without the pad the 32 lanes of a warp hit the same bank pair on every access (stride VT * 8 bytes = 64 or 128 bytes:
// 16- / 32-way conflicts); with it every blocked access pattern of VT = 4, 8, 16 is the 2-wavefront minimum of a
// 64-bit access.
__device__ __forceinline__ int PADIDX(int i) { return i + (i >> 4); }

// 64-bit compare-exchange of two registers (ascending)
__device__ __forceinline__ void cex(uint64_t& a, uint64_t& b) {
  const uint64_t lo = min(a, b), hi = max(a, b);
  a = lo; b = hi;
}

// ---- merge sort of one tile's keys in shared memory ------------------------------------------------
// Thread t owns keys [t*VT, (t+1)*VT): it sorts them in registers (odd-even transposition network), then
// log2(n/VT) merge passes follow; in each pass the thread finds, by a merge-path binary search on its output
// diagonal, where its VT outputs start in the two sorted runs and merges them sequentially.  Work is
// O(n log n) comparisons with n the real list length (only ceil(n/VT) threads take part, the tail is padded
// with +inf to a multiple of VT) — about 2.5x fewer issued instructions per key than the bitonic network
// (O(n log^2 n)) it replaces for the in-window lists, and independent of how the depths are distributed.
// Keys are unique ((depth, id) with one instance per Gaussian and tile), so no stability rule is needed.
// Returns the buffer that holds the sorted keys.
template <int THREADS, int VT>
__device__ __forceinline__ void merge_sort_smem(uint64_t* buf /* PADIDX(THREADS*VT) keys */, int* s_lo /* [THREADS + 1] */,
                                                const uint64_t* __restrict__ bucket, int n) {
  const int t = threadIdx.x;
  const int nchunks = (n + VT - 1) / VT;
  const int n_pad = nchunks * VT;
  uint64_t k[VT];
  if (t < nchunks) {
#pragma unroll
    for (int i = 0; i < VT; i++) { const int idx = t * VT + i; k[i] = idx < n ? bucket[idx] : ~0ull; }
#pragma unroll
    for (int kk = 2; kk <= VT; kk <<= 1) {
#pragma unroll
      for (int j = kk >> 1; j > 0; j >>= 1) {
#pragma unroll
        for (int i = 0; i < VT; i++) {
          const int l = i ^ j;
          if (l > i) {
            const bool up = (i & kk) == 0;
            const uint64_t lo = min(k[i], k[l]), hi = max(k[i], k[l]);
            k[i] = up ? lo : hi; k[l] = up ? hi : lo;
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < VT; i++) buf[PADIDX(t * VT + i)] = k[i];
  }
  __syncthreads();
  for (int L = VT; L < n_pad; L <<= 1) {
    const int out0 = t * VT;
    const int pair0 = out0 & ~(2 * L - 1);                 // 2L is a power of two
    const int lenA = min(L, max(0, n_pad - pair0));
    const int lenB = min(L, max(0, n_pad - pair0 - L));
    const int A0 = pair0, B0 = pair0 + L;
    const int diag = out0 - pair0;
    int lo = 0;
    if (t < nchunks) {
      lo = max(0, diag - lenB);
      int hi = min(diag, lenA);
      while (lo < hi) {                                      // first a with A[a] > B[diag-1-a]
        const int mid = (lo + hi) >> 1;
        if (buf[PADIDX(A0 + mid)] <= buf[PADIDX(B0 + diag - 1 - mid)]) lo = mid + 1; else hi = mid;
      }
    }
    s_lo[t] = lo;
    __syncthreads();
    if (t < nchunks) {
      const bool pair_end = ((out0 + VT) & (2 * L - 1)) == 0 || t + 1 >= nchunks;
      const int a_end = pair_end ? lenA : s_lo[t + 1];
      const int ai = lo, bi = diag - lo;
      const int ca = a_end - ai;
#pragma unroll
      for (int i = 0; i < VT; i++) k[i] = buf[PADIDX(i < ca ? A0 + ai + i : B0 + bi + (VT - 1 - i))];
    }
    __syncthreads();                                         // every thread has its inputs: the buffer may be overwritten
    if (t < nchunks) {
#pragma unroll
      for (int j = VT >> 1; j > 0; j >>= 1) {
#pragma unroll
        for (int i = 0; i < VT; i++) {
          const int l = i ^ j;
          if (l > i) cex(k[i], k[l]);
        }
      }
#pragma unroll
      for (int i = 0; i < VT; i++) buf[PADIDX(out0 + i)] = k[i];
    }
    __syncthreads();
  }
}

// stable LSD radix sort of n 64-bit keys, 8 bits per pass, one CTA of 256 threads, global ping-pong
__device__ void radix_global(uint64_t* a, uint64_t* b, int n, uint32_t* scratch /* >= 2560 words of shared memory */) {
  constexpr int T = 256;
  uint32_t* hist = scratch;                       // [256]
  uint32_t* digit_base = scratch + 256;           // [256]
  uint32_t (*warp_digit_cnt)[256] = reinterpret_cast<uint32_t (*)[256]>(scratch + 512);   // [8][256]
  __shared__ int skip;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  uint64_t* src = a; uint64_t* dst = b;
  for (int pass = 0; pass < 8; pass++) {
    const int shift = pass * 8;
    hist[tid] = 0;
    if (tid == 0) skip = 0;
    __syncthreads();
    for (int i = tid; i < n; i += T) atomicAdd(&hist[(src[i] >> shift) & 255u], 1u);
    __syncthreads();
    if (hist[tid] == (uint32_t)n) skip = 1;   // digit constant over the bucket: nothing to do
    __syncthreads();
    if (skip) { __syncthreads(); continue; }
    if (tid == 0) { uint32_t s = 0; for (int d = 0; d < 256; d++) { digit_base[d] = s; s += hist[d]; } }
    __syncthreads();
    for (int base = 0; base < n; base += T) {
      for (int d = lane; d < 256; d += 32) warp_digit_cnt[wid][d] = 0;
      __syncwarp();
      const int i = base + tid;
      const bool valid = i < n;
      const uint64_t key = valid ? src[i] : 0;
      const uint32_t d = (uint32_t)(key >> shift) & 255u;
      const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : 0xffffffffu);
      const uint32_t rank_in_warp = __popc(peers & ((1u << lane) - 1u));
      if (valid && rank_in_warp == 0) warp_digit_cnt[wid][d] = __popc(peers);
      __syncthreads();
      uint32_t before = 0;
      if (valid) for (int w = 0; w < wid; w++) before += warp_digit_cnt[w][d];
      if (valid) dst[digit_base[d] + before + rank_in_warp] = key;
      __syncthreads();
      { uint32_t tot = 0; for (int w = 0; w < T / 32; w++) tot += warp_digit_cnt[w][tid]; digit_base[tid] += tot; }
      __syncthreads();
    }
    uint64_t* t = src; src = dst; dst = t;
    __syncthreads();
  }
  if (src != a) { for (int i = tid; i < n; i += T) a[i] = src[i]; }
  __syncthreads();
}

// canonical form of a key for the binning buffer (what the reference's sorted key list holds in its low 32 + depth bits)
__device__ __forceinline__ uint64_t key_unpack(uint64_t k) { return (k & 0xffffffff00000000ull) | ((k >> 8) & 0xffffffull); }

// Output of one sorted tile list: Gaussian ids, reach masks, and the sorted keys in canonical form.
// PADDED: `sorted` is a shared-memory sort buffer (PADIDX layout); otherwise plain memory.
template <bool PACK, int STRIDE, bool PADDED>
__device__ __forceinline__ void emit_sorted(const uint64_t* sorted, uint64_t* bucket, int n, int first, uint32_t base,
                                            uint32_t* __restrict__ point_list, unsigned char* __restrict__ inst_mask,
                                            const float* __restrict__ rec, int tile, int gx) {
  const int tile_px = (tile % gx) * SFGS_TILE, tile_py = (tile / gx) * SFGS_TILE;
  for (int i = first; i < n; i += STRIDE) {
    const uint64_t k = sorted[PADDED ? PADIDX(i) : i];
    if (PACK) {
      bucket[i] = key_unpack(k);
      point_list[base + i] = (uint32_t)(k >> 8) & 0xffffffu;
      inst_mask[base + i] = (unsigned char)(k & 0xffu);
    } else {
      const uint32_t id = (uint32_t)k;
      if (PADDED) bucket[i] = k;
      point_list[base + i] = id;
      const float4 r0 = *reinterpret_cast<const float4*>(rec + (size_t)id * REC_FLOATS);
      const float2 r1 = *reinterpret_cast<const float2*>(rec + (size_t)id * REC_FLOATS + 4);
      inst_mask[base + i] = (unsigned char)reach_mask(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, tile_px, tile_py);
    }
  }
}

// ---- lists of up to 512 instances: one WARP per tile ------------------------------------------------------------------
// Every tile of the benchmark frames (130..490 instances) is in this class.  A CTA-wide sort of such a list keeps one or
// two of its warps busy and parks the others at the pass barriers (ncu, round 2a: 4.9 barrier-stall cycles per issued
// instruction, 19 of 32 lanes active, 51 % of the issue slots).  Here a warp owns a tile: lane t sorts VT keys in
// registers (bitonic network, VT = 4 / 8 / 16 by list length), then log2(n/VT) merge-path passes run over two private
// shared-memory buffers with only __syncwarp between them; four independent tiles per CTA, nothing block-wide.
constexpr int WS_MAX = 512;           // longest list of the warp class
constexpr int WS_WARPS = 4;           // tiles per CTA

// Merge passes WITHOUT a serial merge loop.  A sequential two-pointer merge out of shared memory is one dependent
// load -> compare -> select chain per output key (ncu, first version of this kernel: 9.3 short-scoreboard stall cycles
// per issued instruction, 28 % of the issue slots, ~63 k cycles per tile).  Here a lane
//   1. finds its merge-path split (ai, bi) by binary search — the only serial chain left, log2(L) steps;
//   2. learns from its right neighbour's split how many of its VT outputs come from run A (ca) and run B (VT - ca);
//   3. loads exactly those keys with VT INDEPENDENT shared-memory loads — A's ascending, B's in DESCENDING order, so the
//      VT registers hold a bitonic sequence;
//   4. sorts them with the log2(VT)-stage bitonic merge network (compile-time register indices, VT/2 independent
//      compare-exchanges per stage) and stores them over the same buffer (all lanes have loaded: __syncwarp).
// One shared buffer instead of two (4 KB per warp: twice the resident warps) and ~2400 issued instructions per
// 276-key list, most of them independent.
template <int VT>
__device__ __forceinline__ void warp_merge_sort(uint64_t* buf, const uint64_t* __restrict__ bucket, int n, int lane) {
  const int nchunks = (n + VT - 1) / VT;       // <= 32
  const int n_pad = nchunks * VT;
  uint64_t k[VT];
  if (lane < nchunks) {
#pragma unroll
    for (int i = 0; i < VT; i++) { const int idx = lane * VT + i; k[i] = idx < n ? bucket[idx] : ~0ull; }
    // bitonic sorting network over the VT registers (all indices are compile-time constants after unrolling)
#pragma unroll
    for (int kk = 2; kk <= VT; kk <<= 1) {
#pragma unroll
      for (int j = kk >> 1; j > 0; j >>= 1) {
#pragma unroll
        for (int i = 0; i < VT; i++) {
          const int l = i ^ j;
          if (l > i) {
            const bool up = (i & kk) == 0;
            const uint64_t lo = min(k[i], k[l]), hi = max(k[i], k[l]);
            k[i] = up ? lo : hi; k[l] = up ? hi : lo;
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < VT; i++) buf[PADIDX(lane * VT + i)] = k[i];
  }
  __syncwarp();
  for (int L = VT; L < n_pad; L <<= 1) {
    const int out0 = lane * VT;
    const int pair0 = out0 & ~(2 * L - 1);
    const int lenA = min(L, max(0, n_pad - pair0));
    const int lenB = min(L, max(0, n_pad - pair0 - L));
    const int A0 = pair0, B0 = pair0 + L;                    // first keys of the two runs (logical indices)
    const int diag = out0 - pair0;
    int lo = 0;
    if (lane < nchunks) {
      lo = max(0, diag - lenB);
      int hi = min(diag, lenA);
      while (lo < hi) {                                      // first a with A[a] > B[diag-1-a]
        const int mid = (lo + hi) >> 1;
        if (buf[PADIDX(A0 + mid)] <= buf[PADIDX(B0 + diag - 1 - mid)]) lo = mid + 1; else hi = mid;
      }
    }
    // split of the NEXT diagonal (diag + VT): the right neighbour's, or the end of run A at the end of the pair
    const int lo_next = __shfl_down_sync(0xffffffffu, lo, 1);
    if (lane < nchunks) {
      const bool pair_end = ((out0 + VT) & (2 * L - 1)) == 0 || lane + 1 >= nchunks;
      const int a_end = pair_end ? lenA : lo_next;
      const int ai = lo, bi = diag - lo;
      const int ca = a_end - ai;                             // keys taken from run A; VT - ca from run B
#pragma unroll
      for (int i = 0; i < VT; i++) k[i] = buf[PADIDX(i < ca ? A0 + ai + i : B0 + bi + (VT - 1 - i))];
    }
    __syncwarp();                                            // every lane has its inputs: the buffer may be overwritten
    if (lane < nchunks) {
#pragma unroll
      for (int j = VT >> 1; j > 0; j >>= 1) {
#pragma unroll
        for (int i = 0; i < VT; i++) {
          const int l = i ^ j;
          if (l > i) cex(k[i], k[l]);
        }
      }
#pragma unroll
      for (int i = 0; i < VT; i++) buf[PADIDX(out0 + i)] = k[i];
    }
    __syncwarp();
  }
}

template <bool PACK>
__global__ void __launch_bounds__(WS_WARPS * 32)
tile_sort_warp_kernel(int tiles, const uint2* __restrict__ ranges, const uint32_t* __restrict__ hdr, uint64_t* __restrict__ keys,
                      uint32_t* __restrict__ point_list, const float* __restrict__ rec, int gx,
                      unsigned char* __restrict__ inst_mask) {
  if (hdr[HDR_OVERFLOW]) return;
  __shared__ __align__(16) uint64_t s_keys[WS_WARPS][WS_MAX + WS_MAX / 16];      // 17 KB
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int tile = blockIdx.x * WS_WARPS + wid;
  if (tile >= tiles) return;
  const uint2 rg = ranges[tile];
  const int n = (int)(rg.y - rg.x);
  if (n == 0 || n > WS_MAX) return;               // empty, or a tile of the CTA-wide classes
  uint64_t* bucket = keys + rg.x;
  uint64_t* buf = s_keys[wid];
  if (n <= 32 * 4) warp_merge_sort<4>(buf, bucket, n, lane);
  else if (n <= 32 * 8) warp_merge_sort<8>(buf, bucket, n, lane);
  else warp_merge_sort<16>(buf, bucket, n, lane);
  emit_sorted<PACK, 32, true>(buf, bucket, n, lane, rg.x, point_list, inst_mask, rec, tile, gx);
}

// ---- longer lists: one CTA of 256 threads per tile, a small persistent grid strides over the tiles ----------------------
// (a grid of one CTA per tile costs ~8 us of CTA launches even when no tile of the class exists — ncu, round 2b — and
// the benchmark frames have none; here the CTAs return after one header read in that case).  Lists of 513..1024 keys
// are sorted with 4 keys per thread, 1025..4096 with 16, longer ones by the global radix fallback.
constexpr int CS_THREADS = 256;
constexpr int CS_WINDOW = 4096;
template <bool PACK>
__global__ void __launch_bounds__(CS_THREADS, 3)
tile_sort_kernel(int tiles, const uint2* __restrict__ ranges, const uint32_t* __restrict__ hdr, uint64_t* __restrict__ keys,
                 uint64_t* __restrict__ keys_tmp, uint32_t* __restrict__ point_list,
                 const float* __restrict__ rec, int gx, unsigned char* __restrict__ inst_mask) {
  if (hdr[HDR_OVERFLOW] || hdr[HDR_MAXTILE] <= (uint32_t)WS_MAX) return;   // every list is in the warp class
  extern __shared__ __align__(16) unsigned char sort_smem[];
  // [PADIDX(CS_WINDOW)] keys + [CS_THREADS + 1] splits; the oversized-tile radix path reuses the space as 2560 scratch words
  uint64_t* s = reinterpret_cast<uint64_t*>(sort_smem);
  int* s_lo = reinterpret_cast<int*>(s + CS_WINDOW + CS_WINDOW / 16);
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {     // block-uniform
    const uint2 rg = ranges[tile];
    const int n = (int)(rg.y - rg.x);
    if (n <= WS_MAX) continue;                                       // warp class (or empty)
    uint64_t* bucket = keys + rg.x;
    if (n <= CS_WINDOW) {
      if (n <= CS_THREADS * 4) merge_sort_smem<CS_THREADS, 4>(s, s_lo, bucket, n);
      else merge_sort_smem<CS_THREADS, 16>(s, s_lo, bucket, n);
      emit_sorted<PACK, CS_THREADS, true>(s, bucket, n, threadIdx.x, rg.x, point_list, inst_mask, rec, tile, gx);
    } else {
      radix_global(bucket, keys_tmp + rg.x, n, reinterpret_cast<uint32_t*>(s));
      emit_sorted<PACK, CS_THREADS, false>(bucket, bucket, n, threadIdx.x, rg.x, point_list, inst_mask, rec, tile, gx);
    }
    __syncthreads();     // the shared buffer is reused by the next tile
  }
}

}  // namespace

void sfgs_launch_tile_scan(const ImageLayout& im, unsigned long long capacity, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  tile_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(im.tiles, im.tile_count, im.ranges, im.hdr, capacity);
}

// Gaussian ids below 2^24 ride in the key together with the reach mask (see scatter_keys_kernel)
static inline bool sfgs_keys_packed(int P) {
  // SFGS_KEYS_PACKED=0 forces the unpacked path (what P > 2^24 takes) so that the tests can run it on small scenes
  static const bool allow = [] { const char* e = getenv("SFGS_KEYS_PACKED"); return !(e && e[0] == '0'); }();
  return allow && P <= (1 << 24);
}

void sfgs_launch_scatter(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P,
                         unsigned long long capacity, cudaStream_t st) {
  SFGS_COUNT_LAUNCH();
  if (capacity == 0) return;
  auto blocks_for = [&](int it) { return (unsigned)((capacity + 256ull * it - 1) / (256ull * it)); };
  if (sfgs_keys_packed(P)) scatter_keys_kernel<true, 2><<<blocks_for(2), 256, 0, st>>>(b.tmp, im.ranges, im.tile_count, im.hdr, g.rec, im.tiles_x, b.keys);
  else scatter_keys_kernel<false, 4><<<blocks_for(4), 256, 0, st>>>(b.tmp, im.ranges, im.tile_count, im.hdr, g.rec, im.tiles_x, b.keys);
}

template <bool PACK>
static void launch_tile_sorts(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, cudaStream_t st) {
  constexpr size_t smem_cta = (CS_WINDOW + CS_WINDOW / 16) * sizeof(uint64_t) + (CS_THREADS + 1) * sizeof(int);
  static SfgsPerDeviceOnce attr_once;   // function attributes are per device
  if (attr_once.first_use()) {
    cudaFuncSetAttribute(tile_sort_kernel<PACK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cta);
  }
  SFGS_COUNT_LAUNCH();
  tile_sort_warp_kernel<PACK><<<(im.tiles + WS_WARPS - 1) / WS_WARPS, WS_WARPS * 32, 0, st>>>(
      im.tiles, im.ranges, im.hdr, b.keys, b.point_list, g.rec, im.tiles_x, b.inst_mask);
  // lists beyond the warp class: a persistent grid (three resident CTAs per SM) that returns at once when the frame's
  // longest list (header word written by the scan) is inside the warp class
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  { int v = 0; if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) sms = v; }
  const int grid_cta = im.tiles < 3 * sms ? im.tiles : 3 * sms;
  SFGS_COUNT_LAUNCH();
  tile_sort_kernel<PACK><<<grid_cta, CS_THREADS, smem_cta, st>>>(im.tiles, im.ranges, im.hdr, b.keys, b.keys_tmp, b.point_list,
                                                                  g.rec, im.tiles_x, b.inst_mask);
}

void sfgs_launch_tile_sort(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P, cudaStream_t st) {
  if (sfgs_keys_packed(P)) launch_tile_sorts<true>(g, im, b, st);
  else launch_tile_sorts<false>(g, im, b, st);
}
