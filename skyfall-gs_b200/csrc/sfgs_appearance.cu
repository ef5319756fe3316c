// sfgs_appearance.cu — the appearance path of render() as one tensor-core kernel (SURVEY.md 8f rank 2).
//
// Replaces, for the forward pass, gaussian_renderer/__init__.py:105-118 + EmbeddingModel.forward
// (scene/gaussian_model.py:45-69) + eval_sh (utils/sh_utils.py) — in torch: a [P,59] concat, three Linear layers with
// [P,128] fp32 intermediates, a repeat, a [P,3M] tone map, a [P,3,M] transpose, the SH evaluation and four clamps,
// ~25 kernels and ~2.5 KB of HBM traffic per Gaussian at M = 16 — by one kernel that reads each Gaussian's 3M SH
// features, 24 Fourier features and position once and writes its 3 colours (324 B per Gaussian at M = 16):
//
//   inp    = [min(features[:3], 1) | gemb | aemb]                      (59 = 3 + 24 + 32)
//   h      = W3 relu(W2 relu(W1 inp + b1) + b2) + b3 ;  offset, mul = 0.01 h[:3], 0.01 h[3:]
//   toned  = min(min(features, 1) * mul[ch] + [offset/C0 on the DC term], 1)            ([M,3] per Gaussian)
//   colour = max(eval_sh(D, toned, normalize(xyz - campos)) + 0.5, 0)
//
// M = (max_sh_degree + 1)^2 is a template parameter (1, 4, 9 or 16).  Layer 1 reads only the three DC values, so the
// GEMMs do not depend on it; M sets the feature row stride (3M floats), the L2 prefetch span and the length of the
// tone-map / eval_sh loop.  Rows are loaded as float4 only when M % 4 == 0: 12- and 108-byte rows are not 16-byte
// aligned.
//
// The per-camera embedding `aemb` is the same vector for every Gaussian, so its 32 columns of W1 fold into the bias
// (b1' = b1 + W1[:, 27:] aemb, computed once per CTA) and layer 1 contracts over K = 27 (padded to 32).
//
// Tensor cores: a CTA owns a tile of 128 Gaussians per warpgroup; each GEMM — [128x32]x[32x128], [128x128]x[128x128],
// [128x128]x[128x16] — runs as two m64 halves of wgmma.mma_async (bf16 operands from shared memory, fp32 accumulate in
// registers).  Weights are converted to bf16 once per CTA and stay in shared memory in the canonical K-major
// no-swizzle core-matrix layout (8 rows x 16 bytes per core; SBO = 128 B between 8-row groups, LBO = bytes between
// the two 16-byte K chunks of one k16 step); activations never leave the SM: thread m packs row m of the A operand
// into the same layout, the warpgroup issues the MMAs, and each thread applies bias + ReLU + bf16 pack to the
// accumulator fragment it holds, writing the next layer's A operand in place.  CTAs are persistent over tiles and
// run TWO tiles at a time: two warpgroups, each with its own operand buffer, synchronised only inside the group
// (named barriers), so one group's epilogue arithmetic overlaps the other group's MMAs and loads.
//
// Precision: the multiplier head of a trained model is O(1) (h ~ 100 before the x0.01), so plain bf16 operands
// (2^-9 relative) would leave ~1e-2 in the colours (measured on the golden vectors: 8e-3).  Every operand is therefore
// carried as TWO bf16 values, x = hi + lo with lo = bf16(x - hi) (16 mantissa bits together), and every product is
// three tensor-core MMAs into the same fp32 accumulator:  A W ~= Ah Wh + Ah Wl + Al Wh  (the dropped Al Wl term is
// 2^-18 relative).  The GEMMs stay on the tensor cores at 3x the MMA count — still far below the kernel's HBM time —
// and the colours agree with the reference's float32 modules to 1e-4 (tests/test_appearance.py).  Everything after
// the MLP is float32.
#include <cuda_bf16.h>
#include <cstdio>
#include <initializer_list>
#include "sfgs_common.cuh"

namespace {

constexpr int AP_THREADS = 256;       // two warpgroups, each with its own tile in flight
constexpr int AP_GROUPS = 2;
constexpr int AP_M = 128;            // Gaussians per tile
constexpr int AP_H = 128;            // hidden width
constexpr int AP_K1 = 32;            // 3 + 24 padded
constexpr int AP_N3 = 16;            // 6 outputs padded to a multiple of the MMA's N granularity
constexpr int AP_G = 24, AP_E = 32;  // Fourier features per Gaussian, per-camera embedding size

struct alignas(128) ApSmem {                       // [2] = {hi, lo} halves of the split operands
  __nv_bfloat16 A[AP_GROUPS][2][AP_H / 8][AP_M / 8][8][8];   // 2 x 64 KB  activations, K-major cores: [k chunk][row group][row][8 k]
  __nv_bfloat16 W1[2][AP_K1 / 8][AP_H / 8][8][8];   // 16 KB  [k chunk][n group][n][8 k]
  __nv_bfloat16 W2[2][AP_H / 8][AP_H / 8][8][8];    // 64 KB
  __nv_bfloat16 W3[2][AP_H / 8][AP_N3 / 8][8][8];   //  8 KB
  float h3[AP_GROUPS][AP_M][8];                     //  8 KB  layer-3 outputs, row m -> thread m
  float b1[AP_H], b2[AP_H], b3[8];
};
static_assert(sizeof(ApSmem) <= 227 * 1024, "appearance tile buffers exceed the shared memory of one SM");

using ApTile = __nv_bfloat16[2][AP_H / 8][AP_M / 8][8][8];

__device__ __forceinline__ uint64_t smem_desc(const void* p, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  // wgmma shared-memory matrix descriptor, no swizzle: start >> 4 in [0,14), LBO >> 4 in [16,30), SBO >> 4 in [32,46),
  // base offset 0, swizzle mode 0 in [62,64)
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  return (uint64_t)((a >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
// D (+)= A B with A = 64 x 16 and B = 16 x N, both K-major in shared memory; D is the warpgroup's register fragment:
// d[4 j + 2 r + e] is row 16 (warp % 4) + lane / 4 + 8 r, column 8 j + 2 (lane % 4) + e
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
               " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
               " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
               " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
               "%64, %65, p, 1, 1, 0, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                 "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                 "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                 "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1, 0, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// One m64 half of a layer, split-bf16: acc = Ah Wh + Ah Wl + Al Wh over K = 16 KSTEPS.  a_hi / a_lo point at the
// half's first core matrix in K chunk 0 (K chunks of A are AP_M x 8 elements apart); w_hi / w_lo at W's K chunk 0.
template <int N, int KSTEPS>
__device__ __forceinline__ void mma_half(float (&acc)[N / 2], const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo,
                                         const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo) {
#pragma unroll
  for (int i = 0; i < N / 2; i++) acc[i] = 0.f;
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
  for (int ks = 0; ks < KSTEPS; ks++) {
    const uint64_t ah = smem_desc(a_hi + ks * 2 * AP_M * 8, AP_M * 16, 128), al = smem_desc(a_lo + ks * 2 * AP_M * 8, AP_M * 16, 128);
    const uint64_t wh = smem_desc(w_hi + ks * 2 * N * 8, N * 16, 128), wl = smem_desc(w_lo + ks * 2 * N * 8, N * 16, 128);
    if constexpr (N == 128) {
      wgmma_n128(acc, ah, wh, ks > 0); wgmma_n128(acc, ah, wl, 1); wgmma_n128(acc, al, wh, 1);
    } else {
      wgmma_n16(acc, ah, wh, ks > 0); wgmma_n16(acc, ah, wl, 1); wgmma_n16(acc, al, wh, 1);
    }
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// relu(acc + bias) of this thread's fragment -> split bf16 into the A operand (rows row0 + lane/4 + {0, 8})
__device__ __forceinline__ void store_hidden(const float (&acc)[64], const float* bias, ApTile& A, int row0, int lane) {
#pragma unroll
  for (int j = 0; j < AP_H / 8; j++) {
    const int col = 8 * j + 2 * (lane & 3);
    const float b0 = bias[col], b1 = bias[col + 1];
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const int row = row0 + (lane >> 2) + 8 * r;
      const float x0 = fmaxf(acc[4 * j + 2 * r] + b0, 0.f), x1 = fmaxf(acc[4 * j + 2 * r + 1] + b1, 0.f);
      const __nv_bfloat162 hi = __floats2bfloat162_rn(x0, x1);
      const __nv_bfloat162 lo = __floats2bfloat162_rn(x0 - __low2float(hi), x1 - __high2float(hi));
      *reinterpret_cast<__nv_bfloat162*>(&A[0][j][row >> 3][row & 7][col & 7]) = hi;
      *reinterpret_cast<__nv_bfloat162*>(&A[1][j][row >> 3][row & 7][col & 7]) = lo;
    }
  }
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
  __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]), d = __floats2bfloat162_rn(v[6], v[7]);
  return make_uint4(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&b), *reinterpret_cast<uint32_t*>(&c),
                    *reinterpret_cast<uint32_t*>(&d));
}
// x = hi + lo: hi = bf16(x), lo = bf16(x - hi)
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  float r[8];
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = v[i] - __bfloat162float(__float2bfloat16(v[i]));
  hi = pack8(v);
  lo = pack8(r);
}
__device__ __forceinline__ void split_store(__nv_bfloat16* hi, __nv_bfloat16* lo, float x) {
  const __nv_bfloat16 h = __float2bfloat16(x);
  *hi = h;
  *lo = __float2bfloat16(x - __bfloat162float(h));
}

template <int M>
__global__ void __launch_bounds__(AP_THREADS, 1)
appearance_fwd_kernel(int P, int D, const float* __restrict__ features /*[P,M,3]*/, const float* __restrict__ gemb /*[P,24]*/,
                      const float* __restrict__ aemb /*[32]*/, const float* __restrict__ W1 /*[128,59]*/,
                      const float* __restrict__ b1, const float* __restrict__ W2 /*[128,128]*/, const float* __restrict__ b2,
                      const float* __restrict__ W3 /*[6,128]*/, const float* __restrict__ b3,
                      const float* __restrict__ means3D, const float* __restrict__ campos, float* __restrict__ colors) {
  extern __shared__ __align__(128) unsigned char ap_smem[];
  ApSmem& S = *reinterpret_cast<ApSmem*>(ap_smem);
  const int tid = threadIdx.x, lane = tid & 31;
  const int grp = tid >> 7, t = tid & 127;       // warpgroup and row inside the group's tile
  const int wrow = 16 * ((tid >> 5) & 3);        // first accumulator row of this warp inside an m64 half
  constexpr int IN = 3 + AP_G + AP_E;     // 59 columns of W1
  auto group_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory"); };

  // ---- once per CTA: weights -> bf16 core-matrix layout, folded bias
  for (int i = tid; i < AP_H * AP_K1; i += AP_THREADS) {          // W1[n][k], k < 27 (colour 3 + Fourier 24), zero padded
    const int n = i / AP_K1, k = i - n * AP_K1;
    split_store(&S.W1[0][k >> 3][n >> 3][n & 7][k & 7], &S.W1[1][k >> 3][n >> 3][n & 7][k & 7], k < 3 + AP_G ? W1[n * IN + k] : 0.f);
  }
  for (int i = tid; i < AP_H * AP_H; i += AP_THREADS) {
    const int n = i / AP_H, k = i - n * AP_H;
    split_store(&S.W2[0][k >> 3][n >> 3][n & 7][k & 7], &S.W2[1][k >> 3][n >> 3][n & 7][k & 7], W2[i]);
  }
  for (int i = tid; i < AP_N3 * AP_H; i += AP_THREADS) {
    const int n = i / AP_H, k = i - n * AP_H;
    split_store(&S.W3[0][k >> 3][n >> 3][n & 7][k & 7], &S.W3[1][k >> 3][n >> 3][n & 7][k & 7], n < 6 ? W3[n * AP_H + k] : 0.f);
  }
  if (tid < AP_H) {
    float acc = b1[tid];
#pragma unroll 8
    for (int e = 0; e < AP_E; e++) acc = fmaf(W1[tid * IN + 3 + AP_G + e], aemb[e], acc);
    S.b1[tid] = acc;
    S.b2[tid] = b2[tid];
    if (tid < 8) S.b3[tid] = tid < 6 ? b3[tid] : 0.f;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the MMA's async proxy
  __syncthreads();
  ApTile& A = S.A[grp];
  const float cx = campos[0], cy = campos[1], cz = campos[2];

  const int ntiles = (P + AP_M - 1) / AP_M;
  // One thread per group asks L2 for the NEXT tile's rows (three contiguous spans) while this tile is computed: the
  // row-per-thread loads below then find their lines in L2 instead of paying the HBM latency in the critical path.
  auto prefetch_tile = [&](int tl) {
    if (tl >= ntiles) return;
    const int r0 = tl * AP_M;
    const unsigned rows = (unsigned)((P - r0) < AP_M ? (P - r0) : AP_M);
    const float* pf = features + (size_t)r0 * (3 * M);     // r0 * 12M bytes: 16-byte aligned, as r0 is a multiple of 128
    const float* pg = gemb + (size_t)r0 * AP_G;
    const float* pm = means3D + (size_t)r0 * 3;
    const unsigned fb = (rows * (12u * M)) & ~15u;           // zero only for M = 1 and a single row
    if (M % 4 == 0 || fb) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pf), "r"(fb) : "memory");
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pg), "r"(rows * (unsigned)(AP_G * 4)) : "memory");
    const unsigned mb = (rows * 12u) & ~15u;
    if (mb && (reinterpret_cast<uintptr_t>(pm) & 15) == 0)
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pm), "r"(mb) : "memory");
  };
  for (int tile = blockIdx.x * AP_GROUPS + grp; tile < ntiles; tile += gridDim.x * AP_GROUPS) {
    if (t == 0) prefetch_tile(tile + gridDim.x * AP_GROUPS);
    const int g = tile * AP_M + t;
    const bool valid = g < P;
    const int gi = valid ? g : P - 1;                                   // rows past P shadow the last Gaussian
    // ---- A0: row m = [min(dc, 1) (3) | Fourier features (24) | 0 (5)]
    {
      float in[AP_K1];
      const float* f = features + (size_t)gi * (3 * M);
      in[0] = fminf(f[0], 1.f); in[1] = fminf(f[1], 1.f); in[2] = fminf(f[2], 1.f);
      const float4* g4 = reinterpret_cast<const float4*>(gemb + (size_t)gi * AP_G);
#pragma unroll
      for (int q = 0; q < AP_G / 4; q++) {
        const float4 v = g4[q];
        in[3 + 4 * q] = v.x; in[4 + 4 * q] = v.y; in[5 + 4 * q] = v.z; in[6 + 4 * q] = v.w;
      }
#pragma unroll
      for (int k = 3 + AP_G; k < AP_K1; k++) in[k] = 0.f;
#pragma unroll
      for (int kc = 0; kc < AP_K1 / 8; kc++) {
        uint4 hi, lo;
        split8(in + 8 * kc, hi, lo);
        *reinterpret_cast<uint4*>(&A[0][kc][t >> 3][t & 7][0]) = hi;
        *reinterpret_cast<uint4*>(&A[1][kc][t >> 3][t & 7][0]) = lo;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    group_sync();
    // ---- layers 1 and 2: [128 x 32] x [32 x 128], then [128 x 128] x [128 x 128]; h = relu(acc + b) -> A (K = 128).
    // A half's output rows overwrite only that half's input rows, which its own MMAs have finished reading.
#pragma unroll 1
    for (int layer = 0; layer < 2; layer++) {
#pragma unroll 1
      for (int half = 0; half < 2; half++) {
        float acc[64];
        if (layer == 0)
          mma_half<AP_H, AP_K1 / 16>(acc, &A[0][0][8 * half][0][0], &A[1][0][8 * half][0][0], &S.W1[0][0][0][0][0], &S.W1[1][0][0][0][0]);
        else
          mma_half<AP_H, AP_H / 16>(acc, &A[0][0][8 * half][0][0], &A[1][0][8 * half][0][0], &S.W2[0][0][0][0][0], &S.W2[1][0][0][0][0]);
        group_sync();      // the whole warpgroup is past its wait before any row of the half is rewritten
        store_hidden(acc, layer == 0 ? S.b1 : S.b2, A, 64 * half + wrow, lane);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      group_sync();
    }
    // ---- layer 3: [128 x 128] x [128 x 16]; columns 0..7 of row m -> h3[m]
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
      float acc[8];
      mma_half<AP_N3, AP_H / 16>(acc, &A[0][0][8 * half][0][0], &A[1][0][8 * half][0][0], &S.W3[0][0][0][0][0], &S.W3[1][0][0][0][0]);
#pragma unroll
      for (int r = 0; r < 2; r++)
        *reinterpret_cast<float2*>(&S.h3[grp][64 * half + wrow + (lane >> 2) + 8 * r][2 * (lane & 3)]) =
            make_float2(acc[2 * r], acc[2 * r + 1]);
    }
    group_sync();
    float h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = S.h3[grp][t][i];

    // ---- tone map + SH evaluation (fp32), scene/gaussian_model.py:60-69, gaussian_renderer/__init__.py:109-117
    float off[3], mul[3];
#pragma unroll
    for (int c = 0; c < 3; c++) { off[c] = (h[c] + S.b3[c]) * 0.01f / SH_C0; mul[c] = (h[3 + c] + S.b3[3 + c]) * 0.01f; }
    const float px = means3D[3 * (size_t)gi], py = means3D[3 * (size_t)gi + 1], pz = means3D[3 * (size_t)gi + 2];
    float dx = px - cx, dy = py - cy, dz = pz - cz;
    const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
    const float x = dx * inv, y = dy * inv, z = dz * inv;
    float bas[16];
    bas[0] = SH_C0;
    bas[1] = -SH_C1 * y; bas[2] = SH_C1 * z; bas[3] = -SH_C1 * x;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    bas[4] = SH_C2_0 * xy; bas[5] = SH_C2_1 * yz; bas[6] = SH_C2_2 * (2.f * zz - xx - yy); bas[7] = SH_C2_3 * xz;
    bas[8] = SH_C2_4 * (xx - yy);
    bas[9] = SH_C3_0 * y * (3.f * xx - yy); bas[10] = SH_C3_1 * xy * z; bas[11] = SH_C3_2 * y * (4.f * zz - xx - yy);
    bas[12] = SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy); bas[13] = SH_C3_4 * x * (4.f * zz - xx - yy);
    bas[14] = SH_C3_5 * z * (xx - yy); bas[15] = SH_C3_6 * x * (xx - 3.f * yy);
    const int ncoef = (D + 1) * (D + 1);
    float rgb[3] = {0.f, 0.f, 0.f};
    auto tone_sh = [&](int j, float e) {                               // features[k][ch], j = 3 k + ch
      const int k = j / 3, ch = j - 3 * k;
      float tv = fminf(e, 1.f) * mul[ch] + (k == 0 ? off[ch] : 0.f);
      tv = fminf(tv, 1.f);
      if (k < ncoef) rgb[ch] = fmaf(bas[k], tv, rgb[ch]);
    };
    const float* fr = features + (size_t)gi * (3 * M);
    if constexpr (M % 4 == 0) {
      const float4* f4 = reinterpret_cast<const float4*>(fr);
#pragma unroll
      for (int q = 0; q < 3 * M / 4; q++) {
        const float4 v = f4[q];
        tone_sh(4 * q, v.x); tone_sh(4 * q + 1, v.y); tone_sh(4 * q + 2, v.z); tone_sh(4 * q + 3, v.w);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 3 * M; j++) tone_sh(j, fr[j]);
    }
    if (valid) {
      colors[3 * (size_t)g] = fmaxf(rgb[0] + 0.5f, 0.f);
      colors[3 * (size_t)g + 1] = fmaxf(rgb[1] + 0.5f, 0.f);
      colors[3 * (size_t)g + 2] = fmaxf(rgb[2] + 0.5f, 0.f);
    }
    group_sync();      // every thread has read h3 and every MMA has finished with A before the next tile rewrites them
  }
}

}  // namespace

extern "C" int sfgs_set_error(int code, const char* what, int cuda_error);   // sfgs_api.cu

// Argument checks of both appearance entry points, made before any pointer is read or any CUDA call: `params` are the
// camera and MLP arrays, `rows` the per-Gaussian ones (which may be NULL when P = 0).  Returns 0 or the error code.
static int appearance_check(const char* fn, int P, int D, int M, int G, int E, std::initializer_list<const void*> params,
                            std::initializer_list<const void*> rows, const float* features, const float* gemb) {
  char msg[192];
  if ((M != 1 && M != 4 && M != 9 && M != 16) || G != AP_G || E != AP_E || D < 0 || D > 3) {
    snprintf(msg, sizeof(msg), "%s: built for 1, 4, 9 or 16 SH coefficients, 24 Fourier features, a 32-wide embedding", fn);
    return sfgs_set_error(SFGS_E_UNSUPPORTED, msg, 0);
  }
  if ((D + 1) * (D + 1) > M) {
    snprintf(msg, sizeof(msg), "%s: active SH degree D needs (D+1)^2 <= M coefficients", fn);
    return sfgs_set_error(SFGS_E_BADARG, msg, 0);
  }
  bool null = false;
  for (const void* q : params) null |= q == nullptr;
  if (P > 0)
    for (const void* q : rows) null |= q == nullptr;
  if (null) {
    snprintf(msg, sizeof(msg), "%s: null pointer", fn);
    return sfgs_set_error(SFGS_E_BADARG, msg, 0);
  }
  if (P > 0 && ((reinterpret_cast<uintptr_t>(features) & 15) || (reinterpret_cast<uintptr_t>(gemb) & 15))) {
    snprintf(msg, sizeof(msg), "%s: features / gemb must be 16-byte aligned", fn);
    return sfgs_set_error(SFGS_E_BADARG, msg, 0);
  }
  return 0;
}

extern "C" int sfgs_appearance_forward(int P, int D, int M, const float* features, const float* gemb, int G, const float* aemb,
                                       int E, const float* W1, const float* b1, const float* W2, const float* b2,
                                       const float* W3, const float* b3, const float* means3D, const float* campos,
                                       float* colors, void* stream) {
  if (P < 0) return sfgs_set_error(SFGS_E_BADARG, "appearance_forward: P < 0", 0);
  if (P == 0) return SFGS_OK;
  const int bad = appearance_check("appearance_forward", P, D, M, G, E, {aemb, W1, b1, W2, b2, W3, b3, campos},
                                   {features, gemb, means3D, colors}, features, gemb);
  if (bad) return bad;
  using Kernel = void (*)(int, int, const float*, const float*, const float*, const float*, const float*, const float*,
                          const float*, const float*, const float*, const float*, const float*, float*);
  const Kernel kernels[4] = {appearance_fwd_kernel<1>, appearance_fwd_kernel<4>, appearance_fwd_kernel<9>, appearance_fwd_kernel<16>};
  const Kernel kernel = kernels[M == 1 ? 0 : M == 4 ? 1 : M == 9 ? 2 : 3];
  static SfgsPerDeviceOnce once;
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (once.first_use() || (dev >= 0 && dev < 64 && sms[dev] == 0)) {
    for (const Kernel k : kernels) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ApSmem));
    int n = 132;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (dev >= 0 && dev < 64) sms[dev] = n;
  }
  const int nsm = (dev >= 0 && dev < 64 && sms[dev] > 0) ? sms[dev] : 132;
  const int ntiles = (P + AP_M - 1) / AP_M;
  const int pairs = (ntiles + AP_GROUPS - 1) / AP_GROUPS;
  const int grid = pairs < nsm ? pairs : nsm;                // persistent: one CTA (two tile groups) per SM
  SFGS_COUNT_LAUNCH();
  kernel<<<grid, AP_THREADS, sizeof(ApSmem), (cudaStream_t)stream>>>(P, D, features, gemb, aemb, W1, b1, W2, b2, W3, b3,
                                                                   means3D, campos, colors);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : sfgs_set_error(SFGS_E_CUDA, "appearance_forward", (int)e);
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward: sfgs_appearance_backward, float32 on the CUDA cores.
//
// The gradients are float32 arithmetic throughout (FFMA; no tensor cores, no split operands), so they carry float32
// rounding only.  Per tile of AB_T = 64 Gaussians a CTA of 256 threads recomputes the forward in float32 — layer 1
// over K = 27 (the embedding folded into the bias as in the forward), layer 2, layer 3, the tone map and eval_sh —
// then runs the adjoint: colour clamp, eval_sh and normalize, the two clamps of the toned coefficients, the tone
// map, x0.01, dh2 = W3^T dz3, dh1 = W2^T dz2 and d[dc | gemb] = W1[:, :27]^T dz1.  Activations stay in shared
// memory (h1 then dz1 as [p][n], h2 then dz2 as [n][p]); every GEMM is register-blocked over 4 x 8 or 8 x 8 outputs
// per thread, with float4 shared loads laid out so that a warp's loads are broadcasts or conflict-free.
//
// Subgradients are torch's: clamp_max passes the gradient where x <= max, clamp_min where x >= min, ReLU where its
// output is > 0.
//
// Reductions over Gaussians (dW1[:, :27], dW2, dW3, the biases, sum dz1 and sum dL/dxyz) are deterministic: the
// Gaussians are split into chunks of C = max(512, 64 ceil(P / 65536)) — a function of P alone — one CTA per chunk.
// Each output element of a chunk's sums is owned by one thread and accumulated in Gaussian order, in float32 for the
// weight gradients and in float64 for the bias, sum-dz1 and position sums (plain sums of terms that cancel); the
// chunk partials go to scratch as float32, and a second kernel adds them in float64 in chunk order and rounds once.  dW1[:, 27:]
// = (sum dz1) x aemb, db1 = sum dz1 and dL/daemb = W1[:, 27:]^T sum dz1 are formed from the float64 sum dz1.  No
// float atomics anywhere, so repeated calls are bit-identical.
namespace {

constexpr int AB_THREADS = 256;
constexpr int AB_T = 64;                 // Gaussians per tile
constexpr int AB_LDH = AP_H + 4;         // row stride of [row][128] buffers: consecutive rows 4 banks apart
constexpr int AB_LDP = AB_T + 4;         // row stride of the [128][64] buffer
constexpr int AB_K1 = 28;                // layer-1 inputs (3 + 24) and one zero column
constexpr int AB_LDX = 32;
// per-chunk partial sums, in this order
constexpr int RO_W2 = 0, RO_W1 = RO_W2 + AP_H * AP_H, RO_W3 = RO_W1 + AP_H * 27, RO_B1 = RO_W3 + 6 * AP_H,
              RO_B2 = RO_B1 + AP_H, RO_B3 = RO_B2 + AP_H, RO_XYZ = RO_B3 + 6, AB_NRED = RO_XYZ + 3;
constexpr int AB_PSTRIDE = (AB_NRED + 3) & ~3;    // floats per chunk, a multiple of 4 for the float4 stores

enum : unsigned {
  AB_W1 = 1u, AB_B1 = 2u, AB_W2 = 4u, AB_B2 = 8u, AB_W3 = 16u, AB_B3 = 32u, AB_FEAT = 64u, AB_GEMB = 128u,
  AB_AEMB = 256u, AB_XYZ = 512u, AB_CAMPOS = 1024u
};

struct alignas(16) AbSmem {
  float W2[AP_H][AB_LDH];        // W2[n][k]                                   67.6 KB
  float W1t[AB_K1][AP_H];        // W1[n][k] at [k][n], k < 27; row 27 zero     14.3 KB
  float W3[6][AP_H];
  float b1[AP_H], b2[AP_H], b3[8];
  float X0[AB_T][AB_LDX];        // layer-1 input [min(dc, 1) | gemb | 0]
  float H1[AB_T][AB_LDH];        // h1, then dz1                               33.8 KB
  float H2[AP_H][AB_LDP];        // h2, then dz2 (transposed)                   34.8 KB
  float dz3[AB_T][8];            // dL/d(layer-3 output), x0.01 included
  float dc[AB_T][8];             // [0, 3): tone-map part of dL/dmin(dc, 1); [4, 7): the DC features
};
static_assert(sizeof(AbSmem) <= 227 * 1024, "appearance backward buffers exceed the shared memory of one SM");

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
__device__ __forceinline__ float f4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

template <int M>
__global__ void __launch_bounds__(AB_THREADS, 1)
appearance_bwd_kernel(int P, int D, int chunk, unsigned want, const float* __restrict__ features,
                      const float* __restrict__ gemb, const float* __restrict__ aemb, const float* __restrict__ W1,
                      const float* __restrict__ b1, const float* __restrict__ W2, const float* __restrict__ b2,
                      const float* __restrict__ W3, const float* __restrict__ b3, const float* __restrict__ means3D,
                      const float* __restrict__ campos, const float* __restrict__ dL_dcolors,
                      float* __restrict__ dL_dfeatures, float* __restrict__ dL_dgemb, float* __restrict__ dL_dmeans3D,
                      float* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char ab_smem[];
  AbSmem& S = *reinterpret_cast<AbSmem*>(ab_smem);
  constexpr int IN = 3 + AP_G + AP_E;
  const int tid = threadIdx.x;
  const int c16 = tid & 15, r16 = tid >> 4;      // GEMM thread grid: 16 column groups x 16 row groups
  const int p4 = tid >> 2, q4 = tid & 3;         // four threads per Gaussian
  const int n128 = tid & 127, h2i = tid >> 7;    // one hidden unit per thread, two halves
  const bool do_dz2 = want & (AB_W1 | AB_B1 | AB_W2 | AB_B2 | AB_FEAT | AB_GEMB | AB_AEMB);
  const bool do_dh1 = want & (AB_W1 | AB_B1 | AB_FEAT | AB_GEMB | AB_AEMB);
  const bool do_w1 = want & AB_W1, do_s1 = want & (AB_W1 | AB_B1 | AB_AEMB), do_in0 = want & (AB_FEAT | AB_GEMB);
  const bool do_w2 = want & AB_W2, do_w3 = want & (AB_W3 | AB_B3);
  const bool do_dir = (want & (AB_XYZ | AB_CAMPOS)) && D > 0;

  for (int i = tid; i < AP_H * AP_H; i += AB_THREADS) S.W2[i >> 7][i & 127] = W2[i];
  for (int i = tid; i < AB_K1 * AP_H; i += AB_THREADS) {
    const int k = i >> 7, n = i & 127;
    S.W1t[k][n] = k < 3 + AP_G ? W1[n * IN + k] : 0.f;
  }
  for (int i = tid; i < 6 * AP_H; i += AB_THREADS) S.W3[i >> 7][i & 127] = W3[i];
  if (tid < AP_H) {
    float acc = b1[tid];
#pragma unroll 8
    for (int e = 0; e < AP_E; e++) acc = fmaf(W1[tid * IN + 3 + AP_G + e], aemb[e], acc);
    S.b1[tid] = acc;
    S.b2[tid] = b2[tid];
    if (tid < 8) S.b3[tid] = tid < 6 ? b3[tid] : 0.f;
  }
  __syncthreads();
  float w3c[6];
#pragma unroll
  for (int o = 0; o < 6; o++) w3c[o] = S.W3[o][n128];
  const float cx = campos[0], cy = campos[1], cz = campos[2];

  float accW2[8][8];                 // dW2[c16 + 16 i][4 r16 + 64 (j / 4) + j % 4]
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) accW2[i][j] = 0.f;
  float accW1[14];                   // dW1[n128][14 h2i + i]
#pragma unroll
  for (int i = 0; i < 14; i++) accW1[i] = 0.f;
  float accW3[3] = {0.f, 0.f, 0.f};
  double accB3[3] = {0.0, 0.0, 0.0}, accXYZ[3] = {0.0, 0.0, 0.0}, accB1 = 0.0, accB2 = 0.0;   // sums of plain terms: float64

  const int g0 = blockIdx.x * chunk, g1 = min(P, g0 + chunk);
  for (int base = g0; base < g1; base += AB_T) {
    // ---- layer-1 input; rows past the chunk shadow its last Gaussian and get a zero cotangent
    {
      const int gi = min(base + p4, g1 - 1);
      const float* f = features + (size_t)gi * (3 * M);
      const float* ge = gemb + (size_t)gi * AP_G;
#pragma unroll
      for (int k = 8 * q4; k < 8 * q4 + 8; k++) S.X0[p4][k] = k < 3 ? fminf(f[k], 1.f) : k < 3 + AP_G ? ge[k - 3] : 0.f;
    }
    __syncthreads();
    // ---- layer 1: h1[p][n] = relu(sum_k X0[p][k] W1[n][k] + b1'[n]); p = 4 r16 + j, n = 4 c16 + 64 h + e
    {
      float acc[4][8];
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 8; e++) acc[j][e] = 0.f;
#pragma unroll 4
      for (int k = 0; k < AB_K1; k++) {
        const float4 w0 = ld4(&S.W1t[k][4 * c16]), w1 = ld4(&S.W1t[k][4 * c16 + 64]);
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float a = S.X0[4 * r16 + j][k];
#pragma unroll
          for (int e = 0; e < 4; e++) {
            acc[j][e] = fmaf(a, f4(w0, e), acc[j][e]);
            acc[j][4 + e] = fmaf(a, f4(w1, e), acc[j][4 + e]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int n = 4 * c16 + 64 * h;
          st4(&S.H1[4 * r16 + j][n], fmaxf(acc[j][4 * h] + S.b1[n], 0.f), fmaxf(acc[j][4 * h + 1] + S.b1[n + 1], 0.f),
              fmaxf(acc[j][4 * h + 2] + S.b1[n + 2], 0.f), fmaxf(acc[j][4 * h + 3] + S.b1[n + 3], 0.f));
        }
    }
    __syncthreads();
    // ---- layer 2: h2[n][p] = relu(sum_k h1[p][k] W2[n][k] + b2[n]); p = 4 r16 + j, n = c16 + 16 i
    {
      float acc[4][8];
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int i = 0; i < 8; i++) acc[j][i] = 0.f;
#pragma unroll 2
      for (int k = 0; k < AP_H; k += 4) {
        float4 a[4], b[8];
#pragma unroll
        for (int j = 0; j < 4; j++) a[j] = ld4(&S.H1[4 * r16 + j][k]);
#pragma unroll
        for (int i = 0; i < 8; i++) b[i] = ld4(&S.W2[c16 + 16 * i][k]);
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int i = 0; i < 8; i++) {
            acc[j][i] = fmaf(a[j].x, b[i].x, acc[j][i]);
            acc[j][i] = fmaf(a[j].y, b[i].y, acc[j][i]);
            acc[j][i] = fmaf(a[j].z, b[i].z, acc[j][i]);
            acc[j][i] = fmaf(a[j].w, b[i].w, acc[j][i]);
          }
      }
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int n = c16 + 16 * i;
        const float bb = S.b2[n];
        st4(&S.H2[n][4 * r16], fmaxf(acc[0][i] + bb, 0.f), fmaxf(acc[1][i] + bb, 0.f), fmaxf(acc[2][i] + bb, 0.f),
            fmaxf(acc[3][i] + bb, 0.f));
      }
    }
    __syncthreads();
    // ---- layer 3 (four threads per Gaussian, k = q4 + 4 kk), then the tone map and eval_sh and their adjoint
    {
      const int p = p4, g = base + p;
      const bool valid = g < g1;
      const int gi = valid ? g : g1 - 1;
      float z[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
      for (int kk = 0; kk < AP_H / 4; kk++) {
        const int k = q4 + 4 * kk;
        const float hv = S.H2[k][p];
#pragma unroll
        for (int o = 0; o < 6; o++) z[o] = fmaf(hv, S.W3[o][k], z[o]);
      }
#pragma unroll
      for (int o = 0; o < 6; o++) {      // butterfly: all four lanes hold the same bits
        z[o] += __shfl_xor_sync(0xffffffffu, z[o], 1);
        z[o] += __shfl_xor_sync(0xffffffffu, z[o], 2);
      }
      if (q4 == 0) {
        float off[3], mul[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
          off[c] = (z[c] + S.b3[c]) * 0.01f / SH_C0;
          mul[c] = (z[3 + c] + S.b3[3 + c]) * 0.01f;
        }
        const float vx = means3D[3 * (size_t)gi] - cx, vy = means3D[3 * (size_t)gi + 1] - cy,
                    vz = means3D[3 * (size_t)gi + 2] - cz;
        const float nrm = sqrtf(vx * vx + vy * vy + vz * vz);
        const float x = vx / nrm, y = vy / nrm, zz_ = vz / nrm;
        const float xx = x * x, yy = y * y, zz = zz_ * zz_, xy = x * y, yz = y * zz_, xz = x * zz_;
        float bas[16];
        bas[0] = SH_C0;
        bas[1] = -SH_C1 * y; bas[2] = SH_C1 * zz_; bas[3] = -SH_C1 * x;
        bas[4] = SH_C2_0 * xy; bas[5] = SH_C2_1 * yz; bas[6] = SH_C2_2 * (2.f * zz - xx - yy); bas[7] = SH_C2_3 * xz;
        bas[8] = SH_C2_4 * (xx - yy);
        bas[9] = SH_C3_0 * y * (3.f * xx - yy); bas[10] = SH_C3_1 * xy * zz_; bas[11] = SH_C3_2 * y * (4.f * zz - xx - yy);
        bas[12] = SH_C3_3 * zz_ * (2.f * zz - 3.f * xx - 3.f * yy); bas[13] = SH_C3_4 * x * (4.f * zz - xx - yy);
        bas[14] = SH_C3_5 * zz_ * (xx - yy); bas[15] = SH_C3_6 * x * (xx - 3.f * yy);
        const int ncoef = (D + 1) * (D + 1);
        const float* fr = features + (size_t)gi * (3 * M);
        float rgb[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 3 * M; j++) {
          const int k = j / 3, ch = j - 3 * k;
          const float tv = fminf(fr[j], 1.f) * mul[ch] + (k == 0 ? off[ch] : 0.f);
          if (k < ncoef) rgb[ch] = fmaf(bas[k], fminf(tv, 1.f), rgb[ch]);
        }
        float gr[3];
#pragma unroll
        for (int c = 0; c < 3; c++) gr[c] = valid && rgb[c] + 0.5f >= 0.f ? dL_dcolors[3 * (size_t)g + c] : 0.f;
        float dmul[3] = {0.f, 0.f, 0.f}, doff[3] = {0.f, 0.f, 0.f}, dbas[16];
#pragma unroll
        for (int k = 0; k < 16; k++) dbas[k] = 0.f;
#pragma unroll
        for (int j = 0; j < 3 * M; j++) {
          const int k = j / 3, ch = j - 3 * k;
          const float f = fr[j], fc = fminf(f, 1.f);
          const float tv = fc * mul[ch] + (k == 0 ? off[ch] : 0.f);
          float dfc = 0.f;
          if (k < ncoef) {
            dbas[k] = fmaf(fminf(tv, 1.f), gr[ch], dbas[k]);
            const float dtv = tv <= 1.f ? bas[k] * gr[ch] : 0.f;
            dmul[ch] = fmaf(dtv, fc, dmul[ch]);
            if (k == 0) doff[ch] = dtv;
            dfc = dtv * mul[ch];
          }
          if (k == 0) {
            S.dc[p][ch] = dfc;
            S.dc[p][4 + ch] = f;
          } else if (valid && (want & AB_FEAT)) {
            dL_dfeatures[(size_t)g * (3 * M) + j] = f <= 1.f ? dfc : 0.f;
          }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
          S.dz3[p][c] = doff[c] / SH_C0 * 0.01f;
          S.dz3[p][3 + c] = dmul[c] * 0.01f;
        }
        if (valid && (want & (AB_XYZ | AB_CAMPOS))) {
          float dvx = 0.f, dvy = 0.f, dvz = 0.f;
          if (do_dir) {
            const float* s = dbas;
            float dx = -SH_C1 * s[3], dy = -SH_C1 * s[1], dz = SH_C1 * s[2];
            if (D > 1) {
              dx += SH_C2_0 * y * s[4] + SH_C2_2 * 2.f * -x * s[6] + SH_C2_3 * zz_ * s[7] + SH_C2_4 * 2.f * x * s[8];
              dy += SH_C2_0 * x * s[4] + SH_C2_1 * zz_ * s[5] + SH_C2_2 * 2.f * -y * s[6] + SH_C2_4 * 2.f * -y * s[8];
              dz += SH_C2_1 * y * s[5] + SH_C2_2 * 2.f * 2.f * zz_ * s[6] + SH_C2_3 * x * s[7];
              if (D > 2) {
                dx += SH_C3_0 * s[9] * 3.f * 2.f * xy + SH_C3_1 * s[10] * yz + SH_C3_2 * s[11] * -2.f * xy +
                      SH_C3_3 * s[12] * -3.f * 2.f * xz + SH_C3_4 * s[13] * (-3.f * xx + 4.f * zz - yy) +
                      SH_C3_5 * s[14] * 2.f * xz + SH_C3_6 * s[15] * 3.f * (xx - yy);
                dy += SH_C3_0 * s[9] * 3.f * (xx - yy) + SH_C3_1 * s[10] * xz + SH_C3_2 * s[11] * (-3.f * yy + 4.f * zz - xx) +
                      SH_C3_3 * s[12] * -3.f * 2.f * yz + SH_C3_4 * s[13] * -2.f * xy + SH_C3_5 * s[14] * -2.f * yz +
                      SH_C3_6 * s[15] * -3.f * 2.f * xy;
                dz += SH_C3_1 * s[10] * xy + SH_C3_2 * s[11] * 4.f * 2.f * yz + SH_C3_3 * s[12] * 3.f * (2.f * zz - xx - yy) +
                      SH_C3_4 * s[13] * 4.f * 2.f * xz + SH_C3_5 * s[14] * (xx - yy);
              }
            }
            // d = v / |v|:  dL/dv = (dL/dd - d (d . dL/dd)) / |v|
            const float dd = x * dx + y * dy + zz_ * dz;
            dvx = (dx - x * dd) / nrm; dvy = (dy - y * dd) / nrm; dvz = (dz - zz_ * dd) / nrm;
          }
          if (want & AB_XYZ) {
            dL_dmeans3D[3 * (size_t)g] = dvx; dL_dmeans3D[3 * (size_t)g + 1] = dvy; dL_dmeans3D[3 * (size_t)g + 2] = dvz;
          }
          accXYZ[0] += dvx; accXYZ[1] += dvy; accXYZ[2] += dvz;
        }
      }
    }
    __syncthreads();
    // ---- dW3, db3 (thread: k = n128, o = 3 h2i + o3), before dz2 overwrites h2
    if (do_w3) {
#pragma unroll 4
      for (int p = 0; p < AB_T; p += 4) {
        const float4 hv = ld4(&S.H2[n128][p]);
#pragma unroll
        for (int o3 = 0; o3 < 3; o3++) {
          const int o = 3 * h2i + o3;
          accW3[o3] = fmaf(S.dz3[p][o], hv.x, accW3[o3]);
          accW3[o3] = fmaf(S.dz3[p + 1][o], hv.y, accW3[o3]);
          accW3[o3] = fmaf(S.dz3[p + 2][o], hv.z, accW3[o3]);
          accW3[o3] = fmaf(S.dz3[p + 3][o], hv.w, accW3[o3]);
        }
      }
      if (n128 == 0)
        for (int p = 0; p < AB_T; p++)
#pragma unroll
          for (int o3 = 0; o3 < 3; o3++) accB3[o3] += S.dz3[p][3 * h2i + o3];
    }
    if (do_dz2) {
      __syncthreads();
      // dz2[n][p] = (h2 > 0) sum_o dz3[p][o] W3[o][n]; thread: n = n128, p in [32 h2i, 32 h2i + 32)
#pragma unroll 2
      for (int p = 32 * h2i; p < 32 * h2i + 32; p += 4) {
        const float4 hv = ld4(&S.H2[n128][p]);
        float d[4];
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          float dh = 0.f;
#pragma unroll
          for (int o = 0; o < 6; o++) dh = fmaf(S.dz3[p + jj][o], w3c[o], dh);
          d[jj] = f4(hv, jj) > 0.f ? dh : 0.f;
          accB2 += d[jj];
        }
        st4(&S.H2[n128][p], d[0], d[1], d[2], d[3]);
      }
      __syncthreads();
      // dW2[n][k] += sum_p dz2[n][p] h1[p][k]; n = c16 + 16 i, k = 4 r16 + 64 h + e
      if (do_w2) {
#pragma unroll 1
        for (int p = 0; p < AB_T; p += 4) {
          float4 a[8], b[4][2];
#pragma unroll
          for (int i = 0; i < 8; i++) a[i] = ld4(&S.H2[c16 + 16 * i][p]);
#pragma unroll
          for (int jj = 0; jj < 4; jj++) {
            b[jj][0] = ld4(&S.H1[p + jj][4 * r16]);
            b[jj][1] = ld4(&S.H1[p + jj][4 * r16 + 64]);
          }
#pragma unroll
          for (int i = 0; i < 8; i++)
#pragma unroll
            for (int j = 0; j < 8; j++) {
              const int h = j >> 2, e = j & 3;
              float acc = accW2[i][j];
              acc = fmaf(a[i].x, f4(b[0][h], e), acc);
              acc = fmaf(a[i].y, f4(b[1][h], e), acc);
              acc = fmaf(a[i].z, f4(b[2][h], e), acc);
              acc = fmaf(a[i].w, f4(b[3][h], e), acc);
              accW2[i][j] = acc;
            }
        }
        __syncthreads();        // every thread is done reading h1 before dz1 replaces it
      }
      if (do_dh1) {
        // dh1[p][k] = sum_n dz2[n][p] W2[n][k]; p = 4 r16 + j, k = 4 c16 + 64 h + e; dz1 = (h1 > 0) dh1 -> H1
        float acc[4][8];
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int e = 0; e < 8; e++) acc[j][e] = 0.f;
#pragma unroll 4
        for (int n = 0; n < AP_H; n++) {
          const float4 a = ld4(&S.H2[n][4 * r16]);
          const float4 w0 = ld4(&S.W2[n][4 * c16]), w1 = ld4(&S.W2[n][4 * c16 + 64]);
#pragma unroll
          for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
              acc[j][e] = fmaf(f4(a, j), f4(w0, e), acc[j][e]);
              acc[j][4 + e] = fmaf(f4(a, j), f4(w1, e), acc[j][4 + e]);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            float* q = &S.H1[4 * r16 + j][4 * c16 + 64 * h];
            const float4 hv = ld4(q);
            st4(q, hv.x > 0.f ? acc[j][4 * h] : 0.f, hv.y > 0.f ? acc[j][4 * h + 1] : 0.f,
                hv.z > 0.f ? acc[j][4 * h + 2] : 0.f, hv.w > 0.f ? acc[j][4 * h + 3] : 0.f);
          }
        __syncthreads();
        // dW1[n][k] += sum_p dz1[p][n] X0[p][k] (thread: n = n128, k = 14 h2i + i) and sum_p dz1[p][n]
        if (do_s1) {
#pragma unroll 2
          for (int p = 0; p < AB_T; p++) {
            const float d = S.H1[p][n128];
            if (h2i == 0) accB1 += d;
            if (do_w1) {
#pragma unroll
              for (int i = 0; i < 14; i++) accW1[i] = fmaf(d, S.X0[p][14 * h2i + i], accW1[i]);
            }
          }
        }
        // d[dc | gemb][p][k] = sum_n dz1[p][n] W1[n][k]; thread: p = p4, k = q4 + 4 i
        if (do_in0) {
          float acc7[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
          for (int n = 0; n < AP_H; n += 4) {
            const float4 a = ld4(&S.H1[p4][n]);
#pragma unroll
            for (int i = 0; i < 7; i++) {
              const float4 w = ld4(&S.W1t[q4 + 4 * i][n]);
              acc7[i] = fmaf(a.x, w.x, acc7[i]);
              acc7[i] = fmaf(a.y, w.y, acc7[i]);
              acc7[i] = fmaf(a.z, w.z, acc7[i]);
              acc7[i] = fmaf(a.w, w.w, acc7[i]);
            }
          }
          const int g = base + p4;
          if (g < g1) {
#pragma unroll
            for (int i = 0; i < 7; i++) {
              const int k = q4 + 4 * i;
              if (k < 3) {
                if (want & AB_FEAT)
                  dL_dfeatures[(size_t)g * (3 * M) + k] = S.dc[p4][4 + k] <= 1.f ? S.dc[p4][k] + acc7[i] : 0.f;
              } else if (k < 3 + AP_G) {
                if (want & AB_GEMB) dL_dgemb[(size_t)g * AP_G + k - 3] = acc7[i];
              }
            }
          }
        }
      }
    }
    __syncthreads();            // the next tile rewrites every buffer
  }

  // ---- this chunk's sums -> partial[blockIdx.x]
  float* out = partial + (size_t)blockIdx.x * AB_PSTRIDE;
  if (do_w2)
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int h = 0; h < 2; h++)
        st4(&out[RO_W2 + (c16 + 16 * i) * AP_H + 4 * r16 + 64 * h], accW2[i][4 * h], accW2[i][4 * h + 1],
            accW2[i][4 * h + 2], accW2[i][4 * h + 3]);
  if (do_w1)
#pragma unroll
    for (int i = 0; i < 14; i++)
      if (14 * h2i + i < 27) out[RO_W1 + n128 * 27 + 14 * h2i + i] = accW1[i];
  if (do_w3) {
#pragma unroll
    for (int o3 = 0; o3 < 3; o3++) out[RO_W3 + (3 * h2i + o3) * AP_H + n128] = accW3[o3];
    if (n128 == 0)
#pragma unroll
      for (int o3 = 0; o3 < 3; o3++) out[RO_B3 + 3 * h2i + o3] = (float)accB3[o3];
  }
  if (h2i == 0) out[RO_B1 + n128] = (float)accB1;
  double* red = reinterpret_cast<double*>(&S.H2[0][0]);      // float64 scratch over h2, which is no longer needed
  red[tid] = accB2;                                          // db2: the two halves of unit n, added in a fixed order
  __syncthreads();
  if (h2i == 0) out[RO_B2 + n128] = (float)(red[n128] + red[128 + n128]);
  __syncthreads();
  if (q4 == 0) {
    red[3 * p4] = accXYZ[0]; red[3 * p4 + 1] = accXYZ[1]; red[3 * p4 + 2] = accXYZ[2];
  }
  __syncthreads();
  if (tid < 3) {
    double s = 0.0;
    for (int p = 0; p < AB_T; p++) s += red[3 * p + tid];
    out[RO_XYZ + tid] = (float)s;
  }
}

// Sum of the chunk partials, float64 in chunk order, rounded once; element e of the partial layout per thread.
__global__ void __launch_bounds__(256)
appearance_bwd_reduce_kernel(int nchunks, const float* __restrict__ partial, float* __restrict__ dW1, float* __restrict__ db1,
                             float* __restrict__ dW2, float* __restrict__ db2, float* __restrict__ dW3,
                             float* __restrict__ db3, float* __restrict__ dcampos, double* __restrict__ sum_dz1) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= AB_NRED) return;
  const bool need = e < RO_W1 ? dW2 != nullptr : e < RO_W3 ? dW1 != nullptr : e < RO_B1 ? dW3 != nullptr
                  : e < RO_B2 ? sum_dz1 != nullptr : e < RO_B3 ? db2 != nullptr : e < RO_XYZ ? db3 != nullptr
                  : dcampos != nullptr;
  if (!need) return;
  double s = 0.0;
#pragma unroll 16
  for (int c = 0; c < nchunks; c++) s += (double)partial[(size_t)c * AB_PSTRIDE + e];
  if (e < RO_W1) dW2[e] = (float)s;
  else if (e < RO_W3) dW1[((e - RO_W1) / 27) * (3 + AP_G + AP_E) + (e - RO_W1) % 27] = (float)s;
  else if (e < RO_B1) dW3[e - RO_W3] = (float)s;
  else if (e < RO_B2) {
    sum_dz1[e - RO_B1] = s;
    if (db1) db1[e - RO_B1] = (float)s;
  } else if (e < RO_B3) db2[e - RO_B2] = (float)s;
  else if (e < RO_XYZ) db3[e - RO_B3] = (float)s;
  else dcampos[e - RO_XYZ] = (float)(0.0 - s);
}

// The embedding columns: dW1[:, 27:] = (sum dz1) aemb^T and dL/daemb = W1[:, 27:]^T sum dz1, from the float64 sum.
__global__ void __launch_bounds__(256)
appearance_bwd_embed_kernel(const double* __restrict__ sum_dz1, const float* __restrict__ W1, const float* __restrict__ aemb,
                            float* __restrict__ dW1, float* __restrict__ daemb) {
  constexpr int IN = 3 + AP_G + AP_E;
  if (dW1)
    for (int i = threadIdx.x; i < AP_H * AP_E; i += blockDim.x) {
      const int n = i / AP_E, e = i - n * AP_E;
      dW1[n * IN + 3 + AP_G + e] = (float)(sum_dz1[n] * (double)aemb[e] + 0.0);   // + 0.0: no -0 at P = 0
    }
  if (daemb && threadIdx.x < AP_E) {
    double s = 0.0;
    for (int n = 0; n < AP_H; n++) s += (double)W1[n * IN + 3 + AP_G + threadIdx.x] * sum_dz1[n];
    daemb[threadIdx.x] = (float)s;
  }
}

int appearance_bwd_chunk(int P) { return max(512, 64 * ((P + 65535) / 65536)); }

}  // namespace

extern "C" size_t sfgs_appearance_backward_scratch_bytes(int P) {
  const int chunk = appearance_bwd_chunk(P > 0 ? P : 0);
  const size_t nchunks = P > 0 ? (size_t)((P + chunk - 1) / chunk) : 0;
  return nchunks * AB_PSTRIDE * sizeof(float) + AP_H * sizeof(double);
}

extern "C" int sfgs_appearance_backward(int P, int D, int M, const float* features, const float* gemb, int G,
                                        const float* aemb, int E, const float* W1, const float* b1, const float* W2,
                                        const float* b2, const float* W3, const float* b3, const float* means3D,
                                        const float* campos, const float* dL_dcolors, float* dL_dfeatures,
                                        float* dL_dgemb, float* dL_daemb, float* dL_dW1, float* dL_db1, float* dL_dW2,
                                        float* dL_db2, float* dL_dW3, float* dL_db3, float* dL_dmeans3D,
                                        float* dL_dcampos, sfgs_alloc_fn scratch_alloc, void* scratch_user,
                                        void* stream) {
  if (P < 0) return sfgs_set_error(SFGS_E_BADARG, "appearance_backward: P < 0", 0);
  const int bad = appearance_check("appearance_backward", P, D, M, G, E,
                                   {aemb, W1, b1, W2, b2, W3, b3, campos, reinterpret_cast<const void*>(scratch_alloc)},
                                   {features, gemb, means3D, dL_dcolors}, features, gemb);
  if (bad) return bad;
  const unsigned want = (dL_dW1 ? AB_W1 : 0u) | (dL_db1 ? AB_B1 : 0u) | (dL_dW2 ? AB_W2 : 0u) | (dL_db2 ? AB_B2 : 0u) |
                        (dL_dW3 ? AB_W3 : 0u) | (dL_db3 ? AB_B3 : 0u) | (dL_dfeatures ? AB_FEAT : 0u) |
                        (dL_dgemb ? AB_GEMB : 0u) | (dL_daemb ? AB_AEMB : 0u) | (dL_dmeans3D ? AB_XYZ : 0u) |
                        (dL_dcampos ? AB_CAMPOS : 0u);
  if (!want) return SFGS_OK;
  const int chunk = appearance_bwd_chunk(P);
  const int nchunks = P > 0 ? (P + chunk - 1) / chunk : 0;
  char* scratch = scratch_alloc(scratch_user, sfgs_appearance_backward_scratch_bytes(P));
  if (!scratch) return sfgs_set_error(SFGS_E_ALLOC, "appearance_backward: scratch allocation failed", 0);
  float* partial = reinterpret_cast<float*>(scratch + AP_H * sizeof(double));
  double* sum_dz1 = reinterpret_cast<double*>(scratch);
  const cudaStream_t st = (cudaStream_t)stream;
  using Kernel = void (*)(int, int, int, unsigned, const float*, const float*, const float*, const float*, const float*,
                          const float*, const float*, const float*, const float*, const float*, const float*,
                          const float*, float*, float*, float*, float*);
  const Kernel kernels[4] = {appearance_bwd_kernel<1>, appearance_bwd_kernel<4>, appearance_bwd_kernel<9>,
                             appearance_bwd_kernel<16>};
  static SfgsPerDeviceOnce once;
  if (once.first_use())
    for (const Kernel k : kernels) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AbSmem));
  if (nchunks > 0) {
    SFGS_COUNT_LAUNCH();
    kernels[M == 1 ? 0 : M == 4 ? 1 : M == 9 ? 2 : 3]<<<nchunks, AB_THREADS, sizeof(AbSmem), st>>>(
        P, D, chunk, want, features, gemb, aemb, W1, b1, W2, b2, W3, b3, means3D, campos, dL_dcolors, dL_dfeatures,
        dL_dgemb, dL_dmeans3D, partial);
  }
  const bool embed = (want & (AB_W1 | AB_AEMB)) != 0;
  if (want & (AB_W1 | AB_B1 | AB_W2 | AB_B2 | AB_W3 | AB_B3 | AB_AEMB | AB_CAMPOS)) {
    SFGS_COUNT_LAUNCH();
    appearance_bwd_reduce_kernel<<<(AB_NRED + 255) / 256, 256, 0, st>>>(
        nchunks, partial, dL_dW1, dL_db1, dL_dW2, dL_db2, dL_dW3, dL_db3, dL_dcampos,
        (want & (AB_W1 | AB_B1 | AB_AEMB)) ? sum_dz1 : nullptr);
  }
  if (embed) {
    SFGS_COUNT_LAUNCH();
    appearance_bwd_embed_kernel<<<1, 256, 0, st>>>(sum_dz1, W1, aemb, dL_dW1, dL_daemb);
  }
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : sfgs_set_error(SFGS_E_CUDA, "appearance_backward", (int)e);
}
