// sfgs_appearance.cu — the appearance path of render() as one tensor-core kernel (SURVEY.md 8f rank 2).
//
// Replaces, for the forward pass, gaussian_renderer/__init__.py:105-118 + EmbeddingModel.forward
// (scene/gaussian_model.py:45-69) + eval_sh (utils/sh_utils.py) — in torch: a [P,59] concat, three Linear layers with
// [P,128] fp32 intermediates, a repeat, a [P,48] tone map, a [P,3,16] transpose, the SH evaluation and four clamps,
// ~25 kernels and ~2.5 KB of HBM traffic per Gaussian — by one kernel that reads each Gaussian's 48 SH features, 24
// Fourier features and position once and writes its 3 colours (324 B per Gaussian):
//
//   inp    = [min(features[:3], 1) | gemb | aemb]                      (59 = 3 + 24 + 32)
//   h      = W3 relu(W2 relu(W1 inp + b1) + b2) + b3 ;  offset, mul = 0.01 h[:3], 0.01 h[3:]
//   toned  = min(min(features, 1) * mul[ch] + [offset/C0 on the DC term], 1)           ([16,3] per Gaussian)
//   colour = max(eval_sh(D, toned, normalize(xyz - campos)) + 0.5, 0)
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

__global__ void __launch_bounds__(AP_THREADS, 1)
appearance_fwd_kernel(int P, int D, const float* __restrict__ features /*[P,16,3]*/, const float* __restrict__ gemb /*[P,24]*/,
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
    const float* pf = features + (size_t)r0 * 48;
    const float* pg = gemb + (size_t)r0 * AP_G;
    const float* pm = means3D + (size_t)r0 * 3;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pf), "r"(rows * 192u) : "memory");
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
      const float* f = features + (size_t)gi * 48;
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
    const float4* f4 = reinterpret_cast<const float4*>(features + (size_t)gi * 48);
#pragma unroll
    for (int q = 0; q < 12; q++) {
      const float4 v = f4[q];
      const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int j = 4 * q + u, k = j / 3, ch = j - 3 * k;          // features[k][ch]
        float tv = fminf(e[u], 1.f) * mul[ch] + (k == 0 ? off[ch] : 0.f);
        tv = fminf(tv, 1.f);
        if (k < ncoef) rgb[ch] = fmaf(bas[k], tv, rgb[ch]);
      }
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

extern "C" int sfgs_appearance_forward(int P, int D, int M, const float* features, const float* gemb, int G, const float* aemb,
                                       int E, const float* W1, const float* b1, const float* W2, const float* b2,
                                       const float* W3, const float* b3, const float* means3D, const float* campos,
                                       float* colors, void* stream) {
  if (P < 0) return sfgs_set_error(SFGS_E_BADARG, "appearance_forward: P < 0", 0);
  if (P == 0) return SFGS_OK;
  if (M != 16 || G != AP_G || E != AP_E || D < 0 || D > 3)
    return sfgs_set_error(SFGS_E_UNSUPPORTED, "appearance_forward: built for 16 SH coefficients, 24 Fourier features, a 32-wide embedding", 0);
  if (!features || !gemb || !aemb || !W1 || !b1 || !W2 || !b2 || !W3 || !b3 || !means3D || !campos || !colors)
    return sfgs_set_error(SFGS_E_BADARG, "appearance_forward: null pointer", 0);
  if ((reinterpret_cast<uintptr_t>(features) & 15) || (reinterpret_cast<uintptr_t>(gemb) & 15))
    return sfgs_set_error(SFGS_E_BADARG, "appearance_forward: features / gemb must be 16-byte aligned", 0);
  static SfgsPerDeviceOnce once;
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (once.first_use() || (dev >= 0 && dev < 64 && sms[dev] == 0)) {
    cudaFuncSetAttribute(appearance_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ApSmem));
    int n = 132;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (dev >= 0 && dev < 64) sms[dev] = n;
  }
  const int nsm = (dev >= 0 && dev < 64 && sms[dev] > 0) ? sms[dev] : 132;
  const int ntiles = (P + AP_M - 1) / AP_M;
  const int pairs = (ntiles + AP_GROUPS - 1) / AP_GROUPS;
  const int grid = pairs < nsm ? pairs : nsm;                // persistent: one CTA (two tile groups) per SM
  SFGS_COUNT_LAUNCH();
  appearance_fwd_kernel<<<grid, AP_THREADS, sizeof(ApSmem), (cudaStream_t)stream>>>(P, D, features, gemb, aemb, W1, b1, W2, b2,
                                                                                  W3, b3, means3D, campos, colors);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : sfgs_set_error(SFGS_E_CUDA, "appearance_forward", (int)e);
}
