/*
 * sfgs.h — C ABI of the H100-native splat rasterizer (libsfgs.so).
 *
 * Drop-in boundary for the hot path of jayin92/Skyfall-GS: every entry point
 * below replaces one entry of the reference's native interface.  Citations
 * are to the reference tree (RAST = submodules/diff-gaussian-rasterization-depth,
 * SSIM = submodules/fused-ssim, KNN = submodules/simple-knn):
 *
 *   sfgs_rasterize_forward   <- CudaRasterizer::Rasterizer::forward
 *                               RAST/cuda_rasterizer/rasterizer.h:35-68
 *                               (bound by RasterizeGaussiansCUDA, RAST/rasterize_points.cu:35-135)
 *   sfgs_rasterize_backward  <- CudaRasterizer::Rasterizer::backward
 *                               RAST/cuda_rasterizer/rasterizer.h:70-103
 *                               (bound by RasterizeGaussiansBackwardCUDA, RAST/rasterize_points.cu:137-243)
 *   sfgs_mark_visible        <- CudaRasterizer::Rasterizer::markVisible
 *                               RAST/cuda_rasterizer/rasterizer.h:23-33 (RAST/rasterize_points.cu:245-264)
 *   sfgs_fusedssim_forward   <- fusedssim          SSIM/ssim.h:7-14
 *   sfgs_fusedssim_backward  <- fusedssim_backward SSIM/ssim.h:16-26
 *   sfgs_dist2_knn3          <- SimpleKNN::knn     KNN/simple_knn.h (bound by distCUDA2, KNN/spatial.cu:17-35)
 *
 * Conventions: plain C, raw DEVICE pointers (unless a name ends in _host),
 * sizes as int/size_t, a CUDA stream passed as void* (cudaStream_t), int
 * status returns (0 / >=0 = success, <0 = SFGS_E_*), no C++ exceptions and no
 * torch types cross this boundary.  All matrices use the reference's layout:
 * viewmatrix[16]/projmatrix[16] are the row-vector ("transposed") tensors of
 * scene/cameras.py:64-73, i.e. element [4*c + r].
 *
 * Scratch memory is obtained through caller-supplied allocator callbacks, the
 * C equivalent of the reference's std::function<char*(size_t)> resize
 * callbacks (RAST/rasterize_points.cu:27-33).  A callback may be invoked more
 * than once per call (the last returned pointer is the live one) and the
 * memory must stay valid until the matching backward call has run.
 */
#ifndef SFGS_H_INCLUDED
#define SFGS_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SFGS_VERSION 4          /* 4: compute_3d_filter, densification_stats, densify_plan/apply; 3: appearance_forward, overflow_reruns, selftest_expf; 2: out_norm_raw / norm_raw, two-phase backward, activations */
#define SFGS_TILE 16          /* BLOCK_X = BLOCK_Y = 16, RAST/cuda_rasterizer/config.h:15-17 */
#define SFGS_MAX_EXTRA 34     /* MAX_EXTRA_DIMS, RAST/cuda_rasterizer/auxiliary.h:20 */

enum {
  SFGS_OK = 0,
  SFGS_E_CUDA = -1,        /* a CUDA runtime call failed; sfgs_last_error() has the text */
  SFGS_E_BADARG = -2,      /* null pointer / bad size / unsupported combination */
  SFGS_E_ALLOC = -3,       /* an allocator callback returned NULL */
  SFGS_E_UNSUPPORTED = -4  /* feature of the reference API not implemented by this build */
};

/* Allocator callback: return a device pointer to at least `bytes` bytes
 * (256-byte aligned), or NULL on failure. */
typedef char* (*sfgs_alloc_fn)(void* user, size_t bytes);

/* ---- rasterizer forward ------------------------------------------------ */
typedef struct sfgs_forward_args {
  /* scratch: geometry (per Gaussian), binning (per tile instance), image (per pixel / tile) */
  sfgs_alloc_fn geom_alloc;    void* geom_user;
  sfgs_alloc_fn binning_alloc; void* binning_user;
  sfgs_alloc_fn image_alloc;   void* image_user;
  int P;                 /* number of Gaussians */
  int D;                 /* active SH degree (0..3) */
  int M;                 /* SH coefficients per Gaussian in `shs` (0 when colors_precomp is used) */
  int ED;                /* extra attribute channels (0..34) */
  int width, height;
  const float* background;      /* [3] */
  const float* means3D;         /* [P,3] */
  const float* shs;             /* [P,M,3] or NULL */
  const float* colors_precomp;  /* [P,3] or NULL */
  const float* opacities;       /* [P] */
  const float* scales;          /* [P,3] */
  float scale_modifier;
  const float* rotations;       /* [P,4] (w,x,y,z), used as given (not re-normalised) */
  const float* cov3D_precomp;   /* [P,6] or NULL */
  const float* norm3D_precomp;  /* [P,3] or NULL */
  const float* extra_attrs;     /* [P,ED] or NULL */
  const float* viewmatrix;      /* [16] */
  const float* projmatrix;      /* [16] */
  const float* cam_pos;         /* [3] */
  float tan_fovx, tan_fovy;
  float kernel_size;
  int prefiltered;
  /* outputs (every element is written; no pre-zeroing required) */
  float* out_color;   /* [3,H,W] */
  float* out_depth;   /* [1,H,W] */
  float* out_norm;    /* [3,H,W] (un-normalised, as the reference; unit length when out_norm_raw is given) */
  float* out_alpha;   /* [1,H,W] */
  float* out_extra;   /* [ED,H,W] or NULL */
  int*   radii;       /* [P] */
  int debug;          /* synchronise and check after every stage */
  void* stream;       /* cudaStream_t */
  /* optional hint: expected number of tile instances (0 = let the library guess) */
  long long capacity_hint;
  /* optional screen-space shard (multi-GPU tile-row sharding, SURVEY.md 8e): only tile rows
   * [tile_row_begin, tile_row_end) of the full tile grid are binned and blended, and only their pixels are
   * written.  radii still report visibility in the FULL image.  0,0 = the whole image. */
  int tile_row_begin, tile_row_end;
  /* optional fused post-op (SURVEY.md 8f rank 1; the reference normalises the blended normal map in torch,
   * RAST/diff_gauss/__init__.py:48): when non-NULL, out_norm receives F.normalize(blend, p=2, dim=0, eps=1e-12)
   * and the un-normalised blend is stored here ([3,H,W]) for the backward. */
  float* out_norm_raw;
  /* optional: the image all-gather of the tile-row sharded multi-GPU mode fused into the blend kernel.
   * out_peers[r], r = 0..n_out_peers-1 (host array, <= 8), is rank r's [8,H,W] frame block (colour 3, depth 1,
   * alpha 1, normal 3 planes, in this order) as a peer-mapped device pointer; the pixels of this rank's band are
   * stored into every block (NVLink stores), so after a barrier every rank holds the whole frame.  out_color /
   * out_depth / out_alpha / out_norm are then ignored. */
  float* const* out_peers;
  int n_out_peers;
} sfgs_forward_args;

/* Returns num_rendered (>= 0) or a negative SFGS_E_* code. */
int sfgs_rasterize_forward(const sfgs_forward_args* a);

/* ---- rasterizer backward ----------------------------------------------- */
typedef struct sfgs_backward_args {
  int P, D, M, R, ED;
  int width, height;
  const float* background;
  const float* means3D;
  const float* shs;
  const float* colors_precomp;
  const float* scales;
  float scale_modifier;
  const float* rotations;
  const float* cov3D_precomp;
  const float* norm3D_precomp;
  const float* extra_attrs;
  const float* viewmatrix;
  const float* projmatrix;
  const float* cam_pos;
  float tan_fovx, tan_fovy;
  float kernel_size;
  const int* radii;
  char* geom_buffer;       /* the live pointers handed out by the forward allocators */
  char* binning_buffer;
  char* image_buffer;
  const float* accum_alphas;   /* out_alpha of the forward */
  const float* dL_dpix;        /* [3,H,W] */
  const float* dL_dpix_depth;  /* [1,H,W] */
  const float* dL_dpix_norm;   /* [3,H,W] */
  const float* dL_dpix_alpha;  /* [1,H,W] */
  const float* dL_dpix_extra;  /* [ED,H,W] or NULL */
  /* outputs: every element is written by the call (no pre-zeroing required) */
  float* dL_dmean2D;   /* [P,3]  (x*W/2, y*H/2, sum|.|) */
  float* dL_dconic;    /* [P,4]  (xx, xy, unused, yy) */
  float* dL_dopacity;  /* [P] */
  float* dL_dcolor;    /* [P,3] */
  float* dL_ddepth;    /* [P] */
  float* dL_dmean3D;   /* [P,3] */
  float* dL_dcov3D;    /* [P,6] */
  float* dL_dnorm3D;   /* [P,3] */
  float* dL_dsh;       /* [P,M,3] or NULL when M == 0 */
  float* dL_dscale;    /* [P,3] */
  float* dL_drot;      /* [P,4] */
  float* dL_dextra;    /* [P,ED] or NULL */
  /* scratch for the per-Gaussian blend-adjoint accumulators: P*16 floats, need not be zeroed */
  sfgs_alloc_fn scratch_alloc; void* scratch_user;
  int debug;
  void* stream;
  /* the same band the forward used (0,0 = whole image); gradients are then partial sums over the band */
  int tile_row_begin, tile_row_end;
  /* optional: the forward's out_norm_raw.  When non-NULL, dL_dpix_norm is the gradient w.r.t. the UNIT normal
   * map and the blend adjoint applies the adjoint of F.normalize while it loads the pixel. */
  const float* norm_raw;
  /* optional two-phase backward, for the tile-row sharded multi-GPU mode (SURVEY.md 8e): the per-Gaussian
   * blend-adjoint sums are linear in the pixel cotangents, so ranks exchange the [P,16] sums (64 B/Gaussian)
   * instead of the final gradients (56+12M floats/Gaussian), and each rank finishes only its slice.
   *   phase 0 (default)  both stages in one call; `acc` may be NULL (scratch comes from scratch_alloc).
   *   phase 1            blend adjoint only: `acc` ([P,16] floats, caller-owned) is cleared and receives the sums
   *                      of this rank's tile-row band; no gradient output is touched.
   *   phase 2            per-Gaussian adjoint only, for Gaussians [gauss_begin, gauss_end): `acc` points at the
   *                      row of Gaussian gauss_begin (e.g. the result of a reduce-scatter); gradient rows
   *                      [gauss_begin, gauss_end) of the full-size output arrays are written, others untouched. */
  int phase;
  float* acc;
  int gauss_begin, gauss_end;
  /* optional, phase 1 only: the reduce-scatter FUSED into the blend adjoint (one node, NVLink / NVSwitch peer
   * access).  acc_peers[r], r = 0..n_peers-1 (host array, n_peers <= 8), is rank r's [peer_slice,16] accumulator
   * slice as a peer-mapped device pointer; Gaussian g is accumulated into acc_peers[g / peer_slice] +
   * (g % peer_slice)*16 with system-scope vector reductions that travel over NVLink tile by tile while the kernel
   * computes, so no separate collective follows.  The call clears nothing and `acc` is ignored: every rank clears
   * its own slice and synchronises with its peers before and after the call (sfgs/multigpu.py). */
  float* const* acc_peers;
  int n_peers, peer_slice;
} sfgs_backward_args;

int sfgs_rasterize_backward(const sfgs_backward_args* a);

/* The same backward with bit-reproducible outputs: no floating-point atomics or reductions; every per-Gaussian sum
 * runs in an order fixed by the inputs alone (not by scheduling, SM count or addresses), and the cross-tile sums are
 * formed in float64.  Same struct, same validation, plus:
 *   phase 0 and phase 1 (the blend adjoint) need `radii` and `scratch_alloc`: the extra scratch is
 *     4 P + 524 R bytes (+ alignment; R = instances of the forward), on top of the P*16 floats of `acc` when that is
 *     not given;
 *   (sfgs_rasterize_backward_camera adds 35 * 8 * ceil(P / 96) bytes for the camera partials,
 *   sfgs_rasterize_backward_camera_intrinsics 37 * 8 * ceil(P / 96));
 *   phase 2 runs the per-Gaussian adjoint, which has no reduction, exactly as sfgs_rasterize_backward does;
 *   acc_peers (system-scope reductions) and ED > 0 (extra_attrs) return SFGS_E_UNSUPPORTED before any CUDA work.
 * The outputs equal sfgs_rasterize_backward's up to the rounding of the sums' order. */
int sfgs_rasterize_backward_deterministic(const sfgs_backward_args* a);

/* ---- subpixel offsets (Mip-Splatting's ray jitter: GaussianRasterizationSettings.subpixel_offset) -------------
 * The three calls above with per-pixel sample positions: pixel (x, y) (centres at integer coordinates) blends the
 * splats of its own tile's list at (x + off[y][x][0], y + off[y][x][1]).  subpixel_offset is a DEVICE [H,W,2] float
 * array indexed by the full-frame pixel (also under a tile-row band); NULL means exactly the call without the suffix.
 *   - Tile lists are not changed: radii, tiles_touched, keys, point_list and ranges are those of the call without
 *     offsets.  Every per-pixel rule (power > 0 and alpha < 1/255 skips, the T < 1e-4 stop, n_contrib, background)
 *     is unchanged; only the sample position moves.
 *   - Any finite offset is allowed; a NaN or Inf offset makes the forward return SFGS_E_BADARG.
 *   - No gradient is formed with respect to the offsets.
 *   - The backward must get the same buffer, with the same contents, as the forward (like norm_raw).
 *   - A tile-row band takes offsets: the reach masks are dilated by the bound over the WHOLE frame's offsets, so a
 *     band's lists and masks are those of the one-call frame and the bands reassemble its images bit for bit.
 *   - ED > 0 (extra_attrs), out_peers and acc_peers return SFGS_E_UNSUPPORTED before any CUDA work; the fused peer
 *     exchanges take offsets through the _subpixel_peers entries below. */
int sfgs_rasterize_forward_subpixel(const sfgs_forward_args* a, const float* subpixel_offset);
int sfgs_rasterize_backward_subpixel(const sfgs_backward_args* a, const float* subpixel_offset);
int sfgs_rasterize_backward_deterministic_subpixel(const sfgs_backward_args* a, const float* subpixel_offset);

/* ---- subpixel offsets with the fused exchanges of the tile-row sharded mode ----------------------------------------
 * sfgs_rasterize_forward_subpixel and sfgs_rasterize_backward_subpixel that also accept out_peers (the image
 * all-gather fused into the band forward) and acc_peers (the reduce-scatter fused into phase 1 of the backward);
 * everything else, validation included, is theirs.  Every rank passes the whole frame's offsets.  ED > 0
 * (extra_attrs) returns SFGS_E_UNSUPPORTED before any CUDA work.  The deterministic backward has no acc_peers form
 * (sfgs_rasterize_backward_deterministic_subpixel keeps rejecting them). */
int sfgs_rasterize_forward_subpixel_peers(const sfgs_forward_args* a, const float* subpixel_offset);
int sfgs_rasterize_backward_subpixel_peers(const sfgs_backward_args* a, const float* subpixel_offset);

/* ---- camera gradients (pose refinement: Camera(..., optimizing=True) of scene/cameras.py) -------------------------
 * The backward above that also writes dL_dcamera, a DEVICE [35] float array: dL/dviewmatrix[16], dL/dprojmatrix[16],
 * dL/dcampos[3], each in its input's element order [4*c + r].  subpixel_offset == NULL and deterministic == 0 give the
 * default backward; a non-NULL offset follows sfgs_rasterize_backward_subpixel and deterministic != 0
 * sfgs_rasterize_backward_deterministic, with their validation (e.g. ED > 0 with either returns SFGS_E_UNSUPPORTED).
 *   - The gradients are the adjoint of the chain dL_dmean3D differentiates: the projected centre through projmatrix
 *     (with its 1/(w + 1e-7) divide), the view-space point through viewmatrix (the depth, and J(t)·W of the EWA
 *     covariance with the Mip coefficient, the same limx/limy clamps), and the SH view direction
 *     normalize(mean - campos).  Discrete decisions (culling, tile lists, clamp sets, alpha and T thresholds, the normal's
 *     sign flip) and the abs-gradient channel contribute nothing; entries the forward never reads (viewmatrix[3], [7],
 *     [11], [15], projmatrix[2], [6], [10], [14]) are exactly 0; with colors_precomp dL/dcampos is exactly 0.
 *   - The sum over Gaussians runs in float64, in an order fixed by P alone, and is rounded to float once: the camera
 *     gradients are bit-reproducible whenever the blend-adjoint sums are (deterministic != 0).
 *   - Every other output is bit-identical to the same backward without camera gradients.
 *   - scratch_alloc is required; the extra scratch is 35 * 8 * ceil(P / 96) bytes (+ alignment) on top of what the
 *     backward it follows needs.
 *   - Phase 0 only: phases 1 and 2 and acc_peers return SFGS_E_UNSUPPORTED, a NULL dL_dcamera SFGS_E_BADARG, before
 *     any CUDA work.  The two-phase (tile-row sharded) backward forms its camera gradients with
 *     sfgs_rasterize_backward_camera_partial.
 * No gradient is formed for tan_fovx / tan_fovy (see sfgs_rasterize_backward_camera_intrinsics) or the subpixel
 * offsets. */
int sfgs_rasterize_backward_camera(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                   float* dL_dcamera);

/* ---- camera and focal-length gradients (focal refinement) ----------------------------------------------------------
 * sfgs_rasterize_backward_camera with dL_dcamera a DEVICE [37] float array: the 35 camera gradients in the layout
 * above, then dL/dtan_fovx and dL/dtan_fovy.  The focal lengths W / (2 tan_fovx) and H / (2 tan_fovy) enter the EWA
 * Jacobian J (and through it the 2D covariance, the Mip coefficient and the conic); the frustum clamp bounds
 * ±1.3 tan_fov move with them, so a clamped t_x / t_y contributes through the bound.  The principal point and the
 * projection entries of the field of view enter through projmatrix and are in dL/dprojmatrix.  The cull, the radius
 * and the tile lists are discrete and contribute nothing.
 *   - The first 35 entries and every other output are bit-identical to sfgs_rasterize_backward_camera's.
 *   - Summation, reproducibility, arguments and rejections as for sfgs_rasterize_backward_camera; the extra scratch is
 *     37 * 8 * ceil(P / 96) bytes (+ alignment). */
int sfgs_rasterize_backward_camera_intrinsics(const sfgs_backward_args* a, const float* subpixel_offset,
                                              int deterministic, float* dL_dcamera);

/* ---- camera partials of a Gaussian slice (camera gradients of the tile-row sharded backward) --------------------
 * Phase 2 of the backward (the per-Gaussian adjoint of Gaussians [gauss_begin, gauss_end)) that also writes
 * dL_dcamera_partial, a DEVICE [ncam] float64 array: the slice's camera terms in the layout above (ncam = 35: pose;
 * ncam = 37: pose and focal), summed in float64 and NOT rounded.  The ranks of a sharded frame add their slices'
 * partials and round once (sfgs/multigpu.py reduce_camera_gradients), so the frame's gradients are rounded once, as
 * the one-call entries round them; they differ from those only by the grouping of the float64 sums.
 *   - The slice's span partials (96 Gaussians each, counted from gauss_begin) are added in an order fixed by the slice
 *     length alone, so with bit-reproducible `acc` the partials are bit-reproducible.  deterministic has no effect on
 *     phase 2 (it has no reductions) and is accepted for symmetry with the other camera entries.
 *   - Every gradient row [gauss_begin, gauss_end) is bit-identical to the same phase-2 call without camera terms.
 *   - An empty slice (and P == 0) writes zeros.
 *   - scratch_alloc is required; the scratch is ncam * 8 * ceil((gauss_end - gauss_begin) / 96) bytes (+ alignment).
 *   - Before any CUDA work: a NULL args or dL_dcamera_partial, ncam other than 35 or 37, or a NULL scratch_alloc
 *     return SFGS_E_BADARG; phase 0 or 1 and ED > 0 (extra_attrs) return SFGS_E_UNSUPPORTED. */
int sfgs_rasterize_backward_camera_partial(const sfgs_backward_args* a, const float* subpixel_offset,
                                           int deterministic, int ncam, double* dL_dcamera_partial);

/* ---- markVisible --------------------------------------------------------- */
int sfgs_mark_visible(int P, const float* means3D, const float* viewmatrix,
                      const float* projmatrix, unsigned char* present, void* stream);

/* ---- introspection of the opaque scratch buffers (used by the parity tests) */
typedef struct sfgs_geom_view {
  const float* rec;            /* [P,16] packed blend record: mx,my, conic.x,.y,.z, opac*coef, depth, pad, r,g,b, nx,ny,nz, pad,pad */
  const float* cov3D;          /* [P,6] */
  const unsigned char* clamped;/* [P] bit0..2 = r,g,b clamped */
  const uint32_t* tiles_touched; /* [P] */
} sfgs_geom_view;
typedef struct sfgs_image_view {
  const uint32_t* n_contrib;   /* [H*W] */
  const uint32_t* ranges;      /* [tiles,2] (start,end) into point_list */
  const uint32_t* tile_count;  /* [tiles] scratch: the per-tile instance histogram, counted back to zero by the key scatter (all zero after a forward) */
} sfgs_image_view;
typedef struct sfgs_binning_view {
  const uint64_t* keys;        /* [R] (depth_bits<<32 | gaussian) grouped by tile, sorted inside each tile */
  const uint32_t* point_list;  /* [R] sorted Gaussian ids */
} sfgs_binning_view;
size_t sfgs_geom_bytes(int P);
size_t sfgs_image_bytes(int width, int height);
size_t sfgs_binning_bytes(long long capacity);
int sfgs_geom_layout(char* base, int P, sfgs_geom_view* out);
int sfgs_image_layout(char* base, int width, int height, sfgs_image_view* out);
int sfgs_binning_layout(char* base, long long capacity, sfgs_binning_view* out);
/* capacity (in tile instances) the last forward on this buffer was sized for; stored in the image buffer header */
long long sfgs_last_capacity(void);
/* how many forwards since load had to run twice because the binning buffer estimate was too small.  The estimate is
 * kept per (device, P, width, height, tile-row band), so alternating frame sizes of one scene costs one re-run per new
 * size at most, not one per switch. */
long long sfgs_overflow_reruns(void);

/* ---- fused per-Gaussian activations (SURVEY.md 8f rank 1) ------------------
 * The torch pre-ops of every render() call as one kernel each way:
 *   scales    = sqrt(exp(scaling_raw)^2 + filter_3D^2)          get_scaling_with_3D_filter, scene/gaussian_model.py:207-213
 *   opacity   = sigmoid(opacity_raw) * sqrt(prod exp(s)^2 / prod(exp(s)^2 + f^2))   get_opacity_with_3D_filter, :237-249
 *   rotations = rotation_raw / max(|rotation_raw|, 1e-12)       get_rotation, :215-217
 * filter_3D is float64 [P] like the reference's (compute_3D_filter, :254-308); the mixed float32/float64
 * promotion of the torch expressions is reproduced and the results are float32 (the `.float()` of
 * gaussian_renderer/__init__.py:137-138).  rotation pointers must be 16-byte aligned. */
int sfgs_activations_forward(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                             const double* filter_3D, float* opacity, float* scales, float* rotations, void* stream);
int sfgs_activations_backward(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                              const double* filter_3D, const float* g_opacity, const float* g_scales,
                              const float* g_rotations, float* g_opacity_raw, float* g_scaling_raw,
                              float* g_rotation_raw, void* stream);

/* ---- appearance path (SURVEY.md 8f rank 2) ----------------------------------
 * The --appearance_enabled branch of render() (gaussian_renderer/__init__.py:105-118), forward, as one tensor-core
 * kernel: EmbeddingModel.forward (scene/gaussian_model.py:45-69: [P,59] -> 128 -> 128 -> 6 MLP on [min(dc,1) | Fourier
 * features | per-camera embedding], x0.01, offset/C0 on the DC term, per-channel multiplier, clamp at 1), eval_sh of
 * the toned coefficients along normalize(xyz - campos) (utils/sh_utils.py), +0.5, clamp at 0  ->  colors_precomp [P,3].
 * W1 is [128, 3+G+E] row-major (torch.nn.Linear.weight), W2 [128,128], W3 [6,128]; features [P,M,3] with M = 1, 4,
 * 9 or 16 ((max_sh_degree+1)^2), gemb [P,G] with G = 24 (4 Fourier frequencies), aemb [E] with E = 32; D = active SH
 * degree, 0..3.  Another M, G or E returns SFGS_E_UNSUPPORTED; (D+1)^2 > M returns SFGS_E_BADARG.  Tensor-core
 * operands are split bf16 pairs (hi + lo, three wgmma per product), fp32 accumulation in registers; the result is
 * within 1e-4 of the float32 torch evaluation.  features and gemb must be 16-byte aligned. */
int sfgs_appearance_forward(int P, int D, int M, const float* features, const float* gemb, int G, const float* aemb,
                            int E, const float* W1, const float* b1, const float* W2, const float* b2,
                            const float* W3, const float* b3, const float* means3D, const float* campos,
                            float* colors, void* stream);
/* Backward of sfgs_appearance_forward, in float32 on the CUDA cores: recomputes the forward from the same inputs (not
 * from its output) and writes dL/d of every input from dL_dcolors [P,3].  Outputs have the inputs' shapes
 * (dL_dfeatures [P,M,3], dL_dgemb [P,G], dL_daemb [E], dL_dW1 [128, 3+G+E], ..., dL_dmeans3D [P,3], dL_dcampos [3]).
 * A NULL output is not computed and skips the work only it needs; every non-NULL output is fully written (no
 * pre-zeroing).  Subgradients at ties are torch's (clamp_max passes where x <= max, clamp_min where x >= min, ReLU
 * where its output is > 0).  Deterministic: sums over Gaussians go through per-chunk float32 partials (chunks of
 * max(512, 64 ceil(P/65536)) Gaussians, a function of P alone) added in float64 in a fixed order and rounded once; no
 * atomics, so repeated calls give identical bits.  P = 0 writes zero sums.  Same argument checks as the forward, also
 * before any CUDA work; scratch_alloc must not be NULL and is called once for
 * sfgs_appearance_backward_scratch_bytes(P) bytes = ceil(P/C) * 20876 * 4 + 1024 (about 80 MB at P = 1M). */
size_t sfgs_appearance_backward_scratch_bytes(int P);
int sfgs_appearance_backward(int P, int D, int M, const float* features, const float* gemb, int G, const float* aemb,
                             int E, const float* W1, const float* b1, const float* W2, const float* b2,
                             const float* W3, const float* b3, const float* means3D, const float* campos,
                             const float* dL_dcolors,
                             float* dL_dfeatures, float* dL_dgemb, float* dL_daemb, float* dL_dW1, float* dL_db1,
                             float* dL_dW2, float* dL_db2, float* dL_dW3, float* dL_db3, float* dL_dmeans3D,
                             float* dL_dcampos, sfgs_alloc_fn scratch_alloc, void* scratch_user, void* stream);

/* ---- 3D smoothing filter (SURVEY.md 8f rank 3) -----------------------------
 * GaussianModel.compute_3D_filter (scene/gaussian_model.py:254-308) as one pass over the Gaussians: for every Gaussian
 * the smallest view depth over the cameras that see it (depth > 0.2, projection inside the image grown by 15 %), the
 * largest such depth for Gaussians no camera sees, divided by the largest focal length, times sqrt(0.2).  float64
 * arithmetic like the reference.  cams: DEVICE array [C][18] doubles per camera = R[9] (camera.R, row-major, used as
 * xyz @ R), T[3], focal_x, focal_y, cx_ori, cy_ori (principal point in pixels: c/2*size + size/2), width, height.
 * filter_3D: [P] doubles out; scratch8: 8 bytes of device scratch. */
int sfgs_compute_3d_filter(int P, const float* xyz, int C, const double* cams, double focal_max, double* filter_3D,
                           void* scratch8, void* stream);

/* ---- adaptive density control (SURVEY 8f rank 3) -------------------------- */
/* train.py:314-315 + GaussianModel.add_densification_stats (scene/gaussian_model.py:744-749) as one in-place pass:
 * for every Gaussian with radii > 0: max_radii2D = max(max_radii2D, radii); grad_accum += |grad[:2]|;
 * grad_accum_abs += |grad[2:]|; grad_accum_abs_max = max(., |grad[2:]|); denom += 1.
 * viewspace_grad: [P,4] floats (16-byte aligned), the .grad of render()'s viewspace_points. */
int sfgs_densification_stats(int P, const float* viewspace_grad, const int* radii, float* max_radii2D,
                             float* grad_accum, float* grad_accum_abs, float* grad_accum_abs_max, float* denom,
                             void* stream);
/* GaussianModel.densify_and_prune (scene/gaussian_model.py:564-742) in two calls.
 * plan: decides every Gaussian's fate from its own values (clone / split / prune rules of :653-735) and returns
 *   totals_host = {surviving originals K, surviving clones KC, split sources S, surviving split sources KS, clone
 *   selections C}; the new point count is K + KC + 2 KS.  abs_threshold: DEVICE scalar (the quantile of :708);
 *   split_scale = percent_dense * extent; world_scale = 0.1 * extent; screen_test = (max_screen_size is truthy).
 *   action: [P] bytes out; block_offsets: 5 * sfgs_densify_plan_blocks(P) ints out; totals_dev: 5 ints of device
 *   scratch.  Synchronises the stream once (the caller must size the new tensors).
 * apply: moves every surviving row of every field to its final place — originals with their Adam moments, clones and
 *   split children with zero moments; a child's position is xyz + R(rotation) (noise * exp(scaling)), its scale
 *   log(exp(scaling) / 1.6).  noise: [2 S, 3] standard-normal floats (child n of source s uses row n S + s, the
 *   reference's .repeat(N, 1) order).  Fields: 0 xyz(3) 1 f_dc 2 f_rest 3 opacity(1) 4 scaling(3) 5 rotation(4), then
 *   up to two more per-Gaussian parameters; src/dst[_exp_avg[_sq]] are host arrays of n_fields device pointers (the
 *   three moment arrays may all be NULL when the optimizer has no state yet). */
int sfgs_densify_plan_blocks(int P);
int sfgs_densify_plan(int P, const float* grad_accum, const float* grad_accum_abs, const float* denom,
                      const float* scaling, const float* opacity, float max_grad, const float* abs_threshold,
                      float split_scale, float min_opacity, int screen_test, float max_screen_size, float world_scale,
                      unsigned char* action, int* block_offsets, int* totals_dev, int totals_host[5], void* stream);
int sfgs_densify_apply(int P, const unsigned char* action, const int* block_offsets, const int totals[5],
                       const float* noise, int n_fields, const int* widths, const float* const* src,
                       const float* const* src_exp_avg, const float* const* src_exp_avg_sq, float* const* dst,
                       float* const* dst_exp_avg, float* const* dst_exp_avg_sq, void* stream);

/* ---- fused SSIM ---------------------------------------------------------- */
int sfgs_fusedssim_forward(float C1, float C2, int B, int CH, int H, int W,
                           const float* img1, const float* img2, int train,
                           float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq,
                           float* dm_dsigma12, void* stream);
int sfgs_fusedssim_backward(float C1, float C2, int B, int CH, int H, int W,
                            const float* img1, const float* img2, const float* dL_dmap,
                            const float* dm_dmu1, const float* dm_dsigma1_sq,
                            const float* dm_dsigma12, float* dL_dimg1, void* stream);

/* ---- simple-knn ---------------------------------------------------------- */
/* mean squared distance to the 3 nearest neighbours; scratch via callback */
int sfgs_dist2_knn3(int P, const float* points, float* mean_dist2,
                    sfgs_alloc_fn scratch_alloc, void* scratch_user, void* stream);

/* ---- optional per-stage device timing ---------------------------------------- */
/* Stage order: 0 fwd zero-fill, 1 preprocess, 2 tile scan, 3 key emission, 4 tile sort, 5 blend fwd,
 * 6 bwd zero-fill, 7 blend bwd, 8 per-Gaussian bwd.  When enabled, every stage is bracketed by CUDA events
 * on the caller's stream; sfgs_profile_read() synchronises those events and returns accumulated
 * milliseconds and launch counts per stage (returns the number of stages).  Off by default. */
#define SFGS_NUM_STAGES 9
int sfgs_profile_enable(int on);
int sfgs_profile_read(double* ms_total, long long* launches, int n);

/* Queue a one-thread kernel that spins ~20 us and writes the SM clock it observed (MHz) to *out_mhz_device.
 * Used by bench.py to sample clocks in-stream during the timed loop without touching NVML. */
int sfgs_sm_clock_probe(float* out_mhz_device, void* stream);

/* Self-test hook for the parity tests: y_replica[i] = the expf routine the blend kernels use (csrc/sfgs_common.cuh,
 * sfgs_expf), y_expf[i] = the compiler's expf(x[i]); the two must agree bit for bit, because the alpha thresholds
 * that decide n_contrib are evaluated on it. */
int sfgs_selftest_expf(int n, const float* x, float* y_replica, float* y_expf, void* stream);

/* ---- misc ---------------------------------------------------------------- */
const char* sfgs_last_error(void);
/* sizeof() of the ABI structs as compiled (0 forward_args, 1 backward_args, 2 geom_view, 3 image_view,
 * 4 binning_view) so that foreign-language bindings can verify their mirror definitions */
size_t sfgs_sizeof(int which);
int sfgs_version(void);
/* number of kernel launches issued by this library since load (for bench.py's gpu_launches) */
long long sfgs_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* SFGS_H_INCLUDED */
