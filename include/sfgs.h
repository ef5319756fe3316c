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
 * W1 is [128, 3+G+E] row-major (torch.nn.Linear.weight), W2 [128,128], W3 [6,128]; features [P,M,3] with M = 16,
 * gemb [P,G] with G = 24 (4 Fourier frequencies), aemb [E] with E = 32; D = active SH degree.  Tensor-core
 * operands are split bf16 pairs (hi + lo, three wgmma per product), fp32 accumulation in registers; the result is
 * within 1e-4 of the float32 torch evaluation.  features and gemb must be 16-byte aligned. */
int sfgs_appearance_forward(int P, int D, int M, const float* features, const float* gemb, int G, const float* aemb,
                            int E, const float* W1, const float* b1, const float* W2, const float* b2,
                            const float* W3, const float* b3, const float* means3D, const float* campos,
                            float* colors, void* stream);

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
