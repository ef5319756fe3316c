// sfgs_api.cu — C ABI entry points (see include/sfgs.h) and stage orchestration.
//
// Forward  = zero tile histogram -> preprocess -> tile scan -> key emission ->
//            per-tile sort -> blend, all queued on the caller's stream with no
//            host round trip in between.  num_rendered is final after the tile
//            scan; its 32-byte copy is queued there and the host waits on that
//            event only, AFTER every kernel of the forward has been queued, so it
//            returns while sort + blend are still running and the caller can queue
//            the backward without a bubble (the reference blocks on a cudaMemcpy in
//            the middle of its forward, rasterizer_impl.cu:286-287, because it must
//            size the binning buffer before it can launch anything else).
//            The binning buffer is sized from a running estimate instead and the
//            tail of the pipeline is re-run in the rare case it was too small.
// Backward = zero accumulators -> tile blend adjoint -> per-Gaussian adjoint.
// Deterministic backward = clear the written flags -> ORDERED blend adjoint (partial rows, no reductions) ->
//            fixed-order float64 sum of each Gaussian's rows into acc (sfgs_bwd_order.cu) -> per-Gaussian adjoint.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <mutex>
#include <vector>
#include "sfgs_common.cuh"

std::atomic<long long> g_sfgs_launches{0};

void sfgs_launch_preprocess(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, unsigned long long capacity, float focal_x, float focal_y,
                            const float* tan_fov, bool ortho, bool ray_depth, bool plane_normals, cudaStream_t st);
void sfgs_launch_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present,
                              cudaStream_t st);
void sfgs_launch_tile_scan(const ImageLayout& im, unsigned long long capacity, cudaStream_t st);
void sfgs_launch_forward_status(const ImageLayout& im, unsigned int* status, cudaStream_t st);
void sfgs_launch_scatter(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P,
                         unsigned long long capacity, bool dilate, cudaStream_t st);
void sfgs_launch_tile_sort(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P, bool dilate,
                           cudaStream_t st);
void sfgs_launch_offset_bound(const ImageLayout& im, int W, int H, const float* off, cudaStream_t st);
void sfgs_launch_render_fwd(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, const float* off, float t, float* out_depth_q,
                            uint32_t* out_depth_q_pos, float* out_dist, float* out_dist_state, bool ray_depth,
                            cudaStream_t st);
void sfgs_launch_render_bwd(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, float* acc, float* part, unsigned char* written, const float* off,
                            bool guarded, const float* dist_state, const float* dL_dpix_dist, bool ray_depth,
                            cudaStream_t st);
void sfgs_launch_depth_q_adjoint(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                                 const BinningLayout& b, const uint32_t* depth_q_pos, const float* dL_dpix_depth_q,
                                 float* acc, float* part, bool ray_depth, const float* off, cudaStream_t st);
size_t sfgs_order_scratch_bytes(int P, long long R);
SfgsOrderScratch sfgs_order_scratch(char* base, int P, long long R);
void sfgs_launch_order_prepare(int P, const GeomLayout& g, const ImageLayout& im, const BinningLayout& b,
                               const int* radii, int band0, int band1, const SfgsOrderScratch& o, bool guarded,
                               cudaStream_t st);
void sfgs_launch_order_reduce(int P, const GeomLayout& g, const int* radii, bool all_rows, const SfgsOrderScratch& o,
                              float* acc, const uint32_t* hdr_guard, cudaStream_t st);
int sfgs_launch_activations_fwd(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                                const double* filter_3D, float* opacity, float* scales, float* rotations,
                                cudaStream_t st);
int sfgs_launch_activations_bwd(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                                const double* filter_3D, const float* g_opacity, const float* g_scales,
                                const float* g_rotations, float* g_opacity_raw, float* g_scaling_raw,
                                float* g_rotation_raw, cudaStream_t st);
void sfgs_launch_gauss_bwd(const sfgs_backward_args* a, const GeomLayout& g, float focal_x, float focal_y,
                           const float* acc, int g_begin, int g_end, int acc_row0, double* cam_part, int ncam,
                           const float* tan_fov, bool ortho, bool ray_depth, bool plane_normals, cudaStream_t st);
size_t sfgs_camera_scratch_bytes(int P, int ncam);
void sfgs_launch_camera_reduce(int P, int ncam, const double* cam_part, float* dL_dcamera, cudaStream_t st);
void sfgs_launch_camera_partial_reduce(int n, int ncam, const double* cam_part, double* dL_dcamera, cudaStream_t st);
void sfgs_launch_acc_clear_visible(int P, const int* radii, float* acc, cudaStream_t st);

namespace {

// One thread spins ~20 us and reports SM cycles per microsecond: the SM clock actually applied while the
// surrounding work runs, measured in-stream (polling NVML from the host during a run perturbs it).
__global__ void sm_clock_probe_kernel(float* out_mhz) {
  unsigned long long t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  const long long c0 = clock64();
  do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < 20000ull);
  const long long c1 = clock64();
  *out_mhz = (float)((double)(c1 - c0) * 1000.0 / (double)(t1 - t0));
}

// self-test hook: the blend kernels' expf replica next to the compiler's expf (tests sweep them for bit equality)
__global__ void expf_selftest_kernel(int n, const float* __restrict__ x, float* __restrict__ y_replica,
                                     float* __restrict__ y_expf) {
  const SfgsExpConsts ek = sfgs_exp_consts(n < 0 ? 1u : 0u);   // a zero the compiler cannot fold, like the kernels' one
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    y_replica[i] = sfgs_expf(x[i], ek);
    y_expf[i] = exp(x[i]);
  }
}

thread_local char t_err[512] = "";
std::atomic<long long> g_last_capacity{0};
std::atomic<long long> g_overflow_reruns{0};   // forwards that had to run twice because the binning estimate was too small

// Running estimate of the instance count, keyed by what determines it to first order: (device, P, image size, band).
// A training loop alternates 1080p train views, 1024^2 pseudo-views and low-resolution evaluation renders of the
// same scene; one process-wide estimate would overflow (and re-run the forward) on every switch upward.
struct CapKey { int dev, P, W, H, b0, b1; };
struct CapEntry { CapKey k; long long R; unsigned long long stamp; };
std::mutex g_cap_mu;
std::vector<CapEntry> g_cap_tab;
unsigned long long g_cap_clock = 0;
constexpr size_t CAP_TAB_MAX = 64;
bool cap_same(const CapKey& a, const CapKey& b) { return a.dev == b.dev && a.P == b.P && a.W == b.W && a.H == b.H && a.b0 == b.b0 && a.b1 == b.b1; }
long long cap_lookup(const CapKey& k) {
  std::lock_guard<std::mutex> lk(g_cap_mu);
  for (auto& e : g_cap_tab) if (cap_same(e.k, k)) { e.stamp = ++g_cap_clock; return e.R; }
  return -1;
}
void cap_store(const CapKey& k, long long R) {
  std::lock_guard<std::mutex> lk(g_cap_mu);
  for (auto& e : g_cap_tab) if (cap_same(e.k, k)) { e.R = R; e.stamp = ++g_cap_clock; return; }
  if (g_cap_tab.size() >= CAP_TAB_MAX) {   // evict the least recently used entry
    size_t lru = 0;
    for (size_t i = 1; i < g_cap_tab.size(); i++) if (g_cap_tab[i].stamp < g_cap_tab[lru].stamp) lru = i;
    g_cap_tab[lru] = CapEntry{k, R, ++g_cap_clock};
  } else {
    g_cap_tab.push_back(CapEntry{k, R, ++g_cap_clock});
  }
}

int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
  if (e != cudaSuccess) snprintf(t_err, sizeof(t_err), "%s: %s", what, cudaGetErrorString(e));
  else snprintf(t_err, sizeof(t_err), "%s", what);
  return code;
}
// a rejection by an entry point's checks
int fail_in(const char* entry, int code, const char* what) {
  snprintf(t_err, sizeof(t_err), "%s: %s", entry, what);
  return code;
}

#define CU(call)                                                   \
  do {                                                             \
    cudaError_t _e = (call);                                       \
    if (_e != cudaSuccess) return fail(SFGS_E_CUDA, #call, _e);    \
  } while (0)

#define STAGE_CHECK(name)                                                              \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) return fail(SFGS_E_CUDA, "launch " name, _e);               \
    if (debug) {                                                                       \
      _e = cudaStreamSynchronize(st);                                                  \
      if (_e != cudaSuccess) return fail(SFGS_E_CUDA, "stage " name, _e);              \
    }                                                                                  \
  } while (0)

// ---- optional per-stage device timing (bench.py's roofline uses it; off by default) ----
enum { ST_FWD_ZERO = 0, ST_PREPROCESS, ST_SCAN, ST_EMIT, ST_SORT, ST_RENDER_FWD, ST_BWD_ZERO, ST_RENDER_BWD, ST_GAUSS_BWD,
       ST_BWD_ORDER, ST_COUNT };
struct StageProf {
  bool on = false;
  struct Span { cudaEvent_t a, b; int stage; };
  std::vector<Span> spans;
  std::vector<Span> pool;
  double ms[ST_COUNT] = {0};
  long long n[ST_COUNT] = {0};
  std::mutex mu;   // begin/end may be called from several host threads (one per device)
  void begin(int stage, cudaStream_t st) {
    if (!on) return;
    std::lock_guard<std::mutex> lk(mu);
    Span s;
    if (!pool.empty()) { s = pool.back(); pool.pop_back(); }
    else { cudaEventCreate(&s.a); cudaEventCreate(&s.b); }
    s.stage = stage;
    cudaEventRecord(s.a, st);
    spans.push_back(s);
  }
  void end(cudaStream_t st) {
    if (!on) return;
    std::lock_guard<std::mutex> lk(mu);
    if (spans.empty()) return;
    cudaEventRecord(spans.back().b, st);
  }
  void collect() {
    std::lock_guard<std::mutex> lk(mu);
    for (auto& s : spans) {
      float t = 0.f;
      if (cudaEventSynchronize(s.b) == cudaSuccess && cudaEventElapsedTime(&t, s.a, s.b) == cudaSuccess) { ms[s.stage] += t; n[s.stage]++; }
      pool.push_back(s);
    }
    spans.clear();
  }
};
StageProf g_prof;
std::mutex g_prof_mu;
#define PROF_BEGIN(stage) g_prof.begin(stage, st)
#define PROF_END() g_prof.end(st)

// Pinned landing zone of the image header + the event the host waits on: one per (host thread, device) — a CUDA
// event belongs to the device that was current when it was created and cannot be recorded on another device's stream.
struct PinnedHdr {
  uint32_t* p = nullptr;
  cudaEvent_t ev = nullptr;
  ~PinnedHdr() { /* leaked on purpose: the CUDA context may already be gone at exit */ }
  uint32_t* get() {
    if (!p) {
      if (cudaHostAlloc((void**)&p, IMG_HDR_WORDS * sizeof(uint32_t), cudaHostAllocPortable) != cudaSuccess) p = nullptr;
      if (p && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) { ev = nullptr; }
    }
    return (p && ev) ? p : nullptr;
  }
};
constexpr int MAX_DEVICES = 64;
thread_local PinnedHdr t_hdr_dev[MAX_DEVICES];

// What one rasterizer entry point asks for, beyond its sfgs_forward_args / sfgs_backward_args.  The entry's checks
// (check_forward, check_backward) and the stages read their options from here.
struct FwdCall {
  const char* name;                   // the entry point without its sfgs_rasterize_ prefix: the errors name it
  bool graph;                         // sfgs_rasterize_forward_graph: one pass at capacity_hint, no host wait
  const float* off = nullptr;         // subpixel offsets [H,W,2], or NULL
  bool peers_with_off = false;        // out_peers may come with offsets (the _subpixel_peers entry)
  const float* tan_fov = nullptr;     // graph: NULL or the DEVICE [2] intrinsics
  unsigned int* status = nullptr;     // graph: the DEVICE status word the frame's error flags are ORed into
  bool ortho = false;                 // the orthographic camera (sfgs_rasterize_forward_ortho)
  bool depth_q = false;               // the depth quantile (sfgs_rasterize_forward_depth_quantile) ...
  float quantile = 0.f;               // ... at level q: the record crossing T = 1 - q gives depth_q [H,W] ...
  float* out_depth_q = nullptr;
  uint32_t* out_depth_q_pos = nullptr;   // ... and its 1-based list position [H,W]
  bool dist = false;                  // the depth distortion (sfgs_rasterize_forward_distortion): R [H,W] ...
  float* out_distortion = nullptr;
  float* out_distortion_state = nullptr;   // ... and the state (mu, M2) [2,H,W] its adjoint reads
  bool ray_depth = false;             // ray depth (sfgs_rasterize_forward_ray_depth), with or without depth_q
  bool plane_normals = false;         // plane normals (sfgs_rasterize_forward_plane_normals), with ray_depth
};

struct BwdCall {
  const char* name;                   // the entry point without its sfgs_rasterize_ prefix: the errors name it
  enum Kind { EAGER, CAMERA, CAMERA_PARTIAL, GRAPH } kind;
  const float* off = nullptr;         // subpixel offsets [H,W,2] (the forward's), or NULL
  bool peers_with_off = false;        // acc_peers may come with offsets (the _subpixel_peers entry)
  bool deterministic = false;
  int ncam = 0;                       // camera terms: 0, 35 (pose) or 37 (pose and focal)
  float* dL_dcamera = nullptr;        // CAMERA, GRAPH: the DEVICE [ncam] camera gradients
  double* dL_dcamera_partial = nullptr;   // CAMERA_PARTIAL: the DEVICE [ncam] float64 sums of the Gaussian slice
  const float* tan_fov = nullptr;     // GRAPH: NULL or the DEVICE [2] intrinsics the per-Gaussian adjoint reads
  bool ortho = false;                 // the orthographic camera (sfgs_rasterize_backward_ortho)
  bool depth_q = false;               // the depth quantile's adjoint (sfgs_rasterize_backward_depth_quantile) ...
  const uint32_t* depth_q_pos = nullptr;      // ... from the forward's positions [H,W] ...
  const float* dL_dpix_depth_q = nullptr;     // ... and the cotangent of depth_q [H,W]
  bool dist = false;                  // the depth distortion's adjoint (sfgs_rasterize_backward_distortion) ...
  const float* distortion_state = nullptr;    // ... from the forward's state [2,H,W] ...
  const float* dL_dpix_distortion = nullptr;  // ... and the cotangent of R [H,W]
  bool ray_depth = false;             // ray depth's adjoint (sfgs_rasterize_backward_ray_depth), with or without depth_q
  bool plane_normals = false;         // plane normals' adjoint (sfgs_rasterize_backward_plane_normals), with ray_depth
};

int rasterize_forward(const sfgs_forward_args* a, const FwdCall& c);
int rasterize_backward(const sfgs_backward_args* a, const BwdCall& c);

}  // namespace

extern "C" {

// error entry for the other translation units (SSIM, KNN): same thread-local text as the rasterizer's
int sfgs_set_error(int code, const char* what, int cuda_error) { return fail(code, what, (cudaError_t)cuda_error); }

const char* sfgs_last_error(void) { return t_err; }
int sfgs_version(void) { return SFGS_VERSION; }
long long sfgs_launch_count(void) { return g_sfgs_launches.load(); }
long long sfgs_last_capacity(void) { return g_last_capacity.load(); }
long long sfgs_overflow_reruns(void) { return g_overflow_reruns.load(); }

size_t sfgs_geom_bytes(int P) { return GeomLayout(nullptr, (size_t)(P > 0 ? P : 0)).bytes; }
size_t sfgs_image_bytes(int width, int height) { return ImageLayout(nullptr, width, height).bytes; }
size_t sfgs_binning_bytes(long long capacity) { return BinningLayout(nullptr, (size_t)(capacity > 0 ? capacity : 0)).bytes; }

int sfgs_geom_layout(char* base, int P, sfgs_geom_view* out) {
  if (!base || !out) return fail(SFGS_E_BADARG, "sfgs_geom_layout: null");
  GeomLayout g(sfgs_align_ptr(base), (size_t)P);
  out->rec = g.rec; out->cov3D = g.cov3D; out->clamped = g.clamped; out->tiles_touched = g.tiles_touched;
  return SFGS_OK;
}
int sfgs_image_layout(char* base, int width, int height, sfgs_image_view* out) {
  if (!base || !out) return fail(SFGS_E_BADARG, "sfgs_image_layout: null");
  ImageLayout im(sfgs_align_ptr(base), width, height);
  out->n_contrib = im.n_contrib; out->ranges = (const uint32_t*)im.ranges; out->tile_count = im.tile_count;
  return SFGS_OK;
}
int sfgs_binning_layout(char* base, long long capacity, sfgs_binning_view* out) {
  if (!base || !out) return fail(SFGS_E_BADARG, "sfgs_binning_layout: null");
  BinningLayout b(sfgs_align_ptr(base), (size_t)capacity);
  out->keys = b.keys; out->point_list = b.point_list;
  return SFGS_OK;
}

int sfgs_rasterize_forward(const sfgs_forward_args* a) { return rasterize_forward(a, {"forward", false}); }
int sfgs_rasterize_backward(const sfgs_backward_args* a) { return rasterize_backward(a, {"backward", BwdCall::EAGER}); }
int sfgs_rasterize_backward_deterministic(const sfgs_backward_args* a) {
  return rasterize_backward(a, {"backward_deterministic", BwdCall::EAGER, nullptr, false, true});
}

int sfgs_rasterize_forward_subpixel(const sfgs_forward_args* a, const float* subpixel_offset) {
  return rasterize_forward(a, {"forward_subpixel", false, subpixel_offset});
}
int sfgs_rasterize_forward_subpixel_peers(const sfgs_forward_args* a, const float* subpixel_offset) {
  return rasterize_forward(a, {"forward_subpixel_peers", false, subpixel_offset, true});
}
int sfgs_rasterize_backward_subpixel(const sfgs_backward_args* a, const float* subpixel_offset) {
  return rasterize_backward(a, {"backward_subpixel", BwdCall::EAGER, subpixel_offset});
}
int sfgs_rasterize_backward_subpixel_peers(const sfgs_backward_args* a, const float* subpixel_offset) {
  return rasterize_backward(a, {"backward_subpixel_peers", BwdCall::EAGER, subpixel_offset, true});
}
int sfgs_rasterize_backward_deterministic_subpixel(const sfgs_backward_args* a, const float* subpixel_offset) {
  return rasterize_backward(a, {"backward_deterministic_subpixel", BwdCall::EAGER, subpixel_offset, false, true});
}

int sfgs_rasterize_backward_camera(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                   float* dL_dcamera) {
  return rasterize_backward(a, {"backward_camera", BwdCall::CAMERA, subpixel_offset, false, deterministic != 0, 35,
                                dL_dcamera});
}

int sfgs_rasterize_backward_camera_intrinsics(const sfgs_backward_args* a, const float* subpixel_offset,
                                              int deterministic, float* dL_dcamera) {
  return rasterize_backward(a, {"backward_camera_intrinsics", BwdCall::CAMERA, subpixel_offset, false,
                                deterministic != 0, 37, dL_dcamera});
}

int sfgs_rasterize_backward_camera_partial(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                           int ncam, double* dL_dcamera_partial) {
  return rasterize_backward(a, {"backward_camera_partial", BwdCall::CAMERA_PARTIAL, subpixel_offset, false,
                                deterministic != 0, ncam, nullptr, dL_dcamera_partial});
}

int sfgs_rasterize_forward_graph(const sfgs_forward_args* a, const float* subpixel_offset, const float* tan_fov,
                                 unsigned int* status) {
  return rasterize_forward(a, {"forward_graph", true, subpixel_offset, false, tan_fov, status});
}

int sfgs_rasterize_backward_graph(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                  const float* tan_fov, float* dL_dcamera, int ncam) {
  return rasterize_backward(a, {"backward_graph", BwdCall::GRAPH, subpixel_offset, false, deterministic != 0, ncam,
                                ncam != 0 ? dL_dcamera : nullptr, nullptr, tan_fov});
}

long long sfgs_capacity_estimate(int device, int P, int width, int height) {
  return cap_lookup(CapKey{device, P, width, height, 0, 0});
}

int sfgs_rasterize_forward_ortho(const sfgs_forward_args* a, const float* subpixel_offset) {
  return rasterize_forward(a, {"forward_ortho", false, subpixel_offset, false, nullptr, nullptr, true});
}

int sfgs_rasterize_backward_ortho(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic) {
  return rasterize_backward(a, {"backward_ortho", BwdCall::EAGER, subpixel_offset, false, deterministic != 0, 0, nullptr,
                                nullptr, nullptr, true});
}

int sfgs_rasterize_forward_depth_quantile(const sfgs_forward_args* a, const float* subpixel_offset, int ortho,
                                          float quantile, float* out_depth_q, uint32_t* out_depth_q_pos) {
  FwdCall c{"forward_depth_quantile", false, subpixel_offset};
  c.ortho = ortho != 0;
  c.depth_q = true;
  c.quantile = quantile;
  c.out_depth_q = out_depth_q;
  c.out_depth_q_pos = out_depth_q_pos;
  return rasterize_forward(a, c);
}

int sfgs_rasterize_backward_depth_quantile(const sfgs_backward_args* a, const float* subpixel_offset, int ortho,
                                           int deterministic, const uint32_t* depth_q_pos,
                                           const float* dL_dpix_depth_q, float* dL_dcamera, int ncam) {
  // ncam > 0: the checks and the stages of sfgs_rasterize_backward_camera[_intrinsics] (a bad ncam is rejected first)
  BwdCall c{"backward_depth_quantile", ncam > 0 ? BwdCall::CAMERA : BwdCall::EAGER, subpixel_offset, false,
            deterministic != 0, ncam, ncam > 0 ? dL_dcamera : nullptr};
  c.ortho = ortho != 0;
  c.depth_q = true;
  c.depth_q_pos = depth_q_pos;
  c.dL_dpix_depth_q = dL_dpix_depth_q;
  return rasterize_backward(a, c);
}

int sfgs_rasterize_forward_distortion(const sfgs_forward_args* a, const float* subpixel_offset, int ortho,
                                      float* out_distortion, float* out_distortion_state) {
  FwdCall c{"forward_distortion", false, subpixel_offset};
  c.ortho = ortho != 0;
  c.dist = true;
  c.out_distortion = out_distortion;
  c.out_distortion_state = out_distortion_state;
  return rasterize_forward(a, c);
}

int sfgs_rasterize_backward_distortion(const sfgs_backward_args* a, const float* subpixel_offset, int ortho,
                                       int deterministic, const float* distortion_state,
                                       const float* dL_dpix_distortion, float* dL_dcamera, int ncam) {
  // ncam > 0: the checks and the stages of sfgs_rasterize_backward_camera[_intrinsics] (a bad ncam is rejected first)
  BwdCall c{"backward_distortion", ncam > 0 ? BwdCall::CAMERA : BwdCall::EAGER, subpixel_offset, false,
            deterministic != 0, ncam, ncam > 0 ? dL_dcamera : nullptr};
  c.ortho = ortho != 0;
  c.dist = true;
  c.distortion_state = distortion_state;
  c.dL_dpix_distortion = dL_dpix_distortion;
  return rasterize_backward(a, c);
}

int sfgs_rasterize_forward_ray_depth(const sfgs_forward_args* a, const float* subpixel_offset, int ortho,
                                     float quantile, float* out_depth_q, uint32_t* out_depth_q_pos) {
  FwdCall c{"forward_ray_depth", false, subpixel_offset};
  c.ortho = ortho != 0;
  c.ray_depth = true;
  c.depth_q = out_depth_q != nullptr;     // NULL: no quantile
  c.quantile = quantile;
  c.out_depth_q = out_depth_q;
  c.out_depth_q_pos = out_depth_q_pos;
  return rasterize_forward(a, c);
}

int sfgs_rasterize_backward_ray_depth(const sfgs_backward_args* a, const float* subpixel_offset, int ortho,
                                      int deterministic, const uint32_t* depth_q_pos, const float* dL_dpix_depth_q,
                                      float* dL_dcamera, int ncam) {
  // ncam > 0: the checks and the stages of sfgs_rasterize_backward_camera[_intrinsics] (a bad ncam is rejected first)
  BwdCall c{"backward_ray_depth", ncam > 0 ? BwdCall::CAMERA : BwdCall::EAGER, subpixel_offset, false,
            deterministic != 0, ncam, ncam > 0 ? dL_dcamera : nullptr};
  c.ortho = ortho != 0;
  c.ray_depth = true;
  c.depth_q = depth_q_pos != nullptr || dL_dpix_depth_q != nullptr;   // both NULL: no quantile
  c.depth_q_pos = depth_q_pos;
  c.dL_dpix_depth_q = dL_dpix_depth_q;
  return rasterize_backward(a, c);
}

int sfgs_rasterize_forward_plane_normals(const sfgs_forward_args* a, const float* subpixel_offset, int ortho,
                                         float quantile, float* out_depth_q, uint32_t* out_depth_q_pos) {
  FwdCall c{"forward_plane_normals", false, subpixel_offset};
  c.ortho = ortho != 0;
  c.ray_depth = true;
  c.plane_normals = true;
  c.depth_q = out_depth_q != nullptr;     // NULL: no quantile
  c.quantile = quantile;
  c.out_depth_q = out_depth_q;
  c.out_depth_q_pos = out_depth_q_pos;
  return rasterize_forward(a, c);
}

int sfgs_rasterize_backward_plane_normals(const sfgs_backward_args* a, const float* subpixel_offset, int ortho,
                                          int deterministic, const uint32_t* depth_q_pos,
                                          const float* dL_dpix_depth_q, float* dL_dcamera, int ncam) {
  // ncam > 0: the checks and the stages of sfgs_rasterize_backward_camera[_intrinsics] (a bad ncam is rejected first)
  BwdCall c{"backward_plane_normals", ncam > 0 ? BwdCall::CAMERA : BwdCall::EAGER, subpixel_offset, false,
            deterministic != 0, ncam, ncam > 0 ? dL_dcamera : nullptr};
  c.ortho = ortho != 0;
  c.ray_depth = true;
  c.plane_normals = true;
  c.depth_q = depth_q_pos != nullptr || dL_dpix_depth_q != nullptr;   // both NULL: no quantile
  c.depth_q_pos = depth_q_pos;
  c.dL_dpix_depth_q = dL_dpix_depth_q;
  return rasterize_backward(a, c);
}

}  // extern "C"

namespace {

// Every rejection of the forward entries, in the order that decides which one an entry reports; all before any CUDA
// work.  Messages are "<entry>: <what>".
// the orthographic camera's half-extents s_x, s_y (carried by tan_fovx, tan_fovy): finite and > 0
bool ortho_extent_ok(float sx, float sy) { return std::isfinite(sx) && std::isfinite(sy) && sx > 0.f && sy > 0.f; }
// the depth quantile's level q: finite, 0 < q < 1
bool quantile_ok(float q) { return std::isfinite(q) && q > 0.f && q < 1.f; }

// "<entry>: <subject> not supported with <feature>"
int reject_with(const char* entry, const char* subject, const char* feature) {
  char what[128];
  snprintf(what, sizeof(what), "%s not supported with %s", subject, feature);
  return fail_in(entry, SFGS_E_UNSUPPORTED, what);
}

// The forward's rejections of a per-pixel output (the depth quantile, the depth distortion), in order: null outputs,
// the output's own bad argument `bad_arg` (or nullptr), then extra_attrs, tile-row bands and out_peers.
int check_pixel_output(const sfgs_forward_args* a, const char* entry, bool null_out, const char* null_what,
                       const char* bad_arg, const char* feature) {
  if (null_out) return fail_in(entry, SFGS_E_BADARG, null_what);
  if (bad_arg) return fail_in(entry, SFGS_E_BADARG, bad_arg);
  if (a->ED > 0) return reject_with(entry, "extra_attrs are", feature);
  if (a->tile_row_begin != 0 || a->tile_row_end != 0) return reject_with(entry, "tile-row bands are", feature);
  if (a->out_peers != nullptr) return reject_with(entry, "out_peers are", feature);
  return SFGS_OK;
}

int check_forward(const sfgs_forward_args* a, const FwdCall& c) {
  const auto reject = [&c](int code, const char* what) { return fail_in(c.name, code, what); };
  if (!a) return reject(SFGS_E_BADARG, "null args");
  if (c.ray_depth) {
    // with a quantile (out_depth_q given) its own arguments first; every unsupported option is then reported as ray
    // depth's, or as plane normals' (the quantile's check below finds nothing left)
    const char* feature = c.plane_normals ? "plane normals" : "ray depth";
    const char* bad_q = !c.depth_q || quantile_ok(c.quantile) ? nullptr : "the quantile must be finite with 0 < q < 1";
    if (const int rc = check_pixel_output(a, c.name, c.depth_q && !c.out_depth_q_pos, "null out_depth_q_pos", bad_q,
                                          feature))
      return rc;
    // the normal is the ray-depth plane's, not an input
    if (c.plane_normals && a->norm3D_precomp != nullptr) return reject_with(c.name, "norm3D_precomp is", feature);
  }
  if (c.depth_q) {
    const char* bad_q = quantile_ok(c.quantile) ? nullptr : "the quantile must be finite with 0 < q < 1";
    if (const int rc = check_pixel_output(a, c.name, !c.out_depth_q || !c.out_depth_q_pos,
                                          "null out_depth_q or out_depth_q_pos", bad_q, "the depth quantile"))
      return rc;
  }
  if (c.dist) {
    if (const int rc = check_pixel_output(a, c.name, !c.out_distortion || !c.out_distortion_state,
                                          "null out_distortion or out_distortion_state", nullptr, "the depth distortion"))
      return rc;
  }
  if (c.ortho) {
    if (a->tile_row_begin != 0 || a->tile_row_end != 0)
      return reject(SFGS_E_UNSUPPORTED, "tile-row bands are not supported with an orthographic camera");
    if (a->out_peers != nullptr) return reject(SFGS_E_UNSUPPORTED, "out_peers are not supported with an orthographic camera");
    if (!ortho_extent_ok(a->tan_fovx, a->tan_fovy))
      return reject(SFGS_E_BADARG, "the half-extents tan_fovx, tan_fovy must be finite and > 0");
  }
  if (c.graph) {
    if (!c.status) return reject(SFGS_E_BADARG, "null status word");
    if (a->debug) return reject(SFGS_E_BADARG, "debug synchronises after every stage and cannot be captured");
    if (a->capacity_hint <= 0)
      return reject(SFGS_E_BADARG, "capacity_hint must be > 0 (the binning capacity of the captured frame)");
    if (a->tile_row_begin != 0 || a->tile_row_end != 0)
      return reject(SFGS_E_UNSUPPORTED, "tile-row bands are not supported under graph capture");
    if (a->out_peers != nullptr) return reject(SFGS_E_UNSUPPORTED, "out_peers are not supported under graph capture");
  }
  if (c.off != nullptr) {
    // extra_attrs have no kernels with offsets; the _subpixel entry has always rejected the fused peer exchange
    if (a->ED > 0) return reject(SFGS_E_UNSUPPORTED, "extra_attrs are not supported with subpixel offsets");
    if (!c.peers_with_off && a->out_peers != nullptr)
      return reject(SFGS_E_UNSUPPORTED,
                    "out_peers are not supported by this entry; use sfgs_rasterize_forward_subpixel_peers");
  }
  if (a->P < 0 || a->width <= 0 || a->height <= 0) return reject(SFGS_E_BADARG, "bad sizes");
  if (a->ED < 0 || a->ED > SFGS_MAX_EXTRA) return reject(SFGS_E_BADARG, "ED out of range");
  if (a->tile_row_begin < 0 || a->tile_row_end < a->tile_row_begin) return reject(SFGS_E_BADARG, "bad tile-row band");
  const bool peer_out = a->out_peers != nullptr && a->n_out_peers > 0;
  if (peer_out && a->n_out_peers > 8) return reject(SFGS_E_BADARG, "at most 8 out_peers");
  if ((!peer_out && (!a->out_color || !a->out_depth || !a->out_norm || !a->out_alpha)) || (a->P > 0 && !a->radii))
    return reject(SFGS_E_BADARG, "null output");
  if (!a->geom_alloc || !a->binning_alloc || !a->image_alloc) return reject(SFGS_E_BADARG, "null allocator");
  if (a->P > 0) {
    if (!a->means3D || !a->opacities || !a->viewmatrix || !a->projmatrix || !a->cam_pos || !a->background)
      return reject(SFGS_E_BADARG, "null input");
    if (!a->shs && !a->colors_precomp) return reject(SFGS_E_BADARG, "need shs or colors_precomp");
    if (a->colors_precomp == nullptr && (a->M <= 0 || a->D < 0 || a->D > 3 || (a->D + 1) * (a->D + 1) > a->M))
      return reject(SFGS_E_BADARG, "SH degree/M mismatch");
    if (!a->cov3D_precomp && (!a->scales || !a->rotations))
      return reject(SFGS_E_BADARG, "need scales+rotations or cov3D_precomp");
    if (!a->norm3D_precomp && (!a->scales || !a->rotations))
      return reject(SFGS_E_BADARG, "need scales+rotations or norm3D_precomp");
    if (a->ED > 0 && (!a->extra_attrs || !a->out_extra)) return reject(SFGS_E_BADARG, "extra attrs missing");
    if (a->rotations && (reinterpret_cast<uintptr_t>(a->rotations) & 15))
      return reject(SFGS_E_BADARG, "rotations must be 16-byte aligned");
  }
  return SFGS_OK;
}

// graph: the pipeline is queued once at capacity_hint with no host wait, and a kernel ORs the header's error flags
// into *status
int rasterize_forward(const sfgs_forward_args* a, const FwdCall& c) {
  if (const int rc = check_forward(a, c)) return rc;
  const float* off = c.off;
  cudaStream_t st = (cudaStream_t)a->stream;
  const bool debug = a->debug != 0;
  const int P = a->P;

  const float focal_y = a->height / (2.0f * a->tan_fovy);
  const float focal_x = a->width / (2.0f * a->tan_fovx);

  const size_t gbytes = GeomLayout(nullptr, (size_t)P).bytes;
  char* gptr = a->geom_alloc(a->geom_user, gbytes);
  if (!gptr) return fail(SFGS_E_ALLOC, "forward: geometry allocator returned NULL");
  GeomLayout g(sfgs_align_ptr(gptr), (size_t)P);

  const size_t ibytes = ImageLayout(nullptr, a->width, a->height).bytes;
  char* iptr = a->image_alloc(a->image_user, ibytes);
  if (!iptr) return fail(SFGS_E_ALLOC, "forward: image allocator returned NULL");
  ImageLayout im(sfgs_align_ptr(iptr), a->width, a->height);

  // The whole pipeline for one binning capacity.  `after_scan` runs right after the tile scan, when num_rendered and
  // the error flags are final: the eager forward starts the header's copy to the host there, the graph forward
  // launches its status kernel.
  auto queue = [&](long long capacity, auto&& after_scan) -> int {
    const size_t bbytes = BinningLayout(nullptr, (size_t)capacity).bytes;
    char* bptr = a->binning_alloc(a->binning_user, bbytes);
    if (!bptr) return fail(SFGS_E_ALLOC, "forward: binning allocator returned NULL");
    BinningLayout b(sfgs_align_ptr(bptr), (size_t)capacity);

    // tile histogram + header start at zero
    PROF_BEGIN(ST_FWD_ZERO);
    CU(cudaMemsetAsync(im.hdr, 0, im.zero_bytes, st));   // header + tile histogram are adjacent
    if (off) sfgs_launch_offset_bound(im, a->width, a->height, off, st);   // the masks' dilation, before the key scatter
    PROF_END();

    if (P > 0) {
      PROF_BEGIN(ST_PREPROCESS);
      sfgs_launch_preprocess(a, g, im, b, (unsigned long long)capacity, focal_x, focal_y, c.tan_fov, c.ortho,
                             c.ray_depth, c.plane_normals, st);
      PROF_END();
      STAGE_CHECK("preprocess");
    }
    PROF_BEGIN(ST_SCAN);
    sfgs_launch_tile_scan(im, (unsigned long long)capacity, st);
    PROF_END();
    STAGE_CHECK("tile_scan");
    const int rc = after_scan();
    if (rc != SFGS_OK) return rc;
    if (P > 0) {
      PROF_BEGIN(ST_EMIT);
      sfgs_launch_scatter(g, im, b, a->P, (unsigned long long)capacity, off != nullptr, st);
      PROF_END();
      STAGE_CHECK("scatter_keys");
      PROF_BEGIN(ST_SORT);
      sfgs_launch_tile_sort(g, im, b, a->P, off != nullptr, st);
      PROF_END();
      STAGE_CHECK("tile_sort");
    }
    PROF_BEGIN(ST_RENDER_FWD);
    // t = 1 - q in float32: the transmittance the selected record crosses
    sfgs_launch_render_fwd(a, g, im, b, off, 1.0f - c.quantile, c.depth_q ? c.out_depth_q : nullptr, c.out_depth_q_pos,
                           c.dist ? c.out_distortion : nullptr, c.out_distortion_state, c.ray_depth, st);
    PROF_END();
    STAGE_CHECK("render_fwd");
    return SFGS_OK;
  };

  if (c.graph) {
    // captured: one pass at the caller's capacity; the overflow flag reaches the caller through *status, and every
    // kernel after the scan returns at once on it
    return queue(a->capacity_hint, [&]() -> int {
      sfgs_launch_forward_status(im, c.status, st);
      STAGE_CHECK("forward_status");
      return SFGS_OK;
    });
  }

  int dev = 0;
  CU(cudaGetDevice(&dev));
  if (dev < 0 || dev >= MAX_DEVICES) return fail(SFGS_E_UNSUPPORTED, "forward: device ordinal >= 64");
  const CapKey cap_key{dev, P, a->width, a->height, a->tile_row_begin, a->tile_row_end};
  long long capacity = a->capacity_hint;
  if (capacity <= 0) {
    const long long last = cap_lookup(cap_key);
    capacity = last >= 0 ? last + last / 4 + 4096 : (long long)P * 4 + 65536;
  }
  PinnedHdr& t_hdr = t_hdr_dev[dev];
  uint32_t* hhdr = t_hdr.get();
  if (!hhdr) return fail(SFGS_E_CUDA, "forward: pinned header allocation failed");

  long long R = 0;
  for (int attempt = 0; attempt < 3; attempt++) {
    // num_rendered and the overflow flag are final after the scan: start their copy now and let the host wait
    // on this event only, so it returns (and the caller can queue the backward) while sort + blend still run
    const int rc = queue(capacity, [&]() -> int {
      CU(cudaMemcpyAsync(hhdr, im.hdr, HDR_COPY_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      CU(cudaEventRecord(t_hdr.ev, st));
      return SFGS_OK;
    });
    if (rc != SFGS_OK) return rc;

    CU(cudaEventSynchronize(t_hdr.ev));
    if (debug) CU(cudaStreamSynchronize(st));
    R = (long long)hhdr[HDR_R];
    // the reference's checkFrustum traps the kernel when `prefiltered` is set and a point fails the test
    // (RAST/cuda_rasterizer/auxiliary.h:157-161); here the frame is reported as an argument error instead
    if (hhdr[HDR_PREFILTER]) return fail(SFGS_E_BADARG, "forward: prefiltered was set but a Gaussian failed the frustum test");
    if (hhdr[HDR_OFF_BAD]) return fail(SFGS_E_BADARG, "forward_subpixel: a subpixel offset is NaN or Inf");
    if (!hhdr[HDR_OVERFLOW]) break;
    if (attempt == 2) return fail(SFGS_E_CUDA, "forward: binning capacity overflow persisted");
    capacity = R + R / 16 + 4096;   // the exact count is now known; run the pipeline again with room for it
    g_overflow_reruns.fetch_add(1);
  }
  cap_store(cap_key, R);
  g_last_capacity.store(capacity);
  return (int)R;
}

// The backward's rejections of a per-pixel output's adjoint, in order: null inputs, ncam, extra_attrs, tile-row bands,
// acc_peers, phase 2, and camera gradients with phase 1 or the orthographic camera.
int check_pixel_output(const sfgs_backward_args* a, const BwdCall& c, bool null_in, const char* null_what,
                       const char* feature) {
  const auto reject = [&c](int code, const char* what) { return fail_in(c.name, code, what); };
  if (null_in) return reject(SFGS_E_BADARG, null_what);
  if (c.ncam != 0 && c.ncam != 35 && c.ncam != 37) return reject(SFGS_E_BADARG, "ncam must be 0, 35 or 37");
  if (a->ED > 0) return reject_with(c.name, "extra_attrs are", feature);
  if (a->tile_row_begin != 0 || a->tile_row_end != 0) return reject_with(c.name, "tile-row bands are", feature);
  if (a->acc_peers != nullptr) return reject_with(c.name, "acc_peers are", feature);
  if (a->phase == 2) return reject_with(c.name, "phase 2 is", feature);
  if (c.ncam > 0 && a->phase == 1)
    return reject(SFGS_E_UNSUPPORTED, "camera gradients are formed by the one-call backward (phase 0) only");
  if (c.ncam > 0 && c.ortho) return reject(SFGS_E_UNSUPPORTED, "the orthographic camera has no camera gradients");
  return SFGS_OK;
}

// Every rejection of the backward entries, in the order that decides which one an entry reports; all before any CUDA
// work.  Messages are "<entry>: <what>".  P == 0 passes once the checks that hold for it have run.
int check_backward(const sfgs_backward_args* a, const BwdCall& c) {
  const auto reject = [&c](int code, const char* what) { return fail_in(c.name, code, what); };
  if (!a) return reject(SFGS_E_BADARG, "null args");
  if (c.ray_depth) {
    const char* feature = c.plane_normals ? "plane normals" : "ray depth";
    if (const int rc = check_pixel_output(a, c, c.depth_q && (!c.depth_q_pos || !c.dL_dpix_depth_q),
                                          "null depth_q_pos or dL_dpix_depth_q", feature))
      return rc;
    if (c.plane_normals && a->norm3D_precomp != nullptr) return reject_with(c.name, "norm3D_precomp is", feature);
  }
  if (c.depth_q) {
    if (const int rc = check_pixel_output(a, c, !c.depth_q_pos || !c.dL_dpix_depth_q,
                                          "null depth_q_pos or dL_dpix_depth_q", "the depth quantile"))
      return rc;
  }
  if (c.dist) {
    if (const int rc = check_pixel_output(a, c, !c.distortion_state || !c.dL_dpix_distortion,
                                          "null distortion_state or dL_dpix_distortion", "the depth distortion"))
      return rc;
  }
  if (c.ortho) {
    if (a->phase != 0)
      return reject(SFGS_E_UNSUPPORTED, "phases 1 and 2 (the two-phase backward) are not supported with an orthographic camera");
    if (a->acc_peers != nullptr) return reject(SFGS_E_UNSUPPORTED, "acc_peers are not supported with an orthographic camera");
    if (a->tile_row_begin != 0 || a->tile_row_end != 0)
      return reject(SFGS_E_UNSUPPORTED, "tile-row bands are not supported with an orthographic camera");
    if (!ortho_extent_ok(a->tan_fovx, a->tan_fovy))
      return reject(SFGS_E_BADARG, "the half-extents tan_fovx, tan_fovy must be finite and > 0");
  }
  if (c.kind == BwdCall::CAMERA) {
    if (!c.dL_dcamera) return reject(SFGS_E_BADARG, "null dL_dcamera");
    if (a->phase != 0)
      return reject(SFGS_E_UNSUPPORTED, "camera gradients are formed by the one-call backward (phase 0) only");
    if (a->acc_peers != nullptr)
      return reject(SFGS_E_UNSUPPORTED, "acc_peers (the multi-GPU backward) have no camera gradients");
    if (!a->scratch_alloc) return reject(SFGS_E_BADARG, "null scratch allocator");
  } else if (c.kind == BwdCall::CAMERA_PARTIAL) {
    if (!c.dL_dcamera_partial) return reject(SFGS_E_BADARG, "null dL_dcamera_partial");
    if (c.ncam != 35 && c.ncam != 37) return reject(SFGS_E_BADARG, "ncam must be 35 or 37");
    if (a->phase != 2) return reject(SFGS_E_UNSUPPORTED, "camera partials are formed by phase 2 only");
    if (!a->scratch_alloc) return reject(SFGS_E_BADARG, "null scratch allocator");
    if (a->ED > 0) return reject(SFGS_E_UNSUPPORTED, "extra_attrs are not supported by the two-phase backward");
  } else if (c.kind == BwdCall::GRAPH) {
    if (a->debug) return reject(SFGS_E_BADARG, "debug synchronises after every stage and cannot be captured");
    if (a->R <= 0) return reject(SFGS_E_BADARG, "R must be the forward's binning capacity (> 0)");
    if (c.ncam != 0 && c.ncam != 35 && c.ncam != 37) return reject(SFGS_E_BADARG, "ncam must be 0, 35 or 37");
    if (c.ncam != 0 && !c.dL_dcamera) return reject(SFGS_E_BADARG, "null dL_dcamera");
    if (a->phase != 0)
      return reject(SFGS_E_UNSUPPORTED,
                    "phases 1 and 2 (the two-phase backward) are not supported under graph capture");
    if (a->acc_peers != nullptr) return reject(SFGS_E_UNSUPPORTED, "acc_peers are not supported under graph capture");
    if (a->tile_row_begin != 0 || a->tile_row_end != 0)
      return reject(SFGS_E_UNSUPPORTED, "tile-row bands are not supported under graph capture");
  }
  // extra_attrs have no kernels with offsets; the _subpixel entries have always rejected the fused peer exchange (the
  // partial entry rejects extra_attrs above, and acc_peers by their phase below)
  if (c.off != nullptr && c.kind != BwdCall::CAMERA_PARTIAL) {
    if (a->ED > 0) return reject(SFGS_E_UNSUPPORTED, "extra_attrs are not supported with subpixel offsets");
    if (!c.peers_with_off && a->acc_peers != nullptr)
      return reject(SFGS_E_UNSUPPORTED,
                    "acc_peers are not supported by this entry; use sfgs_rasterize_backward_subpixel_peers");
  }
  if (c.kind == BwdCall::GRAPH && c.ncam != 0 && !a->scratch_alloc)
    return reject(SFGS_E_BADARG, "null scratch allocator");
  if (a->P < 0 || a->width <= 0 || a->height <= 0) return reject(SFGS_E_BADARG, "bad sizes");
  if (c.deterministic && a->acc_peers != nullptr)
    return reject(SFGS_E_UNSUPPORTED, "acc_peers (system-scope reductions) have no deterministic implementation");
  if (c.deterministic && a->ED > 0)
    return reject(SFGS_E_UNSUPPORTED, "extra_attrs have no deterministic implementation");
  if (a->P == 0) return SFGS_OK;
  const int phase = a->phase;
  if (phase < 0 || phase > 2) return reject(SFGS_E_BADARG, "phase must be 0, 1 or 2");
  const bool do_blend = phase != 2, do_gauss = phase != 1;
  if (!a->geom_buffer || !a->binning_buffer || !a->image_buffer) return reject(SFGS_E_BADARG, "null scratch buffer");
  if (do_blend && (!a->dL_dpix || !a->dL_dpix_depth || !a->dL_dpix_norm || !a->dL_dpix_alpha || !a->accum_alphas))
    return reject(SFGS_E_BADARG, "null pixel gradient");
  if (do_gauss && (!a->dL_dmean2D || !a->dL_dconic || !a->dL_dopacity || !a->dL_dcolor || !a->dL_ddepth ||
                   !a->dL_dmean3D || !a->dL_dcov3D || !a->dL_dnorm3D || !a->dL_dscale || !a->dL_drot))
    return reject(SFGS_E_BADARG, "null output");
  if (do_gauss && !a->radii) return reject(SFGS_E_BADARG, "radii missing");
  if (do_gauss && a->M > 0 && a->shs && !a->dL_dsh) return reject(SFGS_E_BADARG, "dL_dsh missing");
  if (a->ED < 0 || a->ED > SFGS_MAX_EXTRA) return reject(SFGS_E_BADARG, "ED out of range");
  // extra-attribute gradients are accumulated by the blend stage only and are never exchanged between ranks: the
  // two-phase (multi-GPU) form would return them partial or uninitialised
  if (a->ED > 0 && phase != 0)
    return reject(SFGS_E_UNSUPPORTED, "extra_attrs are not supported by the two-phase backward");
  if (a->tile_row_begin < 0 || a->tile_row_end < a->tile_row_begin) return reject(SFGS_E_BADARG, "bad tile-row band");
  if (a->ED > 0 && (!a->dL_dextra || !a->dL_dpix_extra || !a->extra_attrs))
    return reject(SFGS_E_BADARG, "extra attrs missing");
  const bool peer = a->acc_peers != nullptr;
  if (peer && (phase != 1 || a->n_peers < 1 || a->n_peers > 8 || a->peer_slice < 1 ||
               (long long)a->n_peers * a->peer_slice < a->P))
    return reject(SFGS_E_BADARG, "acc_peers needs phase 1, 1..8 peers and n_peers*peer_slice >= P");
  if (phase != 0 && !a->acc && !peer) return reject(SFGS_E_BADARG, "phases 1 and 2 need the caller's acc buffer");
  if (phase == 0 && !a->acc && !a->scratch_alloc) return reject(SFGS_E_BADARG, "null scratch allocator");
  if (a->acc && (reinterpret_cast<uintptr_t>(a->acc) & 15)) return reject(SFGS_E_BADARG, "acc must be 16-byte aligned");
  if (a->rotations && (reinterpret_cast<uintptr_t>(a->rotations) & 15))
    return reject(SFGS_E_BADARG, "rotations must be 16-byte aligned");
  // the ordered blend adjoint places each partial by the Gaussian's tile rectangle (radii) in scratch_alloc's memory
  const bool ordered = c.deterministic && do_blend;
  if (ordered && !a->radii) return reject(SFGS_E_BADARG, "radii missing");
  if (ordered && !a->scratch_alloc) return reject(SFGS_E_BADARG, "null scratch allocator");
  if (phase == 2 && (a->gauss_begin < 0 || a->gauss_end > a->P || a->gauss_begin > a->gauss_end))
    return reject(SFGS_E_BADARG, "bad Gaussian range");
  return SFGS_OK;
}

// CAMERA, GRAPH with ncam > 0: the [ncam] camera gradients are formed as well; CAMERA_PARTIAL: phase 2 leaves the
// slice's [ncam] float64 camera sums unrounded.  GRAPH: a->R is the forward's binning capacity and only sizes scratch;
// the blend adjoint is always launched and it and the ordering kernels check the overflow flag first.
int rasterize_backward(const sfgs_backward_args* a, const BwdCall& c) {
  if (const int rc = check_backward(a, c)) return rc;
  const bool graph = c.kind == BwdCall::GRAPH;
  float* const dL_dcamera = c.dL_dcamera;
  double* const dL_dcamera_partial = c.dL_dcamera_partial;
  const int ncam = c.ncam;
  const float* const off = c.off;
  const bool cam = dL_dcamera != nullptr || dL_dcamera_partial != nullptr;
  if (a->P == 0) {
    if (dL_dcamera) CU(cudaMemsetAsync(dL_dcamera, 0, (size_t)ncam * sizeof(float), (cudaStream_t)a->stream));
    if (dL_dcamera_partial)
      CU(cudaMemsetAsync(dL_dcamera_partial, 0, (size_t)ncam * sizeof(double), (cudaStream_t)a->stream));
    return SFGS_OK;
  }
  const int phase = a->phase;
  const bool do_blend = phase != 2, do_gauss = phase != 1;
  const bool peer = a->acc_peers != nullptr;
  const bool ordered = c.deterministic && do_blend;
  cudaStream_t st = (cudaStream_t)a->stream;
  const bool debug = a->debug != 0;
  const int P = a->P;
  const int g_begin = phase == 2 ? a->gauss_begin : 0, g_end = phase == 2 ? a->gauss_end : P;

  GeomLayout g(sfgs_align_ptr(a->geom_buffer), (size_t)P);
  ImageLayout im(sfgs_align_ptr(a->image_buffer), a->width, a->height);
  // only point_list is needed; it sits at the head of the layout irrespective of the capacity
  BinningLayout b(sfgs_align_ptr(a->binning_buffer), (size_t)(a->R > 0 ? a->R : 0));

  const float focal_y = a->height / (2.0f * a->tan_fovy);
  const float focal_x = a->width / (2.0f * a->tan_fovx);

  float* acc = a->acc;
  const long long R = a->R > 0 ? a->R : 0;
  SfgsOrderScratch order = {};
  double* cam_part = nullptr;
  // one scratch_alloc call: the allocator may hand out the memory of an earlier call's buffer again
  if ((!acc && !peer) || ordered || cam) {
    const size_t acc_bytes = !acc ? sfgs_align_up((size_t)P * 16 * sizeof(float)) : 0;
    const size_t order_bytes = ordered ? sfgs_order_scratch_bytes(P, R) : 0;
    const size_t abytes = acc_bytes + order_bytes + (cam ? sfgs_camera_scratch_bytes(g_end - g_begin, ncam) : 0) + SFGS_ALIGN;
    char* aptr = a->scratch_alloc(a->scratch_user, abytes);
    if (!aptr) return fail(SFGS_E_ALLOC, "backward: scratch allocator returned NULL");
    char* base = sfgs_align_ptr(aptr);
    if (!acc) acc = (float*)base;
    if (ordered) order = sfgs_order_scratch(base + acc_bytes, P, R);
    if (cam) cam_part = (double*)(base + acc_bytes + order_bytes);
  }
  if (ordered) {
    // every row of acc the per-Gaussian adjoint reads (phase 0) or the caller sums across ranks (phase 1) is
    // written once by the reduction, so nothing is cleared but the written flags
    PROF_BEGIN(ST_BWD_ZERO);
    if (R > 0) CU(cudaMemsetAsync(order.written, 0, (size_t)R * BWD_BLOCKS, st));
    PROF_END();
    if (R > 0) {   // graph: R is the capacity (> 0), so the adjoint always runs
      PROF_BEGIN(ST_RENDER_BWD);
      sfgs_launch_render_bwd(a, g, im, b, acc, order.part, order.written, off, graph,
                             c.dist ? c.distortion_state : nullptr, c.dL_dpix_distortion, c.ray_depth, st);
      if (c.depth_q)
        sfgs_launch_depth_q_adjoint(a, g, im, b, c.depth_q_pos, c.dL_dpix_depth_q, acc, order.part, c.ray_depth, off,
                                    st);
      PROF_END();
      STAGE_CHECK("render_bwd");
    }
    const SfgsBand band = sfgs_band(a->tile_row_begin, a->tile_row_end, im.tiles_y);
    PROF_BEGIN(ST_BWD_ORDER);
    sfgs_launch_order_prepare(P, g, im, b, a->radii, band.b0, band.b1, order, graph, st);
    sfgs_launch_order_reduce(P, g, a->radii, phase == 1, order, acc, graph ? im.hdr : nullptr, st);
    PROF_END();
    STAGE_CHECK("bwd_order");
  } else if (do_blend) {
    // cleared right before the blend adjoint: the memset also makes the accumulator lines L2-resident for the
    // kernel's vector reductions (cleared earlier, those lines would have left L2 by the time the reductions arrive)
    PROF_BEGIN(ST_BWD_ZERO);
    // one call: only rows of rasterized Gaussians are ever accumulated into or read; two-phase: the caller sums
    // whole buffers across ranks, so every row must be defined
    if (peer) { /* the ranks clear their own slices and synchronise around this call */ }
    else if (phase == 0 && a->radii) sfgs_launch_acc_clear_visible(P, a->radii, acc, st);
    else CU(cudaMemsetAsync(acc, 0, (size_t)P * 16 * sizeof(float), st));
    if (a->ED > 0) CU(cudaMemsetAsync(a->dL_dextra, 0, (size_t)P * a->ED * sizeof(float), st));
    PROF_END();
    if (a->R > 0 || graph) {
      PROF_BEGIN(ST_RENDER_BWD);
      sfgs_launch_render_bwd(a, g, im, b, acc, nullptr, nullptr, off, graph, c.dist ? c.distortion_state : nullptr,
                             c.dL_dpix_distortion, c.ray_depth, st);
      if (c.depth_q)
        sfgs_launch_depth_q_adjoint(a, g, im, b, c.depth_q_pos, c.dL_dpix_depth_q, acc, nullptr, c.ray_depth, off, st);
      PROF_END();
      STAGE_CHECK("render_bwd");
    }
  }
  if (do_gauss) {
    PROF_BEGIN(ST_GAUSS_BWD);
    sfgs_launch_gauss_bwd(a, g, focal_x, focal_y, acc, g_begin, g_end, phase == 2 ? g_begin : 0, cam_part, ncam,
                          c.tan_fov, c.ortho, c.ray_depth, c.plane_normals, st);
    if (dL_dcamera) sfgs_launch_camera_reduce(P, ncam, cam_part, dL_dcamera, st);
    // an empty slice has no spans: the reduction writes zeros
    if (dL_dcamera_partial) sfgs_launch_camera_partial_reduce(g_end - g_begin, ncam, cam_part, dL_dcamera_partial, st);
    PROF_END();
    STAGE_CHECK("gauss_bwd");
  }
  return SFGS_OK;
}

}  // namespace

extern "C" {

int sfgs_activations_forward(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                             const double* filter_3D, float* opacity, float* scales, float* rotations, void* stream) {
  if (P < 0) return fail(SFGS_E_BADARG, "activations_forward: P < 0");
  if (P == 0) return SFGS_OK;
  if (!opacity_raw || !scaling_raw || !rotation_raw || !filter_3D || !opacity || !scales || !rotations)
    return fail(SFGS_E_BADARG, "activations_forward: null pointer");
  if (sfgs_launch_activations_fwd(P, opacity_raw, scaling_raw, rotation_raw, filter_3D, opacity, scales, rotations,
                                  (cudaStream_t)stream))
    return fail(SFGS_E_BADARG, "activations_forward: rotation buffers must be 16-byte aligned");
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SFGS_E_CUDA, "activations_forward", e);
  return SFGS_OK;
}

int sfgs_activations_backward(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                              const double* filter_3D, const float* g_opacity, const float* g_scales,
                              const float* g_rotations, float* g_opacity_raw, float* g_scaling_raw,
                              float* g_rotation_raw, void* stream) {
  if (P < 0) return fail(SFGS_E_BADARG, "activations_backward: P < 0");
  if (P == 0) return SFGS_OK;
  if (!opacity_raw || !scaling_raw || !rotation_raw || !filter_3D || !g_opacity || !g_scales || !g_rotations ||
      !g_opacity_raw || !g_scaling_raw || !g_rotation_raw)
    return fail(SFGS_E_BADARG, "activations_backward: null pointer");
  if (sfgs_launch_activations_bwd(P, opacity_raw, scaling_raw, rotation_raw, filter_3D, g_opacity, g_scales, g_rotations,
                                  g_opacity_raw, g_scaling_raw, g_rotation_raw, (cudaStream_t)stream))
    return fail(SFGS_E_BADARG, "activations_backward: rotation buffers must be 16-byte aligned");
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SFGS_E_CUDA, "activations_backward", e);
  return SFGS_OK;
}

int sfgs_selftest_expf(int n, const float* x, float* y_replica, float* y_expf, void* stream) {
  if (n < 0 || (n > 0 && (!x || !y_replica || !y_expf))) return fail(SFGS_E_BADARG, "selftest_expf: bad arguments");
  if (n == 0) return SFGS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  expf_selftest_kernel<<<592, 256, 0, st>>>(n, x, y_replica, y_expf);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? SFGS_OK : fail(SFGS_E_CUDA, "selftest_expf", e);
}

int sfgs_sm_clock_probe(float* out_mhz_device, void* stream) {
  if (!out_mhz_device) return fail(SFGS_E_BADARG, "sm_clock_probe: null");
  sm_clock_probe_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(out_mhz_device);
  return cudaGetLastError() == cudaSuccess ? SFGS_OK : SFGS_E_CUDA;
}

size_t sfgs_sizeof(int which) {
  switch (which) {
    case 0: return sizeof(sfgs_forward_args);
    case 1: return sizeof(sfgs_backward_args);
    case 2: return sizeof(sfgs_geom_view);
    case 3: return sizeof(sfgs_image_view);
    case 4: return sizeof(sfgs_binning_view);
    default: return 0;
  }
}

int sfgs_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.collect();
  g_prof.on = on != 0;
  if (on) for (int i = 0; i < ST_COUNT; i++) { g_prof.ms[i] = 0; g_prof.n[i] = 0; }
  return SFGS_OK;
}

int sfgs_profile_read(double* ms_total, long long* launches, int n) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.collect();
  for (int i = 0; i < n && i < ST_COUNT; i++) { if (ms_total) ms_total[i] = g_prof.ms[i]; if (launches) launches[i] = g_prof.n[i]; }
  return ST_COUNT;
}

int sfgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                      unsigned char* present, void* stream) {
  (void)projmatrix;   // the reference's test only uses the view depth (auxiliary.h:155)
  if (P < 0) return fail(SFGS_E_BADARG, "mark_visible: P < 0");
  if (P == 0) return SFGS_OK;
  if (!means3D || !viewmatrix || !present) return fail(SFGS_E_BADARG, "mark_visible: null");
  sfgs_launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SFGS_E_CUDA, "mark_visible", e);
  return SFGS_OK;
}

}  // extern "C"
