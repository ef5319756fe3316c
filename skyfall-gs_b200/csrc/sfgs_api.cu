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
#include <cstdio>
#include <cstring>
#include <atomic>
#include <mutex>
#include <vector>
#include "sfgs_common.cuh"

std::atomic<long long> g_sfgs_launches{0};

void sfgs_launch_preprocess(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, unsigned long long capacity, float focal_x, float focal_y,
                            cudaStream_t st);
void sfgs_launch_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present,
                              cudaStream_t st);
void sfgs_launch_tile_scan(const ImageLayout& im, unsigned long long capacity, cudaStream_t st);
void sfgs_launch_scatter(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P,
                         unsigned long long capacity, bool dilate, cudaStream_t st);
void sfgs_launch_tile_sort(const GeomLayout& g, const ImageLayout& im, const BinningLayout& b, int P, bool dilate,
                           cudaStream_t st);
void sfgs_launch_offset_bound(const ImageLayout& im, int W, int H, const float* off, cudaStream_t st);
void sfgs_launch_render_fwd(const sfgs_forward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, const float* off, cudaStream_t st);
void sfgs_launch_render_bwd(const sfgs_backward_args* a, const GeomLayout& g, const ImageLayout& im,
                            const BinningLayout& b, float* acc, float* part, unsigned char* written, const float* off,
                            cudaStream_t st);
size_t sfgs_order_scratch_bytes(int P, long long R);
SfgsOrderScratch sfgs_order_scratch(char* base, int P, long long R);
void sfgs_launch_order_prepare(int P, const GeomLayout& g, const ImageLayout& im, const BinningLayout& b,
                               const int* radii, int band0, int band1, const SfgsOrderScratch& o, cudaStream_t st);
void sfgs_launch_order_reduce(int P, const GeomLayout& g, const int* radii, bool all_rows, const SfgsOrderScratch& o,
                              float* acc, cudaStream_t st);
int sfgs_launch_activations_fwd(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                                const double* filter_3D, float* opacity, float* scales, float* rotations,
                                cudaStream_t st);
int sfgs_launch_activations_bwd(int P, const float* opacity_raw, const float* scaling_raw, const float* rotation_raw,
                                const double* filter_3D, const float* g_opacity, const float* g_scales,
                                const float* g_rotations, float* g_opacity_raw, float* g_scaling_raw,
                                float* g_rotation_raw, cudaStream_t st);
void sfgs_launch_gauss_bwd(const sfgs_backward_args* a, const GeomLayout& g, float focal_x, float focal_y,
                           const float* acc, int g_begin, int g_end, int acc_row0, double* cam_part, int ncam,
                           cudaStream_t st);
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

int rasterize_forward(const sfgs_forward_args* a, const float* off);
int rasterize_backward(const sfgs_backward_args* a, bool deterministic, const float* off, float* dL_dcamera,
                       double* dL_dcamera_partial, int ncam);

// the combinations the subpixel-offset entry points reject (checked before any CUDA work): extra_attrs, which have no
// kernels with offsets, and -- unless the entry is a _subpixel_peers one -- the fused peer exchanges, which the
// _subpixel entries have always rejected
int subpixel_unsupported_fwd(const sfgs_forward_args* a, bool peers_ok) {
  if (a->ED > 0) return fail(SFGS_E_UNSUPPORTED, "forward_subpixel: extra_attrs are not supported with subpixel offsets");
  if (!peers_ok && a->out_peers != nullptr)
    return fail(SFGS_E_UNSUPPORTED, "forward_subpixel: out_peers are not supported by this entry; use sfgs_rasterize_forward_subpixel_peers");
  return SFGS_OK;
}
int subpixel_unsupported_bwd(const sfgs_backward_args* a, bool peers_ok) {
  if (a->ED > 0) return fail(SFGS_E_UNSUPPORTED, "backward_subpixel: extra_attrs are not supported with subpixel offsets");
  if (!peers_ok && a->acc_peers != nullptr)
    return fail(SFGS_E_UNSUPPORTED, "backward_subpixel: acc_peers are not supported by this entry; use sfgs_rasterize_backward_subpixel_peers");
  return SFGS_OK;
}

// the camera entries: ncam = 35 (pose terms) or 37 (pose and focal terms); the checks come before any CUDA work
int backward_camera(const char* name, const sfgs_backward_args* a, const float* off, int deterministic,
                    float* dL_dcamera, int ncam) {
  auto reject = [name](int code, const char* what) {
    char m[160];
    snprintf(m, sizeof(m), "%s: %s", name, what);
    return fail(code, m);
  };
  if (!a) return reject(SFGS_E_BADARG, "null args");
  if (!dL_dcamera) return reject(SFGS_E_BADARG, "null dL_dcamera");
  if (a->phase != 0)
    return reject(SFGS_E_UNSUPPORTED, "camera gradients are formed by the one-call backward (phase 0) only");
  if (a->acc_peers != nullptr)
    return reject(SFGS_E_UNSUPPORTED, "acc_peers (the multi-GPU backward) have no camera gradients");
  if (!a->scratch_alloc) return reject(SFGS_E_BADARG, "null scratch allocator");
  if (off != nullptr && subpixel_unsupported_bwd(a, false)) return SFGS_E_UNSUPPORTED;
  return rasterize_backward(a, deterministic != 0, off, dL_dcamera, nullptr, ncam);
}

// the phase-2 camera partials of a Gaussian slice (the tile-row sharded backward); the checks come before any CUDA work
int backward_camera_partial(const sfgs_backward_args* a, const float* off, int deterministic, int ncam,
                            double* dL_dcamera_partial) {
  if (!a) return fail(SFGS_E_BADARG, "backward_camera_partial: null args");
  if (!dL_dcamera_partial) return fail(SFGS_E_BADARG, "backward_camera_partial: null dL_dcamera_partial");
  if (ncam != 35 && ncam != 37) return fail(SFGS_E_BADARG, "backward_camera_partial: ncam must be 35 or 37");
  if (a->phase != 2)
    return fail(SFGS_E_UNSUPPORTED, "backward_camera_partial: camera partials are formed by phase 2 only");
  if (!a->scratch_alloc) return fail(SFGS_E_BADARG, "backward_camera_partial: null scratch allocator");
  if (a->ED > 0)
    return fail(SFGS_E_UNSUPPORTED, "backward_camera_partial: extra_attrs are not supported by the two-phase backward");
  return rasterize_backward(a, deterministic != 0, off, nullptr, dL_dcamera_partial, ncam);
}

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

int sfgs_rasterize_forward(const sfgs_forward_args* a) { return rasterize_forward(a, nullptr); }
int sfgs_rasterize_backward(const sfgs_backward_args* a) { return rasterize_backward(a, false, nullptr, nullptr, nullptr, 0); }
int sfgs_rasterize_backward_deterministic(const sfgs_backward_args* a) { return rasterize_backward(a, true, nullptr, nullptr, nullptr, 0); }

int sfgs_rasterize_forward_subpixel(const sfgs_forward_args* a, const float* subpixel_offset) {
  if (!a) return fail(SFGS_E_BADARG, "forward: null args");
  if (subpixel_offset != nullptr && subpixel_unsupported_fwd(a, false)) return SFGS_E_UNSUPPORTED;
  return rasterize_forward(a, subpixel_offset);
}
int sfgs_rasterize_forward_subpixel_peers(const sfgs_forward_args* a, const float* subpixel_offset) {
  if (!a) return fail(SFGS_E_BADARG, "forward: null args");
  if (subpixel_offset != nullptr && subpixel_unsupported_fwd(a, true)) return SFGS_E_UNSUPPORTED;
  return rasterize_forward(a, subpixel_offset);
}
int sfgs_rasterize_backward_subpixel(const sfgs_backward_args* a, const float* subpixel_offset) {
  if (!a) return fail(SFGS_E_BADARG, "backward: null args");
  if (subpixel_offset != nullptr && subpixel_unsupported_bwd(a, false)) return SFGS_E_UNSUPPORTED;
  return rasterize_backward(a, false, subpixel_offset, nullptr, nullptr, 0);
}
int sfgs_rasterize_backward_subpixel_peers(const sfgs_backward_args* a, const float* subpixel_offset) {
  if (!a) return fail(SFGS_E_BADARG, "backward: null args");
  if (subpixel_offset != nullptr && subpixel_unsupported_bwd(a, true)) return SFGS_E_UNSUPPORTED;
  return rasterize_backward(a, false, subpixel_offset, nullptr, nullptr, 0);
}
int sfgs_rasterize_backward_deterministic_subpixel(const sfgs_backward_args* a, const float* subpixel_offset) {
  if (!a) return fail(SFGS_E_BADARG, "backward: null args");
  if (subpixel_offset != nullptr && subpixel_unsupported_bwd(a, false)) return SFGS_E_UNSUPPORTED;
  return rasterize_backward(a, true, subpixel_offset, nullptr, nullptr, 0);
}

int sfgs_rasterize_backward_camera(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                   float* dL_dcamera) {
  return backward_camera("backward_camera", a, subpixel_offset, deterministic, dL_dcamera, 35);
}

int sfgs_rasterize_backward_camera_intrinsics(const sfgs_backward_args* a, const float* subpixel_offset,
                                              int deterministic, float* dL_dcamera) {
  return backward_camera("backward_camera_intrinsics", a, subpixel_offset, deterministic, dL_dcamera, 37);
}

int sfgs_rasterize_backward_camera_partial(const sfgs_backward_args* a, const float* subpixel_offset, int deterministic,
                                           int ncam, double* dL_dcamera_partial) {
  return backward_camera_partial(a, subpixel_offset, deterministic, ncam, dL_dcamera_partial);
}

}  // extern "C"

namespace {

int rasterize_forward(const sfgs_forward_args* a, const float* off) {
  if (!a) return fail(SFGS_E_BADARG, "forward: null args");
  if (a->P < 0 || a->width <= 0 || a->height <= 0) return fail(SFGS_E_BADARG, "forward: bad sizes");
  if (a->ED < 0 || a->ED > SFGS_MAX_EXTRA) return fail(SFGS_E_BADARG, "forward: ED out of range");
  if (a->tile_row_begin < 0 || a->tile_row_end < a->tile_row_begin) return fail(SFGS_E_BADARG, "forward: bad tile-row band");
  const bool peer_out = a->out_peers != nullptr && a->n_out_peers > 0;
  if (peer_out && a->n_out_peers > 8) return fail(SFGS_E_BADARG, "forward: at most 8 out_peers");
  if ((!peer_out && (!a->out_color || !a->out_depth || !a->out_norm || !a->out_alpha)) || (a->P > 0 && !a->radii))
    return fail(SFGS_E_BADARG, "forward: null output");
  if (!a->geom_alloc || !a->binning_alloc || !a->image_alloc) return fail(SFGS_E_BADARG, "forward: null allocator");
  if (a->P > 0) {
    if (!a->means3D || !a->opacities || !a->viewmatrix || !a->projmatrix || !a->cam_pos || !a->background)
      return fail(SFGS_E_BADARG, "forward: null input");
    if (!a->shs && !a->colors_precomp) return fail(SFGS_E_BADARG, "forward: need shs or colors_precomp");
    if (a->colors_precomp == nullptr && (a->M <= 0 || a->D < 0 || a->D > 3 || (a->D + 1) * (a->D + 1) > a->M))
      return fail(SFGS_E_BADARG, "forward: SH degree/M mismatch");
    if (!a->cov3D_precomp && (!a->scales || !a->rotations)) return fail(SFGS_E_BADARG, "forward: need scales+rotations or cov3D_precomp");
    if (!a->norm3D_precomp && (!a->scales || !a->rotations)) return fail(SFGS_E_BADARG, "forward: need scales+rotations or norm3D_precomp");
    if (a->ED > 0 && (!a->extra_attrs || !a->out_extra)) return fail(SFGS_E_BADARG, "forward: extra attrs missing");
    if (a->rotations && (reinterpret_cast<uintptr_t>(a->rotations) & 15)) return fail(SFGS_E_BADARG, "forward: rotations must be 16-byte aligned");
  }
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
      sfgs_launch_preprocess(a, g, im, b, (unsigned long long)capacity, focal_x, focal_y, st);
      PROF_END();
      STAGE_CHECK("preprocess");
    }
    PROF_BEGIN(ST_SCAN);
    sfgs_launch_tile_scan(im, (unsigned long long)capacity, st);
    PROF_END();
    STAGE_CHECK("tile_scan");
    // num_rendered and the overflow flag are final after the scan: start their copy now and let the host wait
    // on this event only, so it returns (and the caller can queue the backward) while sort + blend still run
    CU(cudaMemcpyAsync(hhdr, im.hdr, HDR_COPY_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(t_hdr.ev, st));
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
    sfgs_launch_render_fwd(a, g, im, b, off, st);
    PROF_END();
    STAGE_CHECK("render_fwd");

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

// dL_dcamera: NULL, or (phase 0 only, checked by the caller) the DEVICE [ncam] camera gradients to form as well;
// dL_dcamera_partial: NULL, or (phase 2 only, checked by the caller) the DEVICE [ncam] float64 camera sums of the
// Gaussian slice, unrounded.  ncam = 35 (pose terms) or 37 (pose and focal terms)
int rasterize_backward(const sfgs_backward_args* a, bool deterministic, const float* off, float* dL_dcamera,
                       double* dL_dcamera_partial, int ncam) {
  if (!a) return fail(SFGS_E_BADARG, "backward: null args");
  if (a->P < 0 || a->width <= 0 || a->height <= 0) return fail(SFGS_E_BADARG, "backward: bad sizes");
  if (deterministic && a->acc_peers != nullptr)
    return fail(SFGS_E_UNSUPPORTED, "backward_deterministic: acc_peers (system-scope reductions) have no deterministic implementation");
  if (deterministic && a->ED > 0)
    return fail(SFGS_E_UNSUPPORTED, "backward_deterministic: extra_attrs have no deterministic implementation");
  const bool cam = dL_dcamera != nullptr || dL_dcamera_partial != nullptr;
  if (a->P == 0) {
    if (dL_dcamera) CU(cudaMemsetAsync(dL_dcamera, 0, (size_t)ncam * sizeof(float), (cudaStream_t)a->stream));
    if (dL_dcamera_partial)
      CU(cudaMemsetAsync(dL_dcamera_partial, 0, (size_t)ncam * sizeof(double), (cudaStream_t)a->stream));
    return SFGS_OK;
  }
  const int phase = a->phase;
  if (phase < 0 || phase > 2) return fail(SFGS_E_BADARG, "backward: phase must be 0, 1 or 2");
  const bool do_blend = phase != 2, do_gauss = phase != 1;
  if (!a->geom_buffer || !a->binning_buffer || !a->image_buffer) return fail(SFGS_E_BADARG, "backward: null scratch buffer");
  if (do_blend && (!a->dL_dpix || !a->dL_dpix_depth || !a->dL_dpix_norm || !a->dL_dpix_alpha || !a->accum_alphas))
    return fail(SFGS_E_BADARG, "backward: null pixel gradient");
  if (do_gauss && (!a->dL_dmean2D || !a->dL_dconic || !a->dL_dopacity || !a->dL_dcolor || !a->dL_ddepth || !a->dL_dmean3D ||
                   !a->dL_dcov3D || !a->dL_dnorm3D || !a->dL_dscale || !a->dL_drot))
    return fail(SFGS_E_BADARG, "backward: null output");
  if (do_gauss && !a->radii) return fail(SFGS_E_BADARG, "backward: radii missing");
  if (do_gauss && a->M > 0 && a->shs && !a->dL_dsh) return fail(SFGS_E_BADARG, "backward: dL_dsh missing");
  if (a->ED < 0 || a->ED > SFGS_MAX_EXTRA) return fail(SFGS_E_BADARG, "backward: ED out of range");
  // extra-attribute gradients are accumulated by the blend stage only and are never exchanged between ranks: the
  // two-phase (multi-GPU) form would return them partial or uninitialised
  if (a->ED > 0 && phase != 0) return fail(SFGS_E_UNSUPPORTED, "backward: extra_attrs are not supported by the two-phase backward");
  if (a->tile_row_begin < 0 || a->tile_row_end < a->tile_row_begin) return fail(SFGS_E_BADARG, "backward: bad tile-row band");
  if (a->ED > 0 && (!a->dL_dextra || !a->dL_dpix_extra || !a->extra_attrs)) return fail(SFGS_E_BADARG, "backward: extra attrs missing");
  const bool peer = a->acc_peers != nullptr;
  if (peer && (phase != 1 || a->n_peers < 1 || a->n_peers > 8 || a->peer_slice < 1 ||
               (long long)a->n_peers * a->peer_slice < a->P))
    return fail(SFGS_E_BADARG, "backward: acc_peers needs phase 1, 1..8 peers and n_peers*peer_slice >= P");
  if (phase != 0 && !a->acc && !peer) return fail(SFGS_E_BADARG, "backward: phases 1 and 2 need the caller's acc buffer");
  if (phase == 0 && !a->acc && !a->scratch_alloc) return fail(SFGS_E_BADARG, "backward: null scratch allocator");
  if (a->acc && (reinterpret_cast<uintptr_t>(a->acc) & 15)) return fail(SFGS_E_BADARG, "backward: acc must be 16-byte aligned");
  if (a->rotations && (reinterpret_cast<uintptr_t>(a->rotations) & 15)) return fail(SFGS_E_BADARG, "backward: rotations must be 16-byte aligned");
  // the ordered blend adjoint places each partial by the Gaussian's tile rectangle (radii) in scratch_alloc's memory
  const bool ordered = deterministic && do_blend;
  if (ordered && !a->radii) return fail(SFGS_E_BADARG, "backward_deterministic: radii missing");
  if (ordered && !a->scratch_alloc) return fail(SFGS_E_BADARG, "backward_deterministic: null scratch allocator");
  cudaStream_t st = (cudaStream_t)a->stream;
  const bool debug = a->debug != 0;
  const int P = a->P;
  int g_begin = 0, g_end = P;
  if (phase == 2) {
    g_begin = a->gauss_begin; g_end = a->gauss_end;
    if (g_begin < 0 || g_end > P || g_begin > g_end) return fail(SFGS_E_BADARG, "backward: bad Gaussian range");
  }

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
    if (R > 0) {
      PROF_BEGIN(ST_RENDER_BWD);
      sfgs_launch_render_bwd(a, g, im, b, acc, order.part, order.written, off, st);
      PROF_END();
      STAGE_CHECK("render_bwd");
    }
    const SfgsBand band = sfgs_band(a->tile_row_begin, a->tile_row_end, im.tiles_y);
    PROF_BEGIN(ST_BWD_ORDER);
    sfgs_launch_order_prepare(P, g, im, b, a->radii, band.b0, band.b1, order, st);
    sfgs_launch_order_reduce(P, g, a->radii, phase == 1, order, acc, st);
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
    if (a->R > 0) {
      PROF_BEGIN(ST_RENDER_BWD);
      sfgs_launch_render_bwd(a, g, im, b, acc, nullptr, nullptr, off, st);
      PROF_END();
      STAGE_CHECK("render_bwd");
    }
  }
  if (do_gauss) {
    PROF_BEGIN(ST_GAUSS_BWD);
    sfgs_launch_gauss_bwd(a, g, focal_x, focal_y, acc, g_begin, g_end, phase == 2 ? g_begin : 0, cam_part, ncam, st);
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
