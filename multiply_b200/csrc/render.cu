// Engine dispatch and the fused eval-mode forward.
//   reference: /root/reference/code/lib/model/multiply.py:174-598 (Multiply.forward, eval branch,
//   using_nerfacc=True): per person  sample -> deform -> SDF -> normals/colour, then the
//   multi-person composite, the background, and the final blend.
#include "common.cuh"
#include <mutex>

namespace mp {

std::atomic<int> g_engine{1};

size_t field_ws_bytes(int N) {
  size_t a = simt_workspace_bytes(N), b = tc_workspace_bytes(N);
  return a > b ? a : b;
}

int field_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (c.cap <= 0) return 0;
  return g_engine == 1 ? tc_run(f, c, ws, ws_bytes, st) : simt_run(f, c, ws, ws_bytes, st);
}

__global__ void gather_rays_kernel(const float* __restrict__ dirs, const float* __restrict__ cam,
                                   const int64_t* __restrict__ idx, int n, const int* __restrict__ n_dev,
                                   float* __restrict__ d_out, float* __restrict__ c_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, *n_dev);
  if (i >= n) return;
  int64_t r = idx[i];
  for (int k = 0; k < 3; ++k) {
    d_out[3 * i + k] = dirs[3 * r + k];
    c_out[3 * i + k] = cam[3 * r + k];
  }
}
__global__ void force_outlier_sdf_kernel(const uint8_t* __restrict__ outl, int n, float* __restrict__ sdf) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && outl[i]) sdf[i] = 4.0f;     // multiply.py:142-143
}
// lattice points of lib/utils/mesh.py:generate_mesh (:88-93), see lattice_coord; point i = (ix * (res+1) + iy) *
// (res+1) + iz
__global__ void grid_points_kernel(float cx, float cy, float cz, float extent, float pad, int res, long long start,
                                   int count, float* __restrict__ pts) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  long long i = start + t;
  const int n1 = res + 1;
  int iz = (int)(i % n1), iy = (int)((i / n1) % n1), ix = (int)(i / ((long long)n1 * n1));
  const float c[3] = {cx, cy, cz};
  const int id[3] = {ix, iy, iz};
  for (int k = 0; k < 3; ++k) pts[3 * (size_t)t + k] = lattice_coord(id[k], res, pad, extent, c[k]);
}

__global__ void iota_kernel(int* p, int n, int* count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
  if (i == 0 && count) *count = n;
}

// Outlier samples may be skipped in the colour pass only if their compositing weight is exactly
// zero: sigma(4; beta) == 0 in fp32, i.e. expm1(-4/beta) == -1 (density.py:24) — true for
// beta < 0.23.  (The SDF clamp itself, multiply.py:142-143, is always exact.)
static bool prune_is_exact(float beta) { return (4.0f / beta) > 18.0f; }

// The persons of a scene and the background are independent until the compositor (multiply.py:266-410 is a Python
// loop over persons; :514-539 only needs the rays).  Each branch runs on its own stream so that the small
// latency-bound kernels of one (deformer, sampler trips) fill the SMs under the persistent MLP kernel of another,
// which issues on a third of the cycles.  mp_set_streams(0) restores the single-stream schedule.
// One set per device, created on first use on that device.  The enqueue section of mp_render_rays (fork ... join)
// holds the set's mutex, so two host threads rendering on the same device serialise their ENQUEUES (the device
// work still overlaps as far as the streams allow); sets of different devices are independent.
struct BranchStreams {
  bool ready = false;
  std::mutex mu;
  cudaStream_t s[MP_MAX_PERSONS + 1];
  cudaEvent_t fork, join[MP_MAX_PERSONS + 1];
  cudaEvent_t pre[MP_MAX_PERSONS];      // person p's chain up to (not including) its shade launch has been enqueued
};
constexpr int kMaxDevices = 64;
static BranchStreams g_bs[kMaxDevices];
static std::atomic<int> g_streams_on{-1};

static int branch_streams_init(BranchStreams& bs) {
  if (bs.ready) return 0;
  for (int i = 0; i <= MP_MAX_PERSONS; ++i) {
    MP_CHECK_CUDA(cudaStreamCreateWithFlags(&bs.s[i], cudaStreamNonBlocking));
    MP_CHECK_CUDA(cudaEventCreateWithFlags(&bs.join[i], cudaEventDisableTiming));
    if (i < MP_MAX_PERSONS) MP_CHECK_CUDA(cudaEventCreateWithFlags(&bs.pre[i], cudaEventDisableTiming));
  }
  MP_CHECK_CUDA(cudaEventCreateWithFlags(&bs.fork, cudaEventDisableTiming));
  bs.ready = true;
  return 0;
}

// rend_util.get_sphere_intersections calls exit() when a ray misses the bounding sphere (rend_util.py:140-142);
// here the condition is reported through mp_render_out_t.status (bit 0) for the caller to raise on.
__global__ void sphere_status_kernel(const float* __restrict__ dirs, const float* __restrict__ cam, int R, float r,
                                     int* __restrict__ status) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  const float* o = cam + 3 * i;
  const float* d = dirs + 3 * i;
  float dot = d[0] * o[0] + d[1] * o[1] + d[2] * o[2];
  float nrm = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
  float under = dot * dot - (nrm * nrm - r * r);
  if (!(under > 0.f)) atomicOr(status, 1);
}

struct PersonBufs {
  float *dirs, *cam, *z, *sdf, *rgb, *nrm, *xc_list, *jinv;
  int *slot_list, *count, *row_of_ray;
  uint8_t* outl;
  uint8_t *off, *in;     // per-row surface flags (training with a canonical mesh only)
};

struct RenderWs {
  float *dirs, *cam, *fg, *nrm, *acc, *accp, *bgT, *bg;
  PersonBufs pb[MP_MAX_PERSONS];
  // scratch of the sampler / MLP engine: one per concurrently running branch (persons, background)
  void* sub[MP_MAX_PERSONS + 1];
  size_t sub_bytes;
};

static void render_carve(Arena& a, const mp_scene_t& sc, int R, RenderWs& w) {
  const mp_sampler_cfg_t& c = sc.sampler;
  int n = samples_per_ray(c);
  w.dirs = a.take<float>((size_t)R * 3);
  w.cam = a.take<float>((size_t)R * 3);
  w.fg = a.take<float>((size_t)R * 3);
  w.nrm = a.take<float>((size_t)R * 3);
  w.acc = a.take<float>(R);
  w.accp = a.take<float>((size_t)R * sc.P);
  w.bgT = a.take<float>(R);
  w.bg = a.take<float>((size_t)R * 3);
  size_t sub = bg_ws_bytes(R);
  for (int p = 0; p < sc.P; ++p) {
    int Rp = sc.hit_count[p];
    PersonBufs& b = w.pb[p];
    b.dirs = a.take<float>((size_t)Rp * 3);
    b.cam = a.take<float>((size_t)Rp * 3);
    b.z = a.take<float>((size_t)Rp * (n + 1));
    b.sdf = a.take<float>((size_t)Rp * n);
    b.rgb = a.take<float>((size_t)Rp * n * 3);
    b.nrm = a.take<float>((size_t)Rp * n * 3);
    b.xc_list = a.take<float>((size_t)Rp * n * 3);
    b.jinv = a.take<float>((size_t)Rp * n * 12);
    b.slot_list = a.take<int>((size_t)Rp * n);
    b.count = a.take<int>(1);
    b.row_of_ray = a.take<int>(R);
    b.outl = a.take<uint8_t>((size_t)Rp * n);
    const bool flags = sc.train && sc.train->cano_mesh[p];
    b.off = flags ? a.take<uint8_t>(Rp) : nullptr;
    b.in = flags ? a.take<uint8_t>(Rp) : nullptr;
    sub = max(sub, sampler_ws_bytes(c, Rp));
    sub = max(sub, field_ws_bytes(Rp * n));
  }
  w.sub_bytes = sub;
  for (int i = 0; i <= sc.P; ++i) w.sub[i] = a.take<char>(sub);     // [P] = background branch
}

// the outliers of mp_deform_inverse, then the MLP's workspace
struct SdfDeformWs {
  uint8_t* outl;
  void* mlp;
  size_t mlp_bytes;
};
static void sdf_deform_carve(Arena& a, int N, SdfDeformWs& w) {
  w.outl = a.take<uint8_t>(N);
  w.mlp_bytes = field_ws_bytes(N);
  w.mlp = a.take<char>(w.mlp_bytes);
}

// the lattice is evaluated in slabs of at most 2^20 points
struct SdfGridWs {
  int chunk;
  float* pts;
  void* mlp;
  size_t mlp_bytes;
};
static void sdf_grid_carve(Arena& a, int res, SdfGridWs& w) {
  const long long n = (long long)(res + 1) * (res + 1) * (res + 1);
  w.chunk = (int)(n < (1 << 20) ? n : (1 << 20));
  w.pts = a.take<float>((size_t)w.chunk * 3);
  w.mlp_bytes = field_ws_bytes(w.chunk);
  w.mlp = a.take<char>(w.mlp_bytes);
}

}  // namespace mp

extern "C" {

int mp_set_engine(int engine) {
  MP_REQUIRE(engine == 0 || engine == 1, "mp_set_engine: engine must be 0 (simt fp32) or 1 (tensor cores)");
  mp::g_engine = engine;
  return 0;
}
int mp_get_engine(void) { return mp::g_engine; }

int mp_set_precision(int mode) {
  MP_REQUIRE(mode >= 0 && mode <= 2, "mp_set_precision: mode must be 0 (parity), 1 (single-term colour layers) or 2 (throughput)");
  mp::g_precision.store(mode);
  return 0;
}
int mp_get_precision(void) { return mp::g_precision.load(); }

int mp_profile_enable(int on) { return mp::prof_enable(on); }
int mp_set_streams(int on) {
  mp::g_streams_on.store(on ? 1 : 0);
  return 0;
}

int mp_profile_read(double* ms_host, long long* launches_host, double* points_host, int reset) {
  MP_REQUIRE(ms_host && launches_host && points_host, "mp_profile_read: null argument");
  return mp::prof_read(ms_host, launches_host, points_host, reset);
}

int mp_profile_read_stalls(unsigned long long* clocks_host, int reset) {
  MP_REQUIRE(clocks_host, "mp_profile_read_stalls: null argument");
  return mp::prof_read_stalls(clocks_host, reset);
}

size_t mp_mlp_workspace_bytes(int N) { return mp::field_ws_bytes(N); }

int mp_implicit_forward(mp_net_t* f, const float* x, int N, float* sdf, float* feat, void* workspace,
                        size_t workspace_bytes, void* stream) {
  MP_REQUIRE(f && x, "mp_implicit_forward: null argument");
  if (N <= 0) return 0;      // networks.py:131
  mp::MlpCall c{};
  c.x = x;
  c.cap = N;
  c.sdf = sdf;
  c.feat = feat;
  return mp::field_run(f->f, c, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mp_implicit_forward_grad(mp_net_t* f, const float* x, int N, float* sdf, float* feat, float* grad,
                             void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(f && x && grad, "mp_implicit_forward_grad: null argument");
  if (N <= 0) return 0;
  mp::MlpCall c{};
  c.x = x;
  c.cap = N;
  c.sdf = sdf;
  c.grad = grad;
  c.feat = feat;
  return mp::field_run(f->f, c, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mp_render_forward(mp_net_t* f, const float* points, const float* normals, const float* feat, int N, float* rgb,
                      void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(f && points && normals && feat && rgb, "mp_render_forward: null argument");
  if (N <= 0) return 0;
  // the standalone colour operator always runs on the fp32 SIMT kernels (the fused tensor-core chain
  // consumes features straight from shared memory and has no (points, normals, feat) entry)
  return mp::simt_render(f->f, points, normals, feat, N, rgb, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mp_bg_nets_forward(mp_net_t* bg_field, const float* pts, const float* view_dirs, int N, float* sdf, float* rgb,
                       void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(bg_field && pts && view_dirs && rgb, "mp_bg_nets_forward: null argument");
  MP_REQUIRE(bg_field->f.is_bg, "mp_bg_nets_forward: not a background field");
  if (N <= 0) return 0;
  mp::MlpCall c{};
  c.x = pts;
  c.cap = N;
  c.dirs = view_dirs;
  c.sdf = sdf;
  c.rgb = rgb;
  return mp::field_run(bg_field->f, c, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t mp_sdf_grid_workspace_bytes(int res) {
  if (res < 1 || res > 1024) return 0;
  mp::Arena a;
  mp::SdfGridWs w;
  mp::sdf_grid_carve(a, res, w);
  return a.off;
}

int mp_sdf_grid(mp_net_t* field, const float* center_host, float extent, float pad, int res, float* values,
                void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(field && center_host && values, "mp_sdf_grid: null argument");
  MP_REQUIRE(res >= 1 && res <= 1024, "mp_sdf_grid: res out of range");
  MP_REQUIRE(!field->f.is_bg, "mp_sdf_grid: a foreground field is required");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)(res + 1) * (res + 1) * (res + 1);
  mp::Arena a(workspace, workspace_bytes);
  mp::SdfGridWs w;
  mp::sdf_grid_carve(a, res, w);
  MP_TRY(a.fits("mp_sdf_grid"));
  const int chunk = w.chunk;
  for (long long s0 = 0; s0 < n; s0 += chunk) {
    const int cnt = (int)((n - s0) < chunk ? (n - s0) : chunk);
    mp::grid_points_kernel<<<mp::div_up(cnt, 256), 256, 0, st>>>(center_host[0], center_host[1], center_host[2], extent,
                                                                  pad, res, s0, cnt, w.pts);
    MP_LAUNCH_CHECK();
    mp::MlpCall c{};
    c.x = w.pts;
    c.cap = cnt;
    c.sdf = values + s0;
    MP_TRY(mp::field_run(field->f, c, w.mlp, w.mlp_bytes, st));
  }
  return 0;
}

size_t mp_sdf_with_deformer_workspace_bytes(int N) {
  mp::Arena a;
  mp::SdfDeformWs w;
  mp::sdf_deform_carve(a, N > 0 ? N : 0, w);
  return a.off;
}

int mp_sdf_with_deformer(mp_body_t* body, mp_net_t* field, const float* x, int N, float* sdf, float* x_c,
                         float* feat, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(body && field && x && sdf && x_c, "mp_sdf_with_deformer: null argument");
  if (N <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  mp::Arena a(workspace, workspace_bytes);
  mp::SdfDeformWs w;
  mp::sdf_deform_carve(a, N, w);
  MP_TRY(a.fits("mp_sdf_with_deformer"));
  MP_TRY(mp_deform_inverse(body, x, N, x_c, w.outl, 1, stream));
  mp::MlpCall c{};
  c.x = x_c;
  c.cap = N;
  c.sdf = sdf;
  c.feat = feat;
  MP_TRY(mp::field_run(field->f, c, w.mlp, w.mlp_bytes, st));
  mp::force_outlier_sdf_kernel<<<mp::div_up(N, 256), 256, 0, st>>>(w.outl, N, sdf);
  MP_LAUNCH_CHECK();
  return 0;
}

size_t mp_render_workspace_bytes(const mp_scene_t* scene, int R) {
  if (!scene || scene->P < 1 || scene->P > MP_MAX_PERSONS) return 0;
  mp::Arena a;
  mp::RenderWs w;
  mp::render_carve(a, *scene, R, w);
  return a.off;
}

namespace mp {

// One person's branch of Multiply.forward (multiply.py:266-410): gather its rays, sample, deform, SDF, normals, colour.
static int render_person(const mp_scene_t* scene, int p, int R, const RenderWs& w, int prune, const mp_render_out_t* out,
                         CompositePersons& cp, cudaStream_t st, cudaEvent_t pre_shade) {
  const mp_sampler_cfg_t& c = scene->sampler;
  const int n = samples_per_ray(c);
  MP_REQUIRE(scene->body[p] && scene->field[p] && scene->hit_index[p] && scene->hit_count[p] >= 1,
             "mp_render_rays: person %d incomplete", p);
  const Body& body = scene->body[p]->b;
  const Field& field = scene->field[p]->f;
  MP_REQUIRE(body.tfs, "mp_render_rays: body %d has no pose", p);
  const int Rp = scene->hit_count[p];                 // rows (capacity when the count lives on the device)
  const int* Rp_dev = scene->hit_count_dev[p];
  const PersonBufs& b = w.pb[p];
  gather_rays_kernel<<<div_up(Rp, 256), 256, 0, st>>>(w.dirs, w.cam, scene->hit_index[p], Rp, Rp_dev, b.dirs, b.cam);
  MP_LAUNCH_CHECK();
  // ray_sampler.get_z_vals (multiply.py:285-289); training mode (scene->train): stochastic, no outlier clamp anywhere
  const mp_train_t* tr = scene->train;
  MP_REQUIRE(!tr || (tr->rng[p] && !Rp_dev), "mp_render_rays: training mode needs the random draws of person %d and "
                                              "host-side hit counts", p);
  if (tr) prune = 0;
  MP_TRY(sample_rays(c, body, field, b.dirs, b.cam, Rp, b.z, nullptr, out->trips ? out->trips + p : nullptr, w.sub[p],
                     w.sub_bytes, st, Rp_dev, tr ? tr->rng[p] : nullptr, tr ? tr->z_eik[p] : nullptr));
  // main pass (multiply.py:295-308, 403-404): deform, SDF, normals, colour
  MP_CHECK_CUDA(cudaMemsetAsync(b.count, 0, sizeof(int), st));
  MP_CHECK_CUDA(cudaMemsetAsync(b.rgb, 0, (size_t)Rp * n * 3 * sizeof(float), st));
  MP_CHECK_CUDA(cudaMemsetAsync(b.nrm, 0, (size_t)Rp * n * 3 * sizeof(float), st));
  MP_TRY(launch_deform_rays(body, b.dirs, b.cam, b.z, n + 1, nullptr, 0, n, Rp, prune, b.sdf, n, b.xc_list,
                            b.slot_list, b.count, b.outl, nullptr, st, Rp_dev));
  MP_TRY(launch_forward_jac(body, b.xc_list, Rp * n, b.count, nullptr, b.jinv, 12, st));
  if (pre_shade) MP_CHECK_CUDA(cudaEventRecord(pre_shade, st));
  MlpCall shade{};
  shade.x = b.xc_list;
  shade.slot = b.slot_list;
  shade.count = b.count;
  shade.cap = Rp * n;
  shade.jinv = b.jinv;
  shade.sdf = b.sdf;
  shade.rgb = b.rgb;
  shade.nrm = b.nrm;
  MP_TRY(field_run(field, shade, w.sub[p], w.sub_bytes, st));
  if (tr && tr->cano_mesh[p]) {     // check_off_in_surface_points_cano_mesh on the main pass's points (:313-316)
    MP_CHECK_CUDA(cudaMemsetAsync(b.off, 1, Rp, st));
    MP_CHECK_CUDA(cudaMemsetAsync(b.in, 0, Rp, st));
    MP_TRY(launch_surface_flags(mesh_of(tr->cano_mesh[p]), b.xc_list, b.slot_list, b.count, Rp * n, n,
                                tr->surface_threshold, b.off, b.in, st));
  }
  if (!prune && !tr) {     // (multiply.py:142-143 is eval-only)
    force_outlier_sdf_kernel<<<div_up(Rp * n, 256), 256, 0, st>>>(b.outl, Rp * n, b.sdf);
    MP_LAUNCH_CHECK();
  }
  MP_TRY(launch_row_of_ray(scene->hit_index[p], Rp, R, b.row_of_ray, st, Rp_dev));
  set_person(cp, p, mp_person_samples_t{Rp, scene->hit_index[p], b.z, b.sdf, b.rgb, b.nrm}, b.row_of_ray);
  auto tap = [&](float* dst, const float* src, size_t cnt) -> int {
    if (dst) MP_CHECK_CUDA(cudaMemcpyAsync(dst, src, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  MP_TRY(tap(out->z_vals[p], b.z, (size_t)Rp * (n + 1)));
  MP_TRY(tap(out->sdf[p], b.sdf, (size_t)Rp * n));
  MP_TRY(tap(out->rgb[p], b.rgb, (size_t)Rp * n * 3));
  MP_TRY(tap(out->normals[p], b.nrm, (size_t)Rp * n * 3));
  return 0;
}

}  // namespace mp

int mp_render_rays(const mp_scene_t* scene, const float* uv, const float* pose, const float* intrinsics, int R,
                   const mp_render_out_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(scene && uv && pose && intrinsics && out, "mp_render_rays: null argument");
  MP_REQUIRE(scene->P >= 1 && scene->P <= MP_MAX_PERSONS, "mp_render_rays: P out of range");
  MP_REQUIRE(R > 0, "mp_render_rays: R must be positive");
  MP_REQUIRE(out->rgb_values, "mp_render_rays: rgb_values output is required");
  const mp_train_t* tr = scene->train;
  int n_mesh = 0;
  for (int p = 0; tr && p < scene->P; ++p) n_mesh += tr->cano_mesh[p] ? 1 : 0;
  MP_REQUIRE(n_mesh == 0 || n_mesh == scene->P, "mp_render_rays: canonical meshes are set for %d of %d persons", n_mesh,
             scene->P);
  MP_REQUIRE(n_mesh == 0 || (tr->index_off_surface && tr->index_in_surface),
             "mp_render_rays: surface flags need index_off_surface and index_in_surface outputs");
  MP_REQUIRE(n_mesh == 0 || !isnan(tr->surface_threshold), "mp_render_rays: surface_threshold is NaN");
  const cudaStream_t caller = (cudaStream_t)stream;
  const mp_sampler_cfg_t& c = scene->sampler;
  const int n = samples_per_ray(c);
  const float beta = sampler_beta(c);
  const int prune = prune_is_exact(beta) ? 1 : 0;
  Arena a(workspace, workspace_bytes);
  RenderWs w;
  render_carve(a, *scene, R, w);
  MP_TRY(a.fits("mp_render_rays"));
  MP_TRY(mp_camera_rays(uv, pose, intrinsics, R, w.dirs, w.cam, stream));     // multiply.py:223-227
  if (out->status) {
    MP_CHECK_CUDA(cudaMemsetAsync(out->status, 0, sizeof(int), caller));
    sphere_status_kernel<<<div_up(R, 256), 256, 0, caller>>>(w.dirs, w.cam, R, c.scene_bounding_sphere, out->status);
    MP_LAUNCH_CHECK();
  }
  if (g_streams_on.load() < 0) {
    const char* e = getenv("MP_RENDER_STREAMS");
    g_streams_on.store(e ? (atoi(e) != 0) : 1);
  }
  const bool fork = g_streams_on.load() == 1;
  int dev = 0;
  MP_CHECK_CUDA(cudaGetDevice(&dev));
  MP_REQUIRE(dev >= 0 && dev < kMaxDevices, "mp_render_rays: device ordinal %d out of range", dev);
  BranchStreams& bs = g_bs[dev];
  std::unique_lock<std::mutex> lock(bs.mu, std::defer_lock);
  if (fork) {
    lock.lock();
    MP_TRY(branch_streams_init(bs));
    MP_CHECK_CUDA(cudaEventRecord(bs.fork, caller));
  }
  // From here on every error path must still join the branch streams back into the caller's stream: the caller
  // may release the workspace / outputs as soon as we return, and branch kernels may be writing them.
  int rc = 0;
  bool forked[MP_MAX_PERSONS + 1] = {false};
  // Schedule.  An MLP launch is one persistent CTA per SM that fills the SM's shared memory, so MLP launches of
  // different branches never co-reside: they run one after the other whatever the stream order, and while one is
  // resident the small kernels of the other branches (sampler, deformer) only get the scraps (one 128-thread block per
  // SM).  The persons' chains up to their shade launch are latency-bound sequences of such small kernels, and the first
  // shade launch cannot start before a chain is through.  The background's MLP launch is independent of everything and
  // ready at once: started first (round 1) it occupies the SMs exactly while the chains need them.  It is therefore
  // enqueued LAST and gated on the persons' pre-shade events: chains at full occupancy, then shade / shade / background
  // back to back: 4.20 -> 4.00 ms per benchmark step.  (Also measured: starting person p's chain only when person p-1's is
  // through, so that each chain has the GPU to itself -- 4.55 ms: a chain in the shadow of a shade launch crawls.)
  CompositePersons cp;
  cp.P = scene->P;
  int n_pre = 0;
  for (int p = 0; p < scene->P && rc == 0; ++p) {
    cudaStream_t sp = fork ? bs.s[p] : caller;
    if (fork) {
      forked[p] = true;
      if (cudaStreamWaitEvent(sp, bs.fork, 0) != cudaSuccess) {
        set_error("mp_render_rays: cudaStreamWaitEvent failed");
        rc = -2;
        break;
      }
    }
    rc = render_person(scene, p, R, w, prune, out, cp, sp, fork ? bs.pre[p] : nullptr);
    if (rc == 0 && fork) n_pre = p + 1;
  }
  const float* bg = nullptr;
  if (scene->bg_field && rc == 0) {       // multiply.py:514-541
    cudaStream_t sb = fork ? bs.s[scene->P] : caller;
    if (fork) {
      forked[scene->P] = true;
      if (cudaStreamWaitEvent(sb, bs.fork, 0) != cudaSuccess) rc = -2;
      for (int p = 0; p < n_pre && rc == 0; ++p)
        if (cudaStreamWaitEvent(sb, bs.pre[p], 0) != cudaSuccess) rc = -2;
    }
    if (rc == 0)
      rc = render_background(scene->bg_field->f, w.dirs, w.cam, R, c.scene_bounding_sphere, w.bg, w.sub[scene->P],
                             w.sub_bytes, sb, scene->train ? scene->train->t_rand_bg : nullptr, out->bg_sdf,
                             out->bg_rgb_samples);
    if (rc == 0 && out->bg_rgb &&
        cudaMemcpyAsync(out->bg_rgb, w.bg, (size_t)R * 3 * sizeof(float), cudaMemcpyDeviceToDevice, sb) != cudaSuccess) {
      set_error("mp_render_rays: bg_rgb tap copy failed");
      rc = -2;
    }
    bg = w.bg;
  }
  if (fork) {
    // join (also after an error: everything enqueued on a branch stream is ordered before the caller's next work)
    for (int i = 0; i <= scene->P; ++i) {
      if (!forked[i]) continue;
      if (cudaEventRecord(bs.join[i], bs.s[i]) != cudaSuccess || cudaStreamWaitEvent(caller, bs.join[i], 0) != cudaSuccess) {
        if (rc == 0) {
          set_error("mp_render_rays: joining branch stream %d failed", i);
          rc = -2;
        }
      }
    }
    lock.unlock();
  }
  if (rc != 0) return rc;
  float* normal = out->normal_values ? out->normal_values : w.nrm;
  float* acc = out->acc_map ? out->acc_map : w.acc;
  float* accp = out->acc_person_list ? out->acc_person_list : w.accp;
  float* bgT = out->bg_T ? out->bg_T : w.bgT;
  MP_TRY(launch_composite(cp, R, n, beta, w.fg, normal, acc, accp, bgT, caller));     // multiply.py:427-480
  MP_TRY(launch_final_compose(w.fg, bgT, bg, R, out->rgb_values, out->fg_rgb_values, caller));   // :544-545, :590
  if (n_mesh) {     // multiply.py:549-560
    MP_CHECK_CUDA(cudaMemsetAsync(tr->index_off_surface, 1, R, caller));
    MP_CHECK_CUDA(cudaMemsetAsync(tr->index_in_surface, 0, R, caller));
    for (int p = 0; p < scene->P; ++p)
      MP_TRY(launch_merge_flags(scene->hit_index[p], scene->hit_count[p], scene->hit_count_dev[p], w.pb[p].off,
                                w.pb[p].in, tr->index_off_surface, tr->index_in_surface, caller));
  }
  return 0;
}
}
