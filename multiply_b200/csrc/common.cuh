// Shared declarations of the multiply_b200 CUDA library (sm_90a only).
#pragma once
#include <atomic>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include "../../include/multiply_b200.h"

namespace mp {

// ---- error handling (no exceptions across the ABI) ----------------------------------------
void set_error(const char* fmt, ...);
extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;

#define MP_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      mp::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,                \
                    cudaGetErrorString(_e));                                             \
      return -2;                                                                         \
    }                                                                                    \
  } while (0)

#define MP_REQUIRE(cond, ...)                                                            \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      mp::set_error(__VA_ARGS__);                                                        \
      return -1;                                                                         \
    }                                                                                    \
  } while (0)

#define MP_LAUNCH_CHECK()                                                                \
  do {                                                                                   \
    mp::g_launches++;                                                                    \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      mp::set_error("%s:%d kernel launch failed: %s", __FILE__, __LINE__,                \
                    cudaGetErrorString(_e));                                             \
      return -3;                                                                         \
    }                                                                                    \
  } while (0)

#define MP_TRY(expr)                                                                     \
  do {                                                                                   \
    int _r = (expr);                                                                     \
    if (_r != 0) return _r;                                                              \
  } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace or storage.  Each call's buffers come from one carve function: the
// call's size query runs it on a sizing Arena (no base) and returns `off`, and the call runs it on the caller's buffer
// and refuses that buffer through fits() before it enqueues anything.  A base is 256-byte aligned (as cudaMalloc and
// torch allocations are), so every take is.
struct Arena {
  char* base;
  size_t cap;
  size_t off;
  bool ok;
  Arena() : Arena(nullptr, 0) {}
  Arena(void* p, size_t n) : base((char*)p), cap(n), off(0), ok(true) {}
  // A zero-element take always fits and moves nothing, so a layout's size is where its last non-empty take ends and a
  // call whose layout is empty accepts a null base.
  template <typename T>
  T* take(size_t n) {
    size_t bytes = n * sizeof(T);
    if (bytes == 0) return base ? (T*)(base + off) : nullptr;
    off = align_up(off, 256);
    if (base == nullptr || off + bytes > cap) {
      ok = false;
      off += bytes;
      return nullptr;
    }
    T* r = (T*)(base + off);
    off += bytes;
    return r;
  }
  // 0 when the carve fitted an aligned base; else -1 with "<who>: <what> too small (<off> needed, <cap> given)"
  int fits(const char* who, const char* what = "workspace") const;
};

int sm_count();

// ---- device structures --------------------------------------------------------------------

// uniform vertex grid for exact nearest-vertex queries (deform.cu)
struct GridHeader {
  float lo[3];
  float inv_h;
  float h;
  int dim[3];
  int ncell;
  int R0;        // search radius in cells that covers the query radius the grid was built for (h * R0 >= radius)
};
constexpr int kMaxCells = 32768;

struct Body {
  int V;
  const float* weights;      // [V,24]
  const float* verts_cano;   // [V,3]
  const float* verts_posed;  // [V,3] (caller memory, valid for the frame)
  const float* tfs;          // [24,4,4]
  float cano_cell;
  // grids (device, inside the body's storage)
  GridHeader* cano_hdr;
  int* cano_cell_start;      // [kMaxCells+1]
  float4* cano_sorted;       // [V]
  GridHeader* posed_hdr;
  int* posed_cell_start;
  float4* posed_sorted;
  int* scratch;              // [kMaxCells + 8]
  float4* vert_tf;           // [V][3] per-vertex inverse blended transform: rows (I_r0, I_r1, I_r2, c_r), x_c = I (x - c)
  // optional root finder (mp_body_set_root_finder): 0 steps = the reference's closed-form inverse only
  int root_steps;
  float root_thr;
};

// packed network (mlp_pack.cu)
constexpr int kHidden = 256;
struct TcBlob;
struct Field {
  int is_bg;
  int d_in, multires, emb_dim, cond_dim, skip_layer, n_imp;   // implicit
  int imp_in[MP_MAX_LAYERS], imp_out[MP_MAX_LAYERS];
  int n_ren, ren_mode, multires_view;
  int ren_in[MP_MAX_LAYERS], ren_out[MP_MAX_LAYERS];
  int ren_extra;          // leading inputs of colour layer 0 handled outside the 256-wide feature block
  // fp32 SIMT layout: Wt[l] is [in][out] (transposed), folded weight norm / skip scale
  float* imp_W[MP_MAX_LAYERS];      // natural [out][in] (backward pass, tensor-core packing)
  float* ren_W[MP_MAX_LAYERS];
  float* imp_Wt[MP_MAX_LAYERS];
  float* imp_b[MP_MAX_LAYERS];     // layer 0: raw bias; imp_b0_eff has the cond folded in
  float* imp_W0cond;               // [cond_dim][out0] transposed cond columns of layer 0
  float* imp_b0_eff;               // [out0]
  float* ren_Wt[MP_MAX_LAYERS];
  float* ren_b[MP_MAX_LAYERS];
  float* ren_b0_eff;               // [out0] (lin_pose(cond) / frame code folded)
  float* ren_W0cond;               // [cdim][out0] : (W0[:, 6:14] @ lin_pose.W) for mode 0 ([69][out0]); W0[:,27:59]^T for mode 1 ([32][out0])
  float* ren_b0_base;              // [out0] : b0 + W0[:,6:14] @ lin_pose.b  (mode 0) ; b0 (mode 1)
  int ren_cond_dim;
  float* ren_cb;                   // [out0] Wc0[:, feat] . b8[1:]  (colour layer 0 folded onto the feature layer)
  float* ren_b0_fold;              // [out0] ren_b0_eff + ren_cb : bias of the folded layer (tensor-core chains)
  bool tc_full;                    // the tensor-core engine has a full program: the fused shade chain (foreground) or the
                                   // background chain
  TcBlob* tc;                      // tensor-core programs (mlp_tc.cu); null until packed
};

// launch helpers
static inline int div_up(int a, int b) { return (a + b - 1) / b; }
static inline int clamp_wpc(size_t v) { return v < 1 ? 1 : (v > 8 ? 8 : (int)v); }

// The sampler's beta (density.py:27-29; one fp32 add, the same with or without -fmad=false) and samples per ray
// (multiply.py:290-292).
static inline float sampler_beta(const mp_sampler_cfg_t& c) { return fabsf(c.beta_param) + c.beta_min; }
static inline int samples_per_ray(const mp_sampler_cfg_t& c) { return c.N_samples + c.N_samples_extra + 1; }

// ---- cross-file launchers: every internal function or type one .cu file uses from another --------

// One evaluation of a field's networks over a list of points, the same for both MLP engines.  Outputs left null are
// not written.  sdf, rgb and nrm go to each point's slot (dense when `slot` is null); grad and feat are always dense.
struct MlpCall {
  const float* x;       // [cap, d_in] points (canonical space; background: [cap, 4])
  const int* slot;      // [cap] output slot of each point, or nullptr (slot = index)
  const int* count;     // device count of valid points, or nullptr (= cap)
  int cap;
  const float* jinv;    // [cap, 12] inverse deformation Jacobians (3x3 row-major, padded to 12): normals and rgb
  const float* dirs;    // [cap, 3] view directions: the background networks
  float* sdf;           // [slots]
  float* rgb;           // [slots, 3]
  float* nrm;           // [slots, 3]
  float* grad;          // [cap, 3] d sdf / d x
  float* feat;          // [cap, 256] ImplicitNet features
};
// Which chain a call runs; the values are also the profile kinds of mp_profile_read.
enum class MlpProg { kSdf = 0, kForward = 1, kFull = 2, kBg = 3 };
static inline MlpProg mlp_prog(const MlpCall& c) {
  if (c.dirs) return MlpProg::kBg;                       // background: sdf + rgb
  if (c.jinv || c.grad) return MlpProg::kFull;           // forward + reverse sweep (+ colour with jinv); a feat request
                                                         // costs the tensor-core engine one more forward launch
  if (c.feat) return MlpProg::kForward;                  // sdf + features
  return MlpProg::kSdf;
}

// fp32 SIMT engine (mlp_simt.cu)
size_t simt_workspace_bytes(int N);
int simt_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st);
int simt_render(const Field& f, const float* pts, const float* nrm, const float* feat, int N, float* rgb, void* ws,
                size_t ws_bytes, cudaStream_t st);

// tensor-core engine (mlp_tc.cu)
size_t tc_workspace_bytes(int N);
int tc_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st);
TcBlob* tc_new();
void tc_free(TcBlob* tb);
void tc_pack_carve(Arena& a, Field& f);
int tc_pack(const Field& f, cudaStream_t st);
int prof_enable(int on);
int prof_read(double* ms, long long* launches, double* points, int reset);
int prof_read_stalls(unsigned long long* clocks, int reset);
extern std::atomic<int> g_precision;

// engine dispatch (render.cu): g_engine 1 = tensor cores, 0 = SIMT; field_ws_bytes covers either engine
extern std::atomic<int> g_engine;
size_t field_ws_bytes(int N);
int field_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st);

// deformer (deform.cu)
int launch_deform_rays(const Body& b, const float* dirs, const float* cam, const float* z, int z_stride,
                       const int* zpos, int zpos_stride, int n_per_ray, int R, int prune, float* sdf_out,
                       int sdf_stride, float* xc_list, int* slot_list, int* count, uint8_t* outlier_out,
                       const int* active, cudaStream_t st, const int* R_dev = nullptr);
int launch_forward_jac(const Body& b, const float* x_c, int N, const int* n_dev, float* x_d, float* Jinv,
                       int jstride, cudaStream_t st);

// error-bound ray sampler (sampler.cu)
int sample_rays(const mp_sampler_cfg_t& c, const Body& body, const Field& field, const float* dirs,
                const float* cam, int R, float* z_final, float* z_bg, int* trips_out, void* ws, size_t ws_bytes,
                cudaStream_t st, const int* R_dev = nullptr, const mp_sampler_rng_t* rng = nullptr,
                float* z_eik = nullptr);
size_t sampler_ws_bytes(const mp_sampler_cfg_t& c, int R);

// multi-person compositor (composite.cu)
struct CompositePersons {
  int P;
  int n_rows[MP_MAX_PERSONS];
  const int* row_of_ray[MP_MAX_PERSONS];   // [R] -> row in the person's hit list or -1
  const float* z[MP_MAX_PERSONS];          // [R_p, n+1]
  const float* sdf[MP_MAX_PERSONS];        // [R_p, n]
  const float* rgb[MP_MAX_PERSONS];        // [R_p, n, 3]
  const float* nrm[MP_MAX_PERSONS];        // [R_p, n, 3]
};
static inline void set_person(CompositePersons& cp, int p, const mp_person_samples_t& s, const int* row_of_ray) {
  cp.n_rows[p] = s.n_rows;
  cp.row_of_ray[p] = row_of_ray;
  cp.z[p] = s.z_vals;
  cp.sdf[p] = s.sdf;
  cp.rgb[p] = s.rgb;
  cp.nrm[p] = s.normal;
}
int launch_composite(const CompositePersons& cp, int R, int n, float beta, float* fg_rgb, float* normal, float* acc,
                     float* acc_person, float* bg_T, cudaStream_t st);
int launch_row_of_ray(const int64_t* idx, int n_rows, int R, int* row_of_ray, cudaStream_t st,
                      const int* n_dev = nullptr);
int launch_final_compose(const float* fg, const float* bgT, const float* bg, int R, float* rgb, float* fg_out,
                         cudaStream_t st);

// background (background.cu)
int render_background(const Field& f, const float* dirs, const float* cam, int R, float bound, float* bg_rgb,
                      void* ws, size_t ws_bytes, cudaStream_t st, const float* t_rand = nullptr,
                      float* tap_sdf = nullptr, float* tap_rgb = nullptr);
size_t bg_ws_bytes(int R);

// canonical meshes (mesh.cu)
struct Mesh;
const Mesh& mesh_of(const mp_mesh_t* h);
int launch_surface_flags(const Mesh& m, const float* xc, const int* slot, const int* count_dev, int cap, int n,
                         float thr, uint8_t* off, uint8_t* in, cudaStream_t st);
int launch_merge_flags(const int64_t* idx, int rows, const int* rows_dev, const uint8_t* off_p, const uint8_t* in_p,
                       uint8_t* off, uint8_t* in, cudaStream_t st);

}  // namespace mp

struct mp_body {
  mp::Body b;
};
struct mp_net {
  mp::Field f;
};

// ---- device helpers -------------------------------------------------------------------------
#ifdef __CUDACC__
namespace mp {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// inclusive warp scan
__device__ __forceinline__ float warp_scan_incl(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// exclusive warp scan (no "inclusive minus own" cancellation when one lane holds a huge term)
__device__ __forceinline__ float warp_scan_excl(float v, int lane) {
  float incl = warp_scan_incl(v, lane);
  float up = __shfl_up_sync(0xffffffffu, incl, 1);
  return lane == 0 ? 0.f : up;
}

// binary searches of v in the ascending a[0, n): upper_bound = #elements <= v, lower_bound = #elements < v
__device__ __forceinline__ int upper_bound(const float* a, int n, float v) {   // first i with a[i] > v
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] > v) hi = mid; else lo = mid + 1;
  }
  return lo;
}
__device__ __forceinline__ int lower_bound(const float* a, int n, float v) {   // first i with a[i] >= v
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] >= v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// One coordinate of a lattice point of lib/utils/mesh.py:generate_mesh (:92-95): ((idx / res - 0.5) * pad) * extent +
// centre, every step rounded to fp32 separately as numpy does.  mp_sdf_grid and mp_mise both place their points here.
__device__ __forceinline__ float lattice_coord(int idx, int res, float pad, float extent, float centre) {
  float v = __fdiv_rn((float)idx, (float)res);
  v = __fadd_rn(v, -0.5f);
  v = __fmul_rn(v, pad);
  v = __fmul_rn(v, extent);
  return __fadd_rn(v, centre);
}

// LaplaceDensity.density_func (lib/model/density.py:20-25):
//   alpha * (0.5 + 0.5 * sign(sdf) * expm1(-|sdf| / beta)),  alpha = 1 / beta
__device__ __forceinline__ float laplace_density(float sdf, float beta) {
  float alpha = __fdiv_rn(1.0f, beta);
  float sg = (sdf > 0.f) ? 1.f : ((sdf < 0.f) ? -1.f : 0.f);
  float e = expm1f(__fdiv_rn(-fabsf(sdf), beta));
  float t = __fmul_rn(__fmul_rn(0.5f, sg), e);
  return __fmul_rn(alpha, __fadd_rn(0.5f, t));
}

// torch.nn.Softplus(beta=100, threshold=20) (networks.py:85)
__device__ __forceinline__ float softplus100(float x) {
  float t = 100.f * x;
  if (t > 20.f) return x;
  return log1pf(expf(t)) / 100.f;
}
// d softplus100 / dx = sigmoid(100 x)  (1 above the threshold, as autograd does)
__device__ __forceinline__ float softplus100_grad(float x) {
  float t = 100.f * x;
  if (t > 20.f) return 1.f;
  float z = expf(t);
  return z / (z + 1.f);
}

}  // namespace mp
#endif
