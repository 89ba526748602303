// Hard depth maps of posed meshes and the K=1 nearest-vertex search, with their backward: the two pytorch3d operators
// of opt_depth's geometric losses.
//   reference: /root/reference/code/lib/model/render.py:135-157 (Renderer.render_multiple_depth_map: MeshRasterizer with
//   faces_per_pixel=10, blur_radius=0; opt_depth reads layer 0 of zbuf, multiply_model.py:396-401) and
//   multiply_model.py:521-551 (pytorch3d.ops.knn_points(K=1, return_nn=True) in get_interpenetration_loss).
//
// Depth map (the definition is oracle/raster.py's).  A vertex v maps to (X, Y, Z) = R v + T and to the image point
// (u, v) = (fx X / Z + cx, fy Y / Z + cy); pixel (r, c) samples (c + 0.5, r + 0.5).  A face with a vertex at Z <= 0 or
// of zero projected area is skipped.  It covers a sample when its three edge functions, signed by the area, are >= 0
// (closed triangle); its depth there is z = 1 / (b0 / Z0 + b1 / Z1 + b2 / Z2) with the screen barycentrics b_i, rounded
// to fp32 once.  zbuf is the smallest such depth (ties: lowest face index), -1 where no face covers the pixel.
//
// Arithmetic.  Everything per vertex and per sample is fp64 on the fp32 inputs, term by term in the order
// oracle/raster.py writes it, and the file is compiled with -fmad=false, so every decision (box, inside, nearest) is
// the oracle's bit for bit.  The nearest-face choice is an atomicMin on a 64-bit key per pixel, fp32 depth bits high
// (a positive float orders like its bits) and face index low: the result does not depend on the schedule.
//
// Sums (the backward): every contribution is an item (target vertex, fp64 3-vector); items are stably sorted by target
// and each target sums its items in item order (scatter_sum).  No float atomics: reruns are bit-identical.
#include "common.cuh"
#include <cub/cub.cuh>

namespace mp {

// ---- camera and faces ----------------------------------------------------------------------------------------------

struct Cam {
  double R[9], T[3], fx, fy, cx, cy;
};

static Cam cam_of(const mp_camera_t& c) {
  Cam k;
  for (int i = 0; i < 9; ++i) k.R[i] = c.R[i];
  for (int i = 0; i < 3; ++i) k.T[i] = c.T[i];
  k.fx = c.fx;
  k.fy = c.fy;
  k.cx = c.cx;
  k.cy = c.cy;
  return k;
}

// One face in view and screen space.  ok = false: skipped (an index outside [0, V), a vertex at Z <= 0, zero area or
// a box that misses the image).  The box [c0, c1] x [r0, r1] holds the pixels whose centres lie in the projected
// bounds, clipped to the image.
struct Tri {
  double X[3], Y[3], Z[3], u[3], v[3], A;
  int c0, c1, r0, r1;
  bool ok;
};

__device__ __forceinline__ Tri tri_setup(const Cam& k, const float* __restrict__ verts, int V,
                                         const int64_t* __restrict__ faces, int f, int H, int W) {
  Tri t;
  t.ok = false;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int64_t vi = faces[3 * (size_t)f + j];
    if (vi < 0 || vi >= V) return t;
    const double x = verts[3 * vi], y = verts[3 * vi + 1], z = verts[3 * vi + 2];
    t.X[j] = ((k.R[0] * x + k.R[1] * y) + k.R[2] * z) + k.T[0];
    t.Y[j] = ((k.R[3] * x + k.R[4] * y) + k.R[5] * z) + k.T[1];
    t.Z[j] = ((k.R[6] * x + k.R[7] * y) + k.R[8] * z) + k.T[2];
    if (!(t.Z[j] > 0.0)) return t;
    t.u[j] = (k.fx * t.X[j]) / t.Z[j] + k.cx;
    t.v[j] = (k.fy * t.Y[j]) / t.Z[j] + k.cy;
  }
  t.A = (t.u[1] - t.u[0]) * (t.v[2] - t.v[0]) - (t.v[1] - t.v[0]) * (t.u[2] - t.u[0]);
  if (!(fabs(t.A) > 0.0)) return t;
  const double ulo = fmin(fmin(t.u[0], t.u[1]), t.u[2]), uhi = fmax(fmax(t.u[0], t.u[1]), t.u[2]);
  const double vlo = fmin(fmin(t.v[0], t.v[1]), t.v[2]), vhi = fmax(fmax(t.v[0], t.v[1]), t.v[2]);
  const double c0 = fmax(ceil(ulo - 0.5), 0.0), c1 = fmin(floor(uhi - 0.5), (double)(W - 1));
  const double r0 = fmax(ceil(vlo - 0.5), 0.0), r1 = fmin(floor(vhi - 0.5), (double)(H - 1));
  if (!(c0 <= c1 && r0 <= r1)) return t;
  t.c0 = (int)c0;
  t.c1 = (int)c1;
  t.r0 = (int)r0;
  t.r1 = (int)r1;
  t.ok = true;
  return t;
}

// Edge function of vertex i (the edge j -> k opposite it) at the sample (px, py).
__device__ __forceinline__ double edge_fn(const Tri& t, int i, double px, double py) {
  const int j = i == 2 ? 0 : i + 1, k = i == 0 ? 2 : i - 1;
  return (t.u[j] - px) * (t.v[k] - py) - (t.v[j] - py) * (t.u[k] - px);
}

// The face's depth at pixel (r, c) as the 64-bit key, or false when the closed triangle does not hold the sample.
__device__ __forceinline__ bool tri_key(const Tri& t, int f, int r, int c, unsigned long long& key) {
  const double px = c + 0.5, py = r + 0.5;
  double e[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    e[i] = edge_fn(t, i, px, py);
    if (t.A > 0.0 ? e[i] < 0.0 : e[i] > 0.0) return false;
  }
  const double s = (e[0] / t.A / t.Z[0] + e[1] / t.A / t.Z[1]) + e[2] / t.A / t.Z[2];
  const float z = (float)(1.0 / s);
  key = ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)f;
  return true;
}

// ---- depth forward -------------------------------------------------------------------------------------------------

constexpr int kSmallBox = 256;      // a face whose box holds more pixels is rasterised by a whole CTA
constexpr int kBigThreads = 256;

__global__ void raster_faces_kernel(Cam k, const float* __restrict__ verts, int V, const int64_t* __restrict__ faces,
                                    int F, int H, int W, unsigned long long* __restrict__ keys, int* __restrict__ big,
                                    int* __restrict__ n_big) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const Tri t = tri_setup(k, verts, V, faces, f, H, W);
  if (!t.ok) return;
  if ((long long)(t.c1 - t.c0 + 1) * (t.r1 - t.r0 + 1) > kSmallBox) {
    big[atomicAdd(n_big, 1)] = f;
    return;
  }
  for (int r = t.r0; r <= t.r1; ++r)
    for (int c = t.c0; c <= t.c1; ++c) {
      unsigned long long key;
      if (tri_key(t, f, r, c, key)) atomicMin(&keys[(size_t)r * W + c], key);
    }
}

// the faces with large boxes: one CTA per face at a time, its threads striding over the box
__global__ void raster_big_kernel(Cam k, const float* __restrict__ verts, int V, const int64_t* __restrict__ faces,
                                  int H, int W, const int* __restrict__ big, const int* __restrict__ n_big,
                                  unsigned long long* __restrict__ keys) {
  const int n = *n_big;
  for (int e = blockIdx.x; e < n; e += gridDim.x) {
    const int f = big[e];
    const Tri t = tri_setup(k, verts, V, faces, f, H, W);
    const long long nc = t.c1 - t.c0 + 1, np = nc * (t.r1 - t.r0 + 1);
    for (long long q = threadIdx.x; q < np; q += blockDim.x) {
      const int r = t.r0 + (int)(q / nc), c = t.c0 + (int)(q % nc);
      unsigned long long key;
      if (tri_key(t, f, r, c, key)) atomicMin(&keys[(size_t)r * W + c], key);
    }
  }
}

__global__ void raster_decode_kernel(const unsigned long long* __restrict__ keys, int n, float* __restrict__ zbuf,
                                     int64_t* __restrict__ pix_to_face) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = keys[i];
  const bool hit = key != ~0ull;
  zbuf[i] = hit ? __uint_as_float((unsigned)(key >> 32)) : -1.f;
  pix_to_face[i] = hit ? (int64_t)(key & 0xffffffffull) : -1;
}

struct RasterWs {
  unsigned long long* keys;
  int* big;
  int* n_big;
};

static void raster_carve(Arena& a, int H, int W, int F, RasterWs& w) {
  w.keys = a.take<unsigned long long>((size_t)H * W);
  w.big = a.take<int>(F);
  w.n_big = a.take<int>(1);
}

// ---- deterministic scatter-sum -------------------------------------------------------------------------------------

// M items, item m adding val[m] (3 doubles) to target key[m] in [0, T); key[m] == T: no target.  out[t] (3 floats) =
// the sum of target t's items in item order, rounded once; every out element is written.
struct ScatterWs {
  int *key, *key_s, *item, *item_s;
  double* val;
  void* cub_tmp;
  size_t cub_bytes;
};

static int key_bits(int n) {     // bits that hold 0 .. n-1
  int b = 1;
  while (b < 31 && (1 << b) < n) ++b;
  return b;
}

static size_t scatter_cub_bytes(int M, int T) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr, M,
                                  0, key_bits(T + 1));
  return b;
}

static void scatter_carve(Arena& a, int M, int T, ScatterWs& w) {
  w.key = a.take<int>(M);
  w.key_s = a.take<int>(M);
  w.item = a.take<int>(M);
  w.item_s = a.take<int>(M);
  w.val = a.take<double>(3 * (size_t)M);
  w.cub_bytes = M > 0 ? scatter_cub_bytes(M, T) : 0;
  w.cub_tmp = a.take<char>(w.cub_bytes);
}

__global__ void iota_kernel(int* __restrict__ a, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}

__device__ __forceinline__ int first_not_below(const int* __restrict__ a, int n, int v) {   // first i with a[i] >= v
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] >= v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__global__ void scatter_gather_kernel(const int* __restrict__ key_s, const int* __restrict__ item_s,
                                      const double* __restrict__ val, int M, int T, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int e0 = first_not_below(key_s, M, t), e1 = first_not_below(key_s, M, t + 1);
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int e = e0; e < e1; ++e) {
    const double* p = val + 3 * (size_t)item_s[e];
    s0 += p[0];
    s1 += p[1];
    s2 += p[2];
  }
  out[3 * (size_t)t] = (float)s0;
  out[3 * (size_t)t + 1] = (float)s1;
  out[3 * (size_t)t + 2] = (float)s2;
}

// w.key / w.val hold the M items (written by the caller's kernel on st)
static int scatter_sum(const ScatterWs& w, int M, int T, float* out, cudaStream_t st) {
  if (T == 0) return 0;
  if (M == 0) {
    MP_CHECK_CUDA(cudaMemsetAsync(out, 0, 3 * (size_t)T * sizeof(float), st));
    return 0;
  }
  iota_kernel<<<div_up(M, 256), 256, 0, st>>>(w.item, M);
  MP_LAUNCH_CHECK();
  size_t cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cb, w.key, w.key_s, w.item, w.item_s, M, 0,
                                                key_bits(T + 1), st));
  scatter_gather_kernel<<<div_up(T, 128), 128, 0, st>>>(w.key_s, w.item_s, w.val, M, T, out);
  MP_LAUNCH_CHECK();
  return 0;
}

// ---- depth backward ------------------------------------------------------------------------------------------------

// Pixel i: the exact derivative of its z with respect to its face's three world-space vertices, the face held fixed,
// times d_zbuf[i]; items 3i + j (j = corner) go to the face's vertices.  A pixel without a face or with d_zbuf = 0
// adds nothing.
__global__ void raster_backward_kernel(Cam k, const float* __restrict__ verts, int V, const int64_t* __restrict__ faces,
                                       int F, int H, int W, const int64_t* __restrict__ pix_to_face,
                                       const float* __restrict__ d_zbuf, int* __restrict__ key,
                                       double* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int64_t f = pix_to_face[i];
  const double g = d_zbuf[i];
  Tri t;
  t.ok = false;
  if (f >= 0 && f < F && g != 0.0) t = tri_setup(k, verts, V, faces, (int)f, H, W);
  if (!t.ok) {
    for (int j = 0; j < 3; ++j) {
      key[3 * (size_t)i + j] = V;
      for (int a = 0; a < 3; ++a) val[9 * (size_t)i + 3 * j + a] = 0.0;
    }
    return;
  }
  const double px = (i % W) + 0.5, py = (i / W) + 0.5;
  double b[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) b[j] = edge_fn(t, j, px, py) / t.A;
  const double s = (b[0] / t.Z[0] + b[1] / t.Z[1]) + b[2] / t.Z[2];
  const double z = 1.0 / s;
  const double gS = -g * z * z;                  // dL/dS, z = 1 / S
  double gb[3], du[3] = {0.0, 0.0, 0.0}, dv[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int j = 0; j < 3; ++j) gb[j] = gS / t.Z[j];
  const double Q = (gb[0] * b[0] + gb[1] * b[1]) + gb[2] * b[2];
#pragma unroll
  for (int a = 0; a < 3; ++a) {                  // b_a = e_a / A, A = e_0 + e_1 + e_2: dL/de_a = (gb_a - Q) / A
    const int j = a == 2 ? 0 : a + 1, m = a == 0 ? 2 : a - 1;
    const double h = (gb[a] - Q) / t.A;
    du[j] += h * (t.v[m] - py);
    du[m] -= h * (t.v[j] - py);
    dv[m] += h * (t.u[j] - px);
    dv[j] -= h * (t.u[m] - px);
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double dX = du[j] * k.fx / t.Z[j], dY = dv[j] * k.fy / t.Z[j];
    const double dZ = -gS * b[j] / (t.Z[j] * t.Z[j]) - (du[j] * k.fx * t.X[j] + dv[j] * k.fy * t.Y[j]) / (t.Z[j] * t.Z[j]);
    key[3 * (size_t)i + j] = (int)faces[3 * (size_t)f + j];
    for (int a = 0; a < 3; ++a) val[9 * (size_t)i + 3 * j + a] = (k.R[a] * dX + k.R[3 + a] * dY) + k.R[6 + a] * dZ;
  }
}

// ---- K = 1 nearest vertex ------------------------------------------------------------------------------------------

constexpr int kKnnThreads = 128;
constexpr int kKnnTile = 1024;
constexpr int kKnnTargetCtas = 1024;     // the p2 range is split until about this many CTAs run

// d2 = (dx*dx + dy*dy) + dz*dz in fp32, each step rounded (oracle/port.py:knn_points).  The arg-min over the CTA's
// chunk of p2 compares the distance's bits (d2 >= 0: finite < inf < NaN) with the first index kept on ties; the chunks
// meet in an atomicMin of (bits, index).
__global__ void __launch_bounds__(kKnnThreads) knn1_kernel(const float* __restrict__ p1, int N1,
                                                           const float* __restrict__ p2, int N2, int chunk,
                                                           unsigned long long* __restrict__ keys) {
  __shared__ float sx[kKnnTile], sy[kKnnTile], sz[kKnnTile];
  const int i = blockIdx.x * kKnnThreads + threadIdx.x;
  float x = 0.f, y = 0.f, z = 0.f;
  if (i < N1) {
    x = p1[3 * (size_t)i];
    y = p1[3 * (size_t)i + 1];
    z = p1[3 * (size_t)i + 2];
  }
  const int j0 = blockIdx.y * chunk, j1 = min(N2, j0 + chunk);
  unsigned best = 0xffffffffu;
  int bi = -1;
  for (int t0 = j0; t0 < j1; t0 += kKnnTile) {
    const int n = min(kKnnTile, j1 - t0);
    __syncthreads();
    for (int q = threadIdx.x; q < n; q += kKnnThreads) {
      sx[q] = p2[3 * (size_t)(t0 + q)];
      sy[q] = p2[3 * (size_t)(t0 + q) + 1];
      sz[q] = p2[3 * (size_t)(t0 + q) + 2];
    }
    __syncthreads();
    for (int q = 0; q < n; ++q) {
      const float dx = __fsub_rn(x, sx[q]), dy = __fsub_rn(y, sy[q]), dz = __fsub_rn(z, sz[q]);
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      const unsigned db = __float_as_uint(d);
      if (db < best) {
        best = db;
        bi = t0 + q;
      }
    }
  }
  if (i < N1 && bi >= 0) atomicMin(&keys[i], ((unsigned long long)best << 32) | (unsigned)bi);
}

__global__ void knn1_decode_kernel(const unsigned long long* __restrict__ keys, int N1, const float* __restrict__ p2,
                                   float* __restrict__ dists, int64_t* __restrict__ idx, float* __restrict__ nn) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N1) return;
  const unsigned long long key = keys[i];
  const int j = (int)(key & 0xffffffffull);
  if (dists) dists[i] = __uint_as_float((unsigned)(key >> 32));
  if (idx) idx[i] = j;
  if (nn)
    for (int a = 0; a < 3; ++a) nn[3 * (size_t)i + a] = p2[3 * (size_t)j + a];
}

// query i: d_p1[i] = 2 (p1 - nn) g; item i adds -2 (p1 - nn) g + d_nn[i] to p2[idx[i]]
__global__ void knn1_backward_kernel(const float* __restrict__ p1, int N1, const float* __restrict__ p2, int N2,
                                     const int64_t* __restrict__ idx, const float* __restrict__ d_dists,
                                     const float* __restrict__ d_nn, float* __restrict__ d_p1, int* __restrict__ key,
                                     double* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N1) return;
  const int64_t j = idx[i];
  const bool ok = j >= 0 && j < N2;
  const double g = d_dists ? (double)d_dists[i] : 0.0;
  for (int a = 0; a < 3; ++a) {
    const double diff = ok ? (double)p1[3 * (size_t)i + a] - (double)p2[3 * (size_t)j + a] : 0.0;
    const double gp = 2.0 * diff * g;
    d_p1[3 * (size_t)i + a] = (float)gp;
    val[3 * (size_t)i + a] = ok ? (d_nn ? (double)d_nn[3 * (size_t)i + a] : 0.0) - gp : 0.0;
  }
  key[i] = ok ? (int)j : N2;
}

static void knn1_carve(Arena& a, int N1, unsigned long long*& keys) { keys = a.take<unsigned long long>(N1); }

}  // namespace mp

extern "C" {

size_t mp_depth_raster_workspace_bytes(int H, int W, int F) {
  if (H < 1 || W < 1 || F < 0 || (long long)H * W * 3 >= (1ll << 31)) return 0;
  mp::Arena a;
  mp::RasterWs w;
  mp::raster_carve(a, H, W, F, w);
  return a.off;
}

int mp_depth_raster(const mp_camera_t* cam_host, const float* verts, int V, const int64_t* faces, int F, int H, int W,
                    float* zbuf, int64_t* pix_to_face, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(cam_host && zbuf && pix_to_face && workspace, "mp_depth_raster: null argument");
  MP_REQUIRE(H >= 1 && W >= 1 && (long long)H * W * 3 < (1ll << 31),
             "mp_depth_raster: need H, W >= 1 and 3 H W < 2^31 (H = %d, W = %d)", H, W);
  MP_REQUIRE(V >= 0 && F >= 0, "mp_depth_raster: need V, F >= 0 (V = %d, F = %d)", V, F);
  MP_REQUIRE(F == 0 || (verts && faces), "mp_depth_raster: null verts or faces");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  RasterWs w;
  raster_carve(a, H, W, F, w);
  MP_TRY(a.fits("mp_depth_raster"));
  const Cam k = cam_of(*cam_host);
  const int n = H * W;
  MP_CHECK_CUDA(cudaMemsetAsync(w.keys, 0xff, (size_t)n * sizeof(unsigned long long), st));
  if (F > 0) {
    MP_CHECK_CUDA(cudaMemsetAsync(w.n_big, 0, sizeof(int), st));
    raster_faces_kernel<<<div_up(F, 128), 128, 0, st>>>(k, verts, V, faces, F, H, W, w.keys, w.big, w.n_big);
    MP_LAUNCH_CHECK();
    raster_big_kernel<<<2 * sm_count(), kBigThreads, 0, st>>>(k, verts, V, faces, H, W, w.big, w.n_big, w.keys);
    MP_LAUNCH_CHECK();
  }
  raster_decode_kernel<<<div_up(n, 256), 256, 0, st>>>(w.keys, n, zbuf, pix_to_face);
  MP_LAUNCH_CHECK();
  return 0;
}

size_t mp_depth_raster_backward_workspace_bytes(int H, int W, int V) {
  if (H < 1 || W < 1 || V < 0 || (long long)H * W * 3 >= (1ll << 31)) return 0;
  mp::Arena a;
  mp::ScatterWs w;
  mp::scatter_carve(a, 3 * H * W, V, w);
  return a.off;
}

int mp_depth_raster_backward(const mp_camera_t* cam_host, const float* verts, int V, const int64_t* faces, int F, int H,
                             int W, const int64_t* pix_to_face, const float* d_zbuf, float* d_verts, void* workspace,
                             size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(cam_host && pix_to_face && d_zbuf, "mp_depth_raster_backward: null argument");
  MP_REQUIRE(H >= 1 && W >= 1 && (long long)H * W * 3 < (1ll << 31),
             "mp_depth_raster_backward: need H, W >= 1 and 3 H W < 2^31 (H = %d, W = %d)", H, W);
  MP_REQUIRE(V >= 0 && F >= 0, "mp_depth_raster_backward: need V, F >= 0 (V = %d, F = %d)", V, F);
  MP_REQUIRE(V == 0 || (verts && d_verts), "mp_depth_raster_backward: null verts or d_verts");
  MP_REQUIRE(F == 0 || faces, "mp_depth_raster_backward: null faces");
  cudaStream_t st = (cudaStream_t)stream;
  const int M = 3 * H * W;
  Arena a(workspace, workspace_bytes);
  ScatterWs w;
  scatter_carve(a, M, V, w);
  MP_TRY(a.fits("mp_depth_raster_backward"));
  if (V == 0) return 0;
  raster_backward_kernel<<<div_up(H * W, 128), 128, 0, st>>>(cam_of(*cam_host), verts, V, faces, F, H, W, pix_to_face,
                                                              d_zbuf, w.key, w.val);
  MP_LAUNCH_CHECK();
  return scatter_sum(w, M, V, d_verts, st);
}

size_t mp_knn1_workspace_bytes(int N1) {
  if (N1 < 0) return 0;
  mp::Arena a;
  unsigned long long* keys;
  mp::knn1_carve(a, N1, keys);
  return a.off;
}

int mp_knn1(const float* p1, int N1, const float* p2, int N2, float* dists, int64_t* idx, float* nn, void* workspace,
            size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(N1 >= 0 && N2 >= 1, "mp_knn1: need N1 >= 0 and N2 >= 1 (N1 = %d, N2 = %d)", N1, N2);
  if (N1 == 0) return 0;
  MP_REQUIRE(p1 && p2 && workspace, "mp_knn1: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  unsigned long long* keys;
  knn1_carve(a, N1, keys);
  MP_TRY(a.fits("mp_knn1"));
  MP_CHECK_CUDA(cudaMemsetAsync(keys, 0xff, (size_t)N1 * sizeof(unsigned long long), st));
  const int qb = div_up(N1, kKnnThreads);
  const int splits = max(1, min(div_up(kKnnTargetCtas, qb), div_up(N2, kKnnTile)));
  const int chunk = div_up(N2, splits);
  knn1_kernel<<<dim3(qb, div_up(N2, chunk)), kKnnThreads, 0, st>>>(p1, N1, p2, N2, chunk, keys);
  MP_LAUNCH_CHECK();
  knn1_decode_kernel<<<div_up(N1, 256), 256, 0, st>>>(keys, N1, p2, dists, idx, nn);
  MP_LAUNCH_CHECK();
  return 0;
}

size_t mp_knn1_backward_workspace_bytes(int N1, int N2) {
  if (N1 < 0 || N2 < 1) return 0;
  mp::Arena a;
  mp::ScatterWs w;
  mp::scatter_carve(a, N1, N2, w);
  return a.off;
}

int mp_knn1_backward(const float* p1, int N1, const float* p2, int N2, const int64_t* idx, const float* d_dists,
                     const float* d_nn, float* d_p1, float* d_p2, void* workspace, size_t workspace_bytes,
                     void* stream) {
  using namespace mp;
  MP_REQUIRE(N1 >= 0 && N2 >= 1, "mp_knn1_backward: need N1 >= 0 and N2 >= 1 (N1 = %d, N2 = %d)", N1, N2);
  MP_REQUIRE(p2 && d_p2, "mp_knn1_backward: null argument");
  MP_REQUIRE(N1 == 0 || (p1 && idx && d_p1 && workspace), "mp_knn1_backward: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  ScatterWs w;
  scatter_carve(a, N1, N2, w);
  MP_TRY(a.fits("mp_knn1_backward"));
  if (N1 > 0) {
    knn1_backward_kernel<<<div_up(N1, 128), 128, 0, st>>>(p1, N1, p2, N2, idx, d_dists, d_nn, d_p1, w.key, w.val);
    MP_LAUNCH_CHECK();
  }
  return scatter_sum(w, N1, N2, d_p2, st);
}

}  // extern "C"
