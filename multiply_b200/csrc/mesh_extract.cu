// Mesh extraction: lib/utils/mesh.py:generate_mesh (:78-132) on the device.
//   1. MISE (:87-109 driving lib/libmise/mise.pyx): octree refinement around sign changes, then to_dense().
//   2. Marching cubes (:111-119) on any dense grid, with the tiling DESIGN §3.7 defines (skimage's Lewiner tables are not
//      reproduced).
//   3. The connected component of largest area (:122-130).
// Every step is deterministic: counts, scans and emits in lattice / cube / face order, no float atomics.  fp64 arithmetic
// (vertex positions, the asymptotic decider, areas) rounds op by op as the CPU restatement (oracle/mesh_extract.py)
// does; the file is compiled with -fmad=false.
#include "common.cuh"
#include <cub/cub.cuh>

namespace mp {

// ---- 1. MISE -------------------------------------------------------------------------------------------------------
//
// State.  `state` [(R+1)^3]: 0 = never added, 1 = added and waiting for its value, 2 = known.  The octree is kept as
// `leaf` [(R/2)^3], one byte per voxel of level depth-1: the level L < depth of the leaf that contains it, or depth once
// the voxel itself has been split (its 8 children are leaves of the finest level, which never split).  A leaf of level
// L is identified by its anchor, the voxel of level depth-1 at its lowest corner; its marks live there (`pos`, `neg`).
//
// One round (mise.pyx: update = set values, subdivide_voxels):
//   count + scan the waiting points in lattice order (the one host read of the round: their number; 0 ends the loop),
//   evaluate them in slabs through the sdf-only MLP program with slot = lattice index, so values land in the grid;
//   mark: every known point marks each leaf whose closed box holds it, positive if value >= level, negative if <= level;
//   split: a leaf below depth marked both ways gets level L+1 and adds the 27 points of its children.
// Marks are complete before any split of the round (two kernels), as subdivide_voxels computes them in a first loop.

constexpr int kMiseBlock = 256;
constexpr int kMiseSlab = 1 << 20;

__global__ void mise_init_kernel(uint8_t* __restrict__ state, int R, int step) {
  const long long n1 = R + 1, n = n1 * n1 * n1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % n1), y = (int)((i / n1) % n1), x = (int)(i / (n1 * n1));
    state[i] = (x % step == 0 && y % step == 0 && z % step == 0) ? 1 : 0;
  }
}

__global__ void mise_count_kernel(const uint8_t* __restrict__ state, long long n, int* __restrict__ blk) {
  typedef cub::BlockReduce<int, kMiseBlock> Red;
  __shared__ typename Red::TempStorage tmp;
  const long long i = blockIdx.x * (long long)kMiseBlock + threadIdx.x;
  const int s = Red(tmp).Sum((i < n && state[i] == 1) ? 1 : 0);
  if (threadIdx.x == 0) blk[blockIdx.x] = s;
}

__global__ void mise_total_kernel(const int* __restrict__ blk_off, const int* __restrict__ blk, int nb, int* __restrict__ total) {
  *total = blk_off[nb - 1] + blk[nb - 1];
}

// waiting points of rank [b0, b0 + cap) in lattice order -> slot (lattice index) and fp32 point
__global__ void mise_emit_kernel(const uint8_t* __restrict__ state, long long n, const int* __restrict__ blk_off, int b0,
                                 int cap, int R, float cx, float cy, float cz, float extent, float pad,
                                 int* __restrict__ slot, float* __restrict__ pts) {
  typedef cub::BlockScan<int, kMiseBlock> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const long long i = blockIdx.x * (long long)kMiseBlock + threadIdx.x;
  const int f = (i < n && state[i] == 1) ? 1 : 0;
  int r;
  Scan(tmp).ExclusiveSum(f, r);
  r += blk_off[blockIdx.x] - b0;
  if (!f || r < 0 || r >= cap) return;
  const long long n1 = R + 1;
  const int z = (int)(i % n1), y = (int)((i / n1) % n1), x = (int)(i / (n1 * n1));
  slot[r] = (int)i;
  pts[3 * (size_t)r + 0] = lattice_coord(x, R, pad, extent, cx);
  pts[3 * (size_t)r + 1] = lattice_coord(y, R, pad, extent, cy);
  pts[3 * (size_t)r + 2] = lattice_coord(z, R, pad, extent, cz);
}

// waiting -> known; each known point marks the leaves around it (mise.pyx:197-218)
__global__ void mise_mark_kernel(uint8_t* __restrict__ state, const float* __restrict__ grid, int R, int depth,
                                 double level, const uint8_t* __restrict__ leaf, uint8_t* __restrict__ pos,
                                 uint8_t* __restrict__ neg) {
  const long long n1 = R + 1, n = n1 * n1 * n1;
  const int Rh = R >> 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t s = state[i];
    if (s == 0) continue;
    if (s == 1) state[i] = 2;
    if (depth == 0) continue;                  // no octree: nothing to mark
    const double v = (double)grid[i];
    const bool p = v >= level, q = v <= level;
    if (!p && !q) continue;
    const int z = (int)(i % n1), y = (int)((i / n1) % n1), x = (int)(i / (n1 * n1));
    for (int d = 0; d < 8; ++d) {
      const int cx = x - ((d >> 2) & 1), cy = y - ((d >> 1) & 1), cz = z - (d & 1);     // an adjacent finest cell
      if (cx < 0 || cy < 0 || cz < 0 || cx >= R || cy >= R || cz >= R) continue;
      const int vx = cx >> 1, vy = cy >> 1, vz = cz >> 1;
      const size_t vi = ((size_t)vx * Rh + vy) * Rh + vz;
      const int L = leaf[vi];
      if (L >= depth) continue;                // a finest-level leaf: never split, its marks are not needed
      const int sh = depth - 1 - L;
      const size_t a = ((size_t)((vx >> sh) << sh) * Rh + ((vy >> sh) << sh)) * Rh + ((vz >> sh) << sh);
      if (p) pos[a] = 1;
      if (q) neg[a] = 1;
    }
  }
}

// mise.pyx:220-280: split the leaves marked both ways; the anchor voxel adds the 27 lattice points of the children
__global__ void mise_split_kernel(uint8_t* __restrict__ leaf, const uint8_t* __restrict__ pos,
                                  const uint8_t* __restrict__ neg, uint8_t* __restrict__ state, int R, int depth) {
  const int Rh = R >> 1;
  const long long n = (long long)Rh * Rh * Rh;
  const long long n1 = R + 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int L = leaf[i];
    if (L >= depth) continue;
    const int vz = (int)(i % Rh), vy = (int)((i / Rh) % Rh), vx = (int)(i / ((long long)Rh * Rh));
    const int sh = depth - 1 - L;
    const int ax = (vx >> sh) << sh, ay = (vy >> sh) << sh, az = (vz >> sh) << sh;
    const size_t a = ((size_t)ax * Rh + ay) * Rh + az;
    if (!(pos[a] && neg[a])) continue;
    leaf[i] = (uint8_t)(L + 1);
    if (vx != ax || vy != ay || vz != az) continue;
    const int cs = 1 << (depth - L - 1);       // child size in finest cells
    const int x0 = 2 * ax, y0 = 2 * ay, z0 = 2 * az;
    for (int u = 0; u < 3; ++u)
      for (int v = 0; v < 3; ++v)
        for (int w = 0; w < 3; ++w) {
          const size_t p = ((size_t)(x0 + u * cs) * n1 + (y0 + v * cs)) * n1 + (z0 + w * cs);
          if (state[p] == 0) state[p] = 1;
        }
  }
}

// to_dense (mise.pyx:130-164): never-added points are NaN, then filled by copying forward along x, y, z
__global__ void mise_nan_kernel(const uint8_t* __restrict__ state, float* __restrict__ grid, uint8_t* __restrict__ evaluated,
                                long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (state[i] == 0) grid[i] = __int_as_float(0x7fc00000);
    if (evaluated) evaluated[i] = state[i] != 0;
  }
}

// one thread per line along `axis` (0 = x, 1 = y, 2 = z)
__global__ void mise_fill_kernel(float* __restrict__ grid, int R, int axis) {
  const long long n1 = R + 1;
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n1 * n1) return;
  const long long a = t / n1, b = t % n1;     // the two other coordinates, in x-major order
  long long base, stride;
  if (axis == 0) { base = a * n1 + b; stride = n1 * n1; }
  else if (axis == 1) { base = a * n1 * n1 + b; stride = n1; }
  else { base = (a * n1 + b) * n1; stride = 1; }
  float prev = grid[base];
  for (long long k = 1; k < n1; ++k) {
    const long long i = base + k * stride;
    float v = grid[i];
    if (isnan(v)) {
      v = prev;
      grid[i] = v;
    }
    prev = v;
  }
}

struct MiseWs {
  uint8_t *state, *leaf, *pos, *neg;
  int *blk, *blk_off, *total, *slot;
  float* pts;
  void* cub_tmp;
  size_t cub_bytes;
  void* mlp;
  size_t mlp_bytes;
};

static size_t mise_cub_bytes(int nb) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, nb);
  return b;
}

static void mise_carve(Arena& a, int res_init, int depth, MiseWs& w) {
  const long long R = (long long)res_init << depth, n1 = R + 1, n = n1 * n1 * n1;
  const long long Rh = R >> 1, nh = depth > 0 ? Rh * Rh * Rh : 1;
  const int nb = (int)((n + kMiseBlock - 1) / kMiseBlock);
  const int slab = (int)(n < kMiseSlab ? n : kMiseSlab);
  w.state = a.take<uint8_t>(n);
  w.leaf = a.take<uint8_t>(nh);
  w.pos = a.take<uint8_t>(nh);
  w.neg = a.take<uint8_t>(nh);
  w.blk = a.take<int>(nb);
  w.blk_off = a.take<int>(nb);
  w.total = a.take<int>(1);
  w.slot = a.take<int>(slab);
  w.pts = a.take<float>((size_t)slab * 3);
  w.cub_bytes = mise_cub_bytes(nb);
  w.cub_tmp = a.take<char>(w.cub_bytes);
  w.mlp_bytes = field_ws_bytes(slab);
  w.mlp = a.take<char>(w.mlp_bytes);
}

static int grid_stride_blocks(long long n) {
  const long long b = (n + 255) / 256, cap = (long long)sm_count() * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// ---- 2. marching cubes ---------------------------------------------------------------------------------------------
//
// Cube corners c = 4 dx + 2 dy + dz.  The 12 cube edges are numbered in the order of their lattice-edge ids
// 3 * (lattice index of the lower corner) + axis, which is the same for every cube: kEdgeLo / kEdgeAxis.  kFaceCorners
// lists each cube face's corners counter-clockwise seen from outside the cube, kFaceEdges the edge between corner j
// and j+1.  Walking a face that way, an edge going from a not-below to a below corner starts a segment and an edge
// going from below to not-below ends one; each segment runs from a start to an end, so the cube's segments chain into
// polygons whose right-hand normal points away from the below region (toward increasing value).

__constant__ int8_t kEdgeLo[12] = {0, 0, 0, 1, 1, 2, 2, 3, 4, 4, 5, 6};
__constant__ int8_t kEdgeAxis[12] = {0, 1, 2, 0, 1, 0, 2, 0, 1, 2, 1, 2};
__constant__ int8_t kFaceCorners[6][4] = {{0, 1, 3, 2}, {4, 6, 7, 5}, {0, 4, 5, 1}, {2, 3, 7, 6}, {0, 2, 6, 4}, {1, 5, 7, 3}};
__constant__ int8_t kFaceEdges[6][4] = {{2, 4, 6, 1}, {8, 11, 10, 9}, {0, 9, 3, 2}, {6, 7, 11, 5}, {1, 5, 8, 0}, {3, 10, 7, 4}};

constexpr int kMcBlock = 256;

__device__ __forceinline__ bool mc_below(float v, double level) { return (double)v < level; }

// next[e] = the edge that follows crossing edge e in its polygon.  fv = value - level of the 8 corners (fp64).
__device__ void cube_next(unsigned below, const double fv[8], int8_t next[12]) {
  for (int f = 0; f < 6; ++f) {
    int starts[2], ns = 0, end = -1;
    for (int j = 0; j < 4; ++j) {
      const unsigned bj = (below >> kFaceCorners[f][j]) & 1u, bn = (below >> kFaceCorners[f][(j + 1) & 3]) & 1u;
      if (!bj && bn) starts[ns++] = j;
      if (bj && !bn) end = j;
    }
    if (ns == 1) {
      next[kFaceEdges[f][starts[0]]] = kFaceEdges[f][end];
    } else if (ns == 2) {
      // diagonal corners alike: asymptotic decider.  The bilinear saddle is not below iff the product of the not-below
      // diagonal >= the product of the below diagonal; then the below corners are cut off separately.
      const int q0 = kFaceCorners[f][0], q1 = kFaceCorners[f][1], q2 = kFaceCorners[f][2], q3 = kFaceCorners[f][3];
      const double p02 = fv[q0] * fv[q2], p13 = fv[q1] * fv[q3];
      const bool q0_below = (below >> q0) & 1u;
      const bool sep_below = q0_below ? (p13 >= p02) : (p02 >= p13);
      for (int s = 0; s < 2; ++s) {
        const int j = starts[s];
        next[kFaceEdges[f][j]] = kFaceEdges[f][sep_below ? ((j + 1) & 3) : ((j + 3) & 3)];
      }
    }
  }
}

__device__ __forceinline__ unsigned cube_cross(unsigned below) {
  unsigned c = 0;
  for (int e = 0; e < 12; ++e) {
    const int lo = kEdgeLo[e], hi = lo | (4 >> kEdgeAxis[e]);
    if (((below >> lo) ^ (below >> hi)) & 1u) c |= 1u << e;
  }
  return c;
}

// corner values of cube (x, y, z) -> below mask and fv
__device__ __forceinline__ unsigned cube_load(const float* __restrict__ g, int n1, int x, int y, int z, double level,
                                              double fv[8]) {
  unsigned below = 0;
  for (int c = 0; c < 8; ++c) {
    const float v = g[((size_t)(x + (c >> 2)) * n1 + (y + ((c >> 1) & 1))) * n1 + (z + (c & 1))];
    fv[c] = (double)v - level;
    if (mc_below(v, level)) below |= 1u << c;
  }
  return below;
}

// triangles of a cube (fan from each polygon's lowest edge); emit(k, e0, e1, e2) for k = 0, 1, ...
template <typename Emit>
__device__ int cube_triangles(unsigned below, const double fv[8], Emit emit) {
  const unsigned cross = cube_cross(below);
  if (!cross) return 0;
  int8_t next[12];
  cube_next(below, fv, next);
  unsigned seen = 0;
  int nt = 0;
  for (int e = 0; e < 12; ++e) {
    if (!((cross >> e) & 1u) || ((seen >> e) & 1u)) continue;
    seen |= 1u << e;
    int a = next[e], b = next[a];
    seen |= 1u << a;
    while (b != e) {
      emit(nt++, e, a, b);
      seen |= 1u << b;
      a = b;
      b = next[b];
    }
  }
  return nt;
}

// crossing bits of lattice point (x, y, z): bit a = the edge to the next point along axis a carries a vertex
__device__ __forceinline__ unsigned point_bits(const float* __restrict__ g, int n1, int x, int y, int z, double level) {
  const size_t i = ((size_t)x * n1 + y) * n1 + z;
  const bool b = mc_below(g[i], level);
  unsigned r = 0;
  if (x + 1 < n1 && mc_below(g[i + (size_t)n1 * n1], level) != b) r |= 1u;
  if (y + 1 < n1 && mc_below(g[i + n1], level) != b) r |= 2u;
  if (z + 1 < n1 && mc_below(g[i + 1], level) != b) r |= 4u;
  return r;
}

// vertices per lattice line (x, y): one block per line
__global__ void mc_line_count_kernel(const float* __restrict__ g, int R, double level, long long* __restrict__ cnt) {
  typedef cub::BlockReduce<int, kMcBlock> Red;
  __shared__ typename Red::TempStorage tmp;
  const int n1 = R + 1, x = blockIdx.x / n1, y = blockIdx.x % n1;
  int s = 0;
  for (int z = threadIdx.x; z < n1; z += kMcBlock) s += __popc(point_bits(g, n1, x, y, z, level));
  s = Red(tmp).Sum(s);
  if (threadIdx.x == 0) cnt[blockIdx.x] = s;
}

// triangles per cube row (x, y): one block per row
__global__ void mc_row_count_kernel(const float* __restrict__ g, int R, double level, long long* __restrict__ cnt) {
  typedef cub::BlockReduce<int, kMcBlock> Red;
  __shared__ typename Red::TempStorage tmp;
  const int n1 = R + 1, x = blockIdx.x / R, y = blockIdx.x % R;
  int s = 0;
  for (int z = threadIdx.x; z < R; z += kMcBlock) {
    double fv[8];
    const unsigned below = cube_load(g, n1, x, y, z, level, fv);
    s += cube_triangles(below, fv, [](int, int, int, int) {});
  }
  s = Red(tmp).Sum(s);
  if (threadIdx.x == 0) cnt[blockIdx.x] = s;
}

__global__ void mc_totals_kernel(const long long* __restrict__ voff, const long long* __restrict__ vcnt, int nl,
                                 const long long* __restrict__ foff, const long long* __restrict__ fcnt, int nr,
                                 long long* __restrict__ totals) {
  totals[0] = voff[nl - 1] + vcnt[nl - 1];
  totals[1] = foff[nr - 1] + fcnt[nr - 1];
}

// world coordinate of lattice coordinate c (generate_mesh :117-118, numpy fp64), rounded to fp32 once
__device__ __forceinline__ float mc_world(double c, int R, double pad, double extent, double centre) {
  return (float)(((c / (double)R - 0.5) * pad) * extent + centre);
}

// vertices of line (x, y) in lattice-edge order
__global__ void mc_vert_kernel(const float* __restrict__ g, int R, double level, const long long* __restrict__ voff,
                               double cx, double cy, double cz, double extent, double pad, float* __restrict__ verts) {
  typedef cub::BlockScan<int, kMcBlock> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  const int n1 = R + 1, x = blockIdx.x / n1, y = blockIdx.x % n1;
  const double ctr[3] = {cx, cy, cz};
  long long base = voff[blockIdx.x];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int z0 = 0; z0 < n1; z0 += kMcBlock) {
    const int z = z0 + threadIdx.x;
    const unsigned bits = z < n1 ? point_bits(g, n1, x, y, z, level) : 0u;
    int r, tot;
    Scan(tmp).ExclusiveSum((int)__popc(bits), r, tot);
    long long o = base + carry + r;
    if (bits) {
      const size_t i = ((size_t)x * n1 + y) * n1 + z;
      const double v0 = (double)g[i];
      const size_t step[3] = {(size_t)n1 * n1, (size_t)n1, 1};
      for (int a = 0; a < 3; ++a) {
        if (!((bits >> a) & 1u)) continue;
        const double v1 = (double)g[i + step[a]];
        const double t = (level - v0) / (v1 - v0);
        double c[3] = {(double)x, (double)y, (double)z};
        c[a] += t;
        for (int k = 0; k < 3; ++k) verts[3 * o + k] = mc_world(c[k], R, pad, extent, ctr[k]);
        ++o;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
}

// faces of cube row (x, y): the crossing bits and in-line vertex ranks of the 4 lattice lines the row touches are
// staged in shared memory, then every cube emits its triangles at the row's offset + its rank in the row
__global__ void mc_face_kernel(const float* __restrict__ g, int R, double level, const long long* __restrict__ voff,
                               const long long* __restrict__ foff, int64_t* __restrict__ faces) {
  typedef cub::BlockScan<int, kMcBlock> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ uint8_t bits_s[4][1025];
  __shared__ int rank_s[4][1025];
  __shared__ int carry;
  const int n1 = R + 1, x = blockIdx.x / R, y = blockIdx.x % R;
  for (int l = 0; l < 4; ++l) {
    const int lx = x + (l >> 1), ly = y + (l & 1);
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int z0 = 0; z0 < n1; z0 += kMcBlock) {
      const int z = z0 + threadIdx.x;
      const unsigned b = z < n1 ? point_bits(g, n1, lx, ly, z, level) : 0u;
      int r, tot;
      Scan(tmp).ExclusiveSum((int)__popc(b), r, tot);
      if (z < n1) {
        bits_s[l][z] = (uint8_t)b;
        rank_s[l][z] = carry + r;
      }
      __syncthreads();
      if (threadIdx.x == 0) carry += tot;
      __syncthreads();
    }
  }
  long long lbase[4];
  for (int l = 0; l < 4; ++l) lbase[l] = voff[(size_t)(x + (l >> 1)) * n1 + (y + (l & 1))];
  const long long base = foff[blockIdx.x];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int z0 = 0; z0 < R; z0 += kMcBlock) {
    const int z = z0 + threadIdx.x;
    double fv[8];
    unsigned below = 0;
    int nt = 0;
    if (z < R) {
      below = cube_load(g, n1, x, y, z, level, fv);
      nt = cube_triangles(below, fv, [](int, int, int, int) {});
    }
    int r, tot;
    Scan(tmp).ExclusiveSum(nt, r, tot);
    if (nt) {
      const long long o = base + carry + r;
      auto vid = [&](int e) -> long long {
        const int c = kEdgeLo[e], a = kEdgeAxis[e];
        const int l = (c >> 1) & 3;                 // line (dx, dy)
        const int zz = z + (c & 1);
        const unsigned b = bits_s[l][zz];
        return lbase[l] + rank_s[l][zz] + __popc(b & ((1u << a) - 1u));
      };
      cube_triangles(below, fv, [&](int k, int e0, int e1, int e2) {
        faces[3 * (o + k) + 0] = vid(e0);
        faces[3 * (o + k) + 1] = vid(e1);
        faces[3 * (o + k) + 2] = vid(e2);
      });
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
}

struct McWs {
  long long *vcnt, *voff, *fcnt, *foff, *totals;
  void* cub_tmp;
  size_t cub_bytes;
};

static size_t mc_cub_bytes(int n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const long long*)nullptr, (long long*)nullptr, n);
  return b;
}

static void mc_carve(Arena& a, int R, McWs& w) {
  const int nl = (R + 1) * (R + 1), nr = R * R;
  w.vcnt = a.take<long long>(nl);
  w.voff = a.take<long long>(nl);
  w.fcnt = a.take<long long>(nr);
  w.foff = a.take<long long>(nr);
  w.totals = a.take<long long>(2);
  w.cub_bytes = mc_cub_bytes(nl);
  w.cub_tmp = a.take<char>(w.cub_bytes);
}

// ---- 3. largest connected component --------------------------------------------------------------------------------
//
// Union-find over the vertices (every face joins its three), linking the larger root under the smaller one, so each
// component's root is its lowest vertex whatever the schedule.  Faces are sorted by root (stable radix sort: face order
// within a component).  A component's area is the fp64 sum of its faces' areas in that order, in chunks: the sorted
// positions are cut at every component start and every multiple of kAreaChunk, each chunk is summed left to right, and
// the component's chunk sums are added left to right.  The largest area wins; on equal areas, the component holding
// the lowest face index.

constexpr int kAreaChunk = 256;

__device__ int uf_find(int* parent, int x) {
  int cur = ((volatile int*)parent)[x];
  if (cur != x) {
    int prev = x, nxt;
    while (cur > (nxt = ((volatile int*)parent)[cur])) {
      ((volatile int*)parent)[prev] = nxt;
      prev = cur;
      cur = nxt;
    }
  }
  return cur;
}

__device__ void uf_union(int* parent, int a, int b) {
  a = uf_find(parent, a);
  b = uf_find(parent, b);
  while (a != b) {
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicCAS(&parent[b], b, a);
    if (old == b) break;
    b = old;
  }
}

__global__ void cc_init_kernel(int* parent, int V) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) parent[v] = v;
}

__global__ void cc_check_kernel(const int64_t* __restrict__ faces, long long n, int V, int* __restrict__ bad) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n && (faces[i] < 0 || faces[i] >= V)) atomicOr(bad, 1);
}

__global__ void cc_union_kernel(const int64_t* __restrict__ faces, int F, int* parent) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int a = (int)faces[3 * (size_t)f], b = (int)faces[3 * (size_t)f + 1], c = (int)faces[3 * (size_t)f + 2];
  uf_union(parent, a, b);
  uf_union(parent, a, c);
}

// The labels go to their own array: a concurrent uf_find compresses a path by writing a grandparent it read earlier,
// which may land on parent[v] after v's own thread stored the root there, leaving v labelled with a non-root ancestor
// (and dropped from its component).  Compression only ever stores ancestors, so every find still ends at the root.
__global__ void cc_label_kernel(int* parent, int V, int* __restrict__ label) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) label[v] = uf_find(parent, v);
}

__global__ void cc_face_key_kernel(const int64_t* __restrict__ faces, int F, const int* __restrict__ label,
                                   int* __restrict__ key, int* __restrict__ idx) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  key[f] = label[faces[3 * (size_t)f]];
  idx[f] = f;
}

__device__ __forceinline__ double face_area(const float* __restrict__ v, const int64_t* __restrict__ faces, int f) {
  const int64_t a = faces[3 * (size_t)f], b = faces[3 * (size_t)f + 1], c = faces[3 * (size_t)f + 2];
  const double ax = v[3 * a], ay = v[3 * a + 1], az = v[3 * a + 2];
  const double e1x = v[3 * b] - ax, e1y = v[3 * b + 1] - ay, e1z = v[3 * b + 2] - az;
  const double e2x = v[3 * c] - ax, e2y = v[3 * c + 1] - ay, e2z = v[3 * c + 2] - az;
  const double cx = e1y * e2z - e1z * e2y, cy = e1z * e2x - e1x * e2z, cz = e1x * e2y - e1y * e2x;
  return 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
}

// chunk sums at chunk heads (sorted positions)
__global__ void cc_chunk_kernel(const float* __restrict__ verts, const int64_t* __restrict__ faces,
                                const int* __restrict__ key, const int* __restrict__ idx, int F, double* __restrict__ csum) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  if (i % kAreaChunk != 0 && key[i] == key[i - 1]) return;
  double s = 0.0;
  int j = i;
  do {
    s += face_area(verts, faces, idx[j]);
    ++j;
  } while (j < F && j % kAreaChunk != 0 && key[j] == key[i]);
  csum[i] = s;
}

// the winner: (area, -first face) maximal over component starts; one block
__global__ void cc_pick_kernel(const int* __restrict__ key, const int* __restrict__ idx, const double* __restrict__ csum,
                               int F, int* __restrict__ winner) {
  __shared__ double s_area[1024];
  __shared__ int s_face[1024], s_key[1024];
  double best = -1.0;
  int bf = 0x7fffffff, bk = -1;
  for (int i = threadIdx.x; i < F; i += blockDim.x) {
    if (i > 0 && key[i] == key[i - 1]) continue;
    double s = csum[i];
    for (int j = (i / kAreaChunk + 1) * kAreaChunk; j < F && key[j] == key[i]; j += kAreaChunk) s += csum[j];
    const int f = idx[i];
    if (s > best || (s == best && f < bf)) {
      best = s;
      bf = f;
      bk = key[i];
    }
  }
  s_area[threadIdx.x] = best;
  s_face[threadIdx.x] = bf;
  s_key[threadIdx.x] = bk;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const double a2 = s_area[threadIdx.x + o];
      const int f2 = s_face[threadIdx.x + o];
      if (a2 > s_area[threadIdx.x] || (a2 == s_area[threadIdx.x] && f2 < s_face[threadIdx.x])) {
        s_area[threadIdx.x] = a2;
        s_face[threadIdx.x] = f2;
        s_key[threadIdx.x] = s_key[threadIdx.x + o];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *winner = s_key[0];
}

__global__ void cc_flag_kernel(const int* __restrict__ lab, int n, const int* __restrict__ winner, int* __restrict__ flag) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = lab[i] == *winner ? 1 : 0;
}

__global__ void cc_vert_out_kernel(const float* __restrict__ verts, int V, const int* __restrict__ flag,
                                   const int* __restrict__ rank, float* __restrict__ out) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V || !flag[v]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)rank[v] + k] = verts[3 * (size_t)v + k];
}

__global__ void cc_face_out_kernel(const int64_t* __restrict__ faces, int F, const int* __restrict__ flag,
                                   const int* __restrict__ rank, const int* __restrict__ vrank, int64_t* __restrict__ out) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || !flag[f]) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)rank[f] + k] = vrank[faces[3 * (size_t)f + k]];
}

__global__ void cc_totals_kernel(const int* __restrict__ vflag, const int* __restrict__ vrank, int V,
                                 const int* __restrict__ fflag, const int* __restrict__ frank, int F, int* __restrict__ out) {
  out[0] = vrank[V - 1] + vflag[V - 1];
  out[1] = frank[F - 1] + fflag[F - 1];
}

struct CcWs {
  int *parent, *label, *key, *idx, *key_s, *idx_s, *fflag, *frank, *vflag, *vrank, *winner, *totals, *bad;
  double* csum;
  void* cub_tmp;
  size_t cub_bytes;
};

static int key_bits(int V) {
  int b = 1;
  while (b < 31 && (1 << b) < V) ++b;
  return b;
}

static size_t cc_cub_bytes(int V, int F) {
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr, F,
                                  0, key_bits(V));
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, F);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const int*)nullptr, (int*)nullptr, V);
  return a > b ? (a > c ? a : c) : (b > c ? b : c);
}

static void cc_carve(Arena& a, int V, int F, CcWs& w) {
  w.parent = a.take<int>(V);
  w.label = a.take<int>(V);
  w.key = a.take<int>(F);
  w.idx = a.take<int>(F);
  w.key_s = a.take<int>(F);
  w.idx_s = a.take<int>(F);
  w.fflag = a.take<int>(F);
  w.frank = a.take<int>(F);
  w.vflag = a.take<int>(V);
  w.vrank = a.take<int>(V);
  w.winner = a.take<int>(1);
  w.totals = a.take<int>(2);
  w.bad = a.take<int>(1);
  w.csum = a.take<double>(F);
  w.cub_bytes = cc_cub_bytes(V, F);
  w.cub_tmp = a.take<char>(w.cub_bytes);
}

}  // namespace mp

extern "C" {

size_t mp_mise_workspace_bytes(int res_init, int depth) {
  if (res_init < 1 || depth < 0 || depth > 10 || ((long long)res_init << depth) > 1024) return 0;
  mp::Arena a;
  mp::MiseWs w;
  mp::mise_carve(a, res_init, depth, w);
  return a.off;
}

int mp_mise(mp_net_t* field, const float* center_host, float extent, float pad, int res_init, int depth, double level,
            float* grid, uint8_t* evaluated, long long* n_evaluated_host, void* workspace, size_t workspace_bytes,
            void* stream) {
  using namespace mp;
  MP_REQUIRE(field && center_host && grid && workspace, "mp_mise: null argument");
  MP_REQUIRE(!field->f.is_bg, "mp_mise: a foreground field is required");
  MP_REQUIRE(res_init >= 1 && depth >= 0 && depth <= 10 && ((long long)res_init << depth) <= 1024,
             "mp_mise: res_init << depth must be in [1, 1024] (res_init = %d, depth = %d)", res_init, depth);
  MP_REQUIRE(!isnan(level), "mp_mise: level is NaN");
  cudaStream_t st = (cudaStream_t)stream;
  const int R = res_init << depth;
  const long long n1 = R + 1, n = n1 * n1 * n1;
  const int nb = (int)((n + kMiseBlock - 1) / kMiseBlock);
  Arena a(workspace, workspace_bytes);
  MiseWs w;
  mise_carve(a, res_init, depth, w);
  MP_TRY(a.fits("mp_mise"));
  const int gs = grid_stride_blocks(n);
  mise_init_kernel<<<gs, 256, 0, st>>>(w.state, R, 1 << depth);
  MP_LAUNCH_CHECK();
  if (depth > 0) MP_CHECK_CUDA(cudaMemsetAsync(w.leaf, 0, (size_t)(R / 2) * (R / 2) * (R / 2), st));
  long long evaluated_total = 0;
  for (;;) {
    mise_count_kernel<<<nb, kMiseBlock, 0, st>>>(w.state, n, w.blk);
    MP_LAUNCH_CHECK();
    size_t cb = w.cub_bytes;
    MP_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_tmp, cb, w.blk, w.blk_off, nb, st));
    mise_total_kernel<<<1, 1, 0, st>>>(w.blk_off, w.blk, nb, w.total);
    MP_LAUNCH_CHECK();
    int total = 0;
    MP_CHECK_CUDA(cudaMemcpyAsync(&total, w.total, sizeof(int), cudaMemcpyDeviceToHost, st));
    MP_CHECK_CUDA(cudaStreamSynchronize(st));
    if (total == 0) break;
    evaluated_total += total;
    for (int b0 = 0; b0 < total; b0 += kMiseSlab) {
      const int cnt = total - b0 < kMiseSlab ? total - b0 : kMiseSlab;
      mise_emit_kernel<<<nb, kMiseBlock, 0, st>>>(w.state, n, w.blk_off, b0, cnt, R, center_host[0], center_host[1],
                                                  center_host[2], extent, pad, w.slot, w.pts);
      MP_LAUNCH_CHECK();
      MlpCall c{};
      c.x = w.pts;
      c.slot = w.slot;
      c.cap = cnt;
      c.sdf = grid;
      MP_TRY(field_run(field->f, c, w.mlp, w.mlp_bytes, st));
    }
    if (depth == 0) {     // no voxel can split: the waiting points only become known
      mise_mark_kernel<<<gs, 256, 0, st>>>(w.state, grid, R, 0, level, nullptr, nullptr, nullptr);
      MP_LAUNCH_CHECK();
      continue;
    }
    const size_t nh = (size_t)(R / 2) * (R / 2) * (R / 2);
    MP_CHECK_CUDA(cudaMemsetAsync(w.pos, 0, nh, st));
    MP_CHECK_CUDA(cudaMemsetAsync(w.neg, 0, nh, st));
    mise_mark_kernel<<<gs, 256, 0, st>>>(w.state, grid, R, depth, level, w.leaf, w.pos, w.neg);
    MP_LAUNCH_CHECK();
    mise_split_kernel<<<grid_stride_blocks((long long)nh), 256, 0, st>>>(w.leaf, w.pos, w.neg, w.state, R, depth);
    MP_LAUNCH_CHECK();
  }
  mise_nan_kernel<<<gs, 256, 0, st>>>(w.state, grid, evaluated, n);
  MP_LAUNCH_CHECK();
  const int lines = div_up((int)(n1 * n1), 256);
  for (int axis = 0; axis < 3; ++axis) {
    mise_fill_kernel<<<lines, 256, 0, st>>>(grid, R, axis);
    MP_LAUNCH_CHECK();
  }
  if (n_evaluated_host) *n_evaluated_host = evaluated_total;
  return 0;
}

size_t mp_marching_cubes_workspace_bytes(int res) {
  if (res < 1 || res > 1024) return 0;
  mp::Arena a;
  mp::McWs w;
  mp::mc_carve(a, res, w);
  return a.off;
}

int mp_marching_cubes_count(const float* grid, int res, double level, long long* V_host, long long* F_host,
                            void* workspace, size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(grid && V_host && F_host && workspace, "mp_marching_cubes_count: null argument");
  MP_REQUIRE(res >= 1 && res <= 1024, "mp_marching_cubes_count: res out of range (%d)", res);
  MP_REQUIRE(!isnan(level), "mp_marching_cubes_count: level is NaN");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  McWs w;
  mc_carve(a, res, w);
  MP_TRY(a.fits("mp_marching_cubes_count"));
  const int nl = (res + 1) * (res + 1), nr = res * res;
  mc_line_count_kernel<<<nl, kMcBlock, 0, st>>>(grid, res, level, w.vcnt);
  MP_LAUNCH_CHECK();
  mc_row_count_kernel<<<nr, kMcBlock, 0, st>>>(grid, res, level, w.fcnt);
  MP_LAUNCH_CHECK();
  size_t cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_tmp, cb, w.vcnt, w.voff, nl, st));
  cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_tmp, cb, w.fcnt, w.foff, nr, st));
  mc_totals_kernel<<<1, 1, 0, st>>>(w.voff, w.vcnt, nl, w.foff, w.fcnt, nr, w.totals);
  MP_LAUNCH_CHECK();
  long long t[2];
  MP_CHECK_CUDA(cudaMemcpyAsync(t, w.totals, sizeof(t), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaStreamSynchronize(st));
  MP_REQUIRE(t[0] < (1ll << 31) && t[1] < (1ll << 31), "mp_marching_cubes_count: %lld vertices / %lld faces (more "
             "than 2^31)", t[0], t[1]);
  *V_host = t[0];
  *F_host = t[1];
  return 0;
}

int mp_marching_cubes_emit(const float* grid, int res, double level, const double* center_host, double extent,
                           double pad, float* verts, int64_t* faces, void* workspace, size_t workspace_bytes,
                           void* stream) {
  using namespace mp;
  MP_REQUIRE(grid && center_host && workspace, "mp_marching_cubes_emit: null argument");
  MP_REQUIRE(res >= 1 && res <= 1024, "mp_marching_cubes_emit: res out of range (%d)", res);
  MP_REQUIRE(!isnan(level), "mp_marching_cubes_emit: level is NaN");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  McWs w;
  mc_carve(a, res, w);
  MP_TRY(a.fits("mp_marching_cubes_emit"));
  const int nl = (res + 1) * (res + 1), nr = res * res;
  if (verts) {
    mc_vert_kernel<<<nl, kMcBlock, 0, st>>>(grid, res, level, w.voff, center_host[0], center_host[1], center_host[2],
                                            extent, pad, verts);
    MP_LAUNCH_CHECK();
  }
  if (faces) {
    mc_face_kernel<<<nr, kMcBlock, 0, st>>>(grid, res, level, w.voff, w.foff, faces);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

size_t mp_largest_component_workspace_bytes(int V, int F) {
  if (V < 0 || F < 0) return 0;
  mp::Arena a;
  mp::CcWs w;
  mp::cc_carve(a, V, F, w);
  return a.off;
}

int mp_largest_component(const float* verts, int V, const int64_t* faces, int F, float* verts_out, int64_t* faces_out,
                         int* V_out_host, int* F_out_host, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(V_out_host && F_out_host, "mp_largest_component: null argument");
  MP_REQUIRE(V >= 0 && F >= 0, "mp_largest_component: negative size");
  *V_out_host = 0;
  *F_out_host = 0;
  if (V == 0 || F == 0) return 0;
  MP_REQUIRE(verts && faces && verts_out && faces_out && workspace, "mp_largest_component: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Arena a(workspace, workspace_bytes);
  CcWs w;
  cc_carve(a, V, F, w);
  MP_TRY(a.fits("mp_largest_component"));
  MP_CHECK_CUDA(cudaMemsetAsync(w.bad, 0, sizeof(int), st));
  cc_check_kernel<<<div_up(3 * F, 256), 256, 0, st>>>(faces, 3ll * F, V, w.bad);
  MP_LAUNCH_CHECK();
  int bad = 0;
  MP_CHECK_CUDA(cudaMemcpyAsync(&bad, w.bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaStreamSynchronize(st));
  MP_REQUIRE(!bad, "mp_largest_component: a face index is outside [0, V)");
  cc_init_kernel<<<div_up(V, 256), 256, 0, st>>>(w.parent, V);
  MP_LAUNCH_CHECK();
  cc_union_kernel<<<div_up(F, 256), 256, 0, st>>>(faces, F, w.parent);
  MP_LAUNCH_CHECK();
  cc_label_kernel<<<div_up(V, 256), 256, 0, st>>>(w.parent, V, w.label);
  MP_LAUNCH_CHECK();
  cc_face_key_kernel<<<div_up(F, 256), 256, 0, st>>>(faces, F, w.label, w.key, w.idx);
  MP_LAUNCH_CHECK();
  size_t cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, cb, w.key, w.key_s, w.idx, w.idx_s, F, 0, key_bits(V), st));
  cc_chunk_kernel<<<div_up(F, 256), 256, 0, st>>>(verts, faces, w.key_s, w.idx_s, F, w.csum);
  MP_LAUNCH_CHECK();
  cc_pick_kernel<<<1, 1024, 0, st>>>(w.key_s, w.idx_s, w.csum, F, w.winner);
  MP_LAUNCH_CHECK();
  cc_flag_kernel<<<div_up(V, 256), 256, 0, st>>>(w.label, V, w.winner, w.vflag);
  MP_LAUNCH_CHECK();
  cc_flag_kernel<<<div_up(F, 256), 256, 0, st>>>(w.key, F, w.winner, w.fflag);
  MP_LAUNCH_CHECK();
  cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_tmp, cb, w.vflag, w.vrank, V, st));
  cb = w.cub_bytes;
  MP_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_tmp, cb, w.fflag, w.frank, F, st));
  cc_vert_out_kernel<<<div_up(V, 256), 256, 0, st>>>(verts, V, w.vflag, w.vrank, verts_out);
  MP_LAUNCH_CHECK();
  cc_face_out_kernel<<<div_up(F, 256), 256, 0, st>>>(faces, F, w.fflag, w.frank, w.vrank, faces_out);
  MP_LAUNCH_CHECK();
  cc_totals_kernel<<<1, 1, 0, st>>>(w.vflag, w.vrank, V, w.fflag, w.frank, F, w.totals);
  MP_LAUNCH_CHECK();
  int t[2];
  MP_CHECK_CUDA(cudaMemcpyAsync(t, w.totals, sizeof(t), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaStreamSynchronize(st));
  *V_out_host = t[0];
  *F_out_host = t[1];
  return 0;
}

}  // extern "C"
