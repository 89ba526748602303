// Canonical-mesh queries: exact point-to-triangle-mesh distance, inside test, per-ray surface flags.
//   reference: /root/reference/code/lib/model/multiply.py:153-167 (check_off_in_surface_points_cano_mesh, kaolin's
//   point_to_mesh_distance and check_sign), called at :313-316 and merged at :549-560.
//
// Acceleration structure: a uniform grid over the mesh's bounds (padded by a caller-given margin).  Every face is
// binned into each cell its bounding box overlaps (count, scan, fill on the device): `cell_start[c] ..
// cell_start[c+1]` indexes `cell_faces`.  The faces' vertices are stored as three float4 per face.
//
// Arithmetic.  The per-triangle work (closest point, crossing test) is fp64 on fp32 inputs, term by term in the order
// the CPU definitions (oracle/mesh_port.py) write it; the file is compiled with -fmad=false so that every product and sum rounds
// exactly as numpy / torch do on the host.  The grid arithmetic (cell of a coordinate, box distances) is fp64 too.
#include "common.cuh"

namespace mp {

struct MeshGrid {
  double lo[3];
  double h, inv_h;
  int dim[3];
  int ncell;
};

struct Mesh {
  int V, F;
  MeshGrid g;
  long long n_refs;
  int* cell_start;     // [ncell + 1]
  int* cell_cursor;    // [ncell] (build scratch)
  int* cell_faces;     // [n_refs]
  float4* tri;         // [F][3]: v0, v1, v2 (w unused)
};

}  // namespace mp

struct mp_mesh {
  mp::Mesh m;
};

namespace mp {

__device__ __forceinline__ int cell_of(const MeshGrid& g, int k, double x) {
  double t = floor((x - g.lo[k]) * g.inv_h);
  int c = t < 0.0 ? 0 : (t >= (double)g.dim[k] ? g.dim[k] - 1 : (int)t);
  return c;
}

// ---- build ---------------------------------------------------------------------------------------------------------

// bounds of the vertices -> grid header (one block).  Cells are cubes; their number is about F (at most 2^21), each
// axis has 1..1024 cells.
__global__ void mesh_header_kernel(const float* __restrict__ verts, int V, int F, float margin, MeshGrid* __restrict__ out) {
  __shared__ float smin[3][32], smax[3][32];
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < V; i += blockDim.x)
    for (int k = 0; k < 3; ++k) {
      float v = verts[3 * (size_t)i + k];
      mn[k] = fminf(mn[k], v);
      mx[k] = fmaxf(mx[k], v);
    }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int k = 0; k < 3; ++k) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
      mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    }
    if (lane == 0) {
      smin[k][w] = mn[k];
      smax[k][w] = mx[k];
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double lo[3], ext[3];
  for (int k = 0; k < 3; ++k) {
    float a = INFINITY, b = -INFINITY;
    for (int j = 0; j < (int)(blockDim.x >> 5); ++j) {
      a = fminf(a, smin[k][j]);
      b = fmaxf(b, smax[k][j]);
    }
    lo[k] = (double)a - margin;
    ext[k] = fmax((double)b + margin - lo[k], 1e-6);
  }
  const double target = (double)min(max(F, 1), 1 << 21);
  double h = cbrt(ext[0] * ext[1] * ext[2] / target);
  for (int k = 0; k < 3; ++k) h = fmax(h, ext[k] / 1024.0);
  MeshGrid g;
  long long nc;
  for (;;) {     // a flat mesh: the thin axis gets one cell, the others must not make up for it
    nc = 1;
    for (int k = 0; k < 3; ++k) {
      g.lo[k] = lo[k];
      g.dim[k] = max(1, min(1024, (int)ceil(ext[k] / h)));
      nc *= g.dim[k];
    }
    if (nc <= 4 * (long long)target) break;
    h *= 1.25;
  }
  g.h = h;
  g.inv_h = 1.0 / h;
  g.ncell = (int)nc;
  *out = g;
}

__device__ __forceinline__ void face_cells(const MeshGrid& g, const float* __restrict__ verts,
                                           const int64_t* __restrict__ faces, int f, int lo[3], int hi[3],
                                           float4 v[3]) {
  for (int j = 0; j < 3; ++j) {
    int64_t vi = faces[3 * (size_t)f + j];
    v[j] = make_float4(verts[3 * vi], verts[3 * vi + 1], verts[3 * vi + 2], 0.f);
  }
  const float c[3][3] = {{v[0].x, v[1].x, v[2].x}, {v[0].y, v[1].y, v[2].y}, {v[0].z, v[1].z, v[2].z}};
  for (int k = 0; k < 3; ++k) {
    lo[k] = cell_of(g, k, (double)fminf(fminf(c[k][0], c[k][1]), c[k][2]));
    hi[k] = cell_of(g, k, (double)fmaxf(fmaxf(c[k][0], c[k][1]), c[k][2]));
  }
}

// plan: total number of (cell, face) references; flags face indices out of range
__global__ void mesh_count_refs_kernel(const MeshGrid* __restrict__ gp, const float* __restrict__ verts, int V,
                                       const int64_t* __restrict__ faces, int F, unsigned long long* __restrict__ total,
                                       int* __restrict__ bad) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  for (int j = 0; j < 3; ++j) {
    int64_t vi = faces[3 * (size_t)f + j];
    if (vi < 0 || vi >= V) {
      atomicOr(bad, 1);
      return;
    }
  }
  const MeshGrid g = *gp;
  int lo[3], hi[3];
  float4 v[3];
  face_cells(g, verts, faces, f, lo, hi, v);
  atomicAdd(total, (unsigned long long)(hi[0] - lo[0] + 1) * (hi[1] - lo[1] + 1) * (hi[2] - lo[2] + 1));
}

__global__ void mesh_count_kernel(MeshGrid g, const float* __restrict__ verts, const int64_t* __restrict__ faces, int F,
                                  int* __restrict__ counts, float4* __restrict__ tri) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int lo[3], hi[3];
  float4 v[3];
  face_cells(g, verts, faces, f, lo, hi, v);
  tri[3 * (size_t)f] = v[0];
  tri[3 * (size_t)f + 1] = v[1];
  tri[3 * (size_t)f + 2] = v[2];
  for (int z = lo[2]; z <= hi[2]; ++z)
    for (int y = lo[1]; y <= hi[1]; ++y)
      for (int x = lo[0]; x <= hi[0]; ++x) atomicAdd(&counts[(z * g.dim[1] + y) * g.dim[0] + x], 1);
}

// exclusive scan of counts -> cell_start (one block: each thread scans a contiguous chunk) and cursor = cell_start
// (counts and cursor may be the same buffer)
__global__ void mesh_scan_kernel(const int* counts, int n, int* __restrict__ start, int* cursor) {
  __shared__ int part[1024];
  const int t = threadIdx.x, T = blockDim.x;
  const int chunk = (n + T - 1) / T;
  const int b = min(n, t * chunk), e = min(n, b + chunk);
  int s = 0;
  for (int i = b; i < e; ++i) s += counts[i];
  part[t] = s;
  __syncthreads();
  if (t == 0) {
    int acc = 0;
    for (int i = 0; i < T; ++i) {
      int x = part[i];
      part[i] = acc;
      acc += x;
    }
    start[n] = acc;
  }
  __syncthreads();
  int acc = part[t];
  for (int i = b; i < e; ++i) {
    const int c = counts[i];
    start[i] = acc;
    cursor[i] = acc;
    acc += c;
  }
}

__global__ void mesh_fill_kernel(MeshGrid g, const float4* __restrict__ tri, int F, int* __restrict__ cursor,
                                 int* __restrict__ cell_faces) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int lo[3], hi[3];
  const float4 v0 = tri[3 * (size_t)f], v1 = tri[3 * (size_t)f + 1], v2 = tri[3 * (size_t)f + 2];
  const float c[3][3] = {{v0.x, v1.x, v2.x}, {v0.y, v1.y, v2.y}, {v0.z, v1.z, v2.z}};
  for (int k = 0; k < 3; ++k) {
    lo[k] = cell_of(g, k, (double)fminf(fminf(c[k][0], c[k][1]), c[k][2]));
    hi[k] = cell_of(g, k, (double)fmaxf(fmaxf(c[k][0], c[k][1]), c[k][2]));
  }
  for (int z = lo[2]; z <= hi[2]; ++z)
    for (int y = lo[1]; y <= hi[1]; ++y)
      for (int x = lo[0]; x <= hi[0]; ++x) {
        int pos = atomicAdd(&cursor[(z * g.dim[1] + y) * g.dim[0] + x], 1);
        cell_faces[pos] = f;
      }
}

// ---- point / triangle ----------------------------------------------------------------------------------------------

struct D3 {
  double x, y, z;
};
__device__ __forceinline__ D3 d3(float4 v) { return {(double)v.x, (double)v.y, (double)v.z}; }
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ double dot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ D3 axpy(D3 a, double s, D3 d) { return {a.x + s * d.x, a.y + s * d.y, a.z + s * d.z}; }

// Squared distance from p to triangle (a, b, c) and the Voronoi region of the closest point (Ericson, Real-Time
// Collision Detection 5.1.5): 0 face interior, 1/2/3 vertex a/b/c, 4/5/6 edge ab/bc/ca.  oracle/mesh_port.py:
// _closest_point_triangle is the same sequence of operations.
__device__ __forceinline__ double point_triangle_d2(D3 p, D3 a, D3 b, D3 c, int& type) {
  const D3 ab = sub(b, a), ac = sub(c, a), ap = sub(p, a);
  const double d1 = dot(ab, ap), d2 = dot(ac, ap);
  D3 q;
  if (d1 <= 0.0 && d2 <= 0.0) {
    type = 1;
    q = a;
  } else {
    const D3 bp = sub(p, b);
    const double d3v = dot(ab, bp), d4 = dot(ac, bp);
    if (d3v >= 0.0 && d4 <= d3v) {
      type = 2;
      q = b;
    } else {
      const double vc = d1 * d4 - d3v * d2;
      if (vc <= 0.0 && d1 >= 0.0 && d3v <= 0.0) {
        type = 4;
        q = axpy(a, d1 / (d1 - d3v), ab);
      } else {
        const D3 cp = sub(p, c);
        const double d5 = dot(ab, cp), d6 = dot(ac, cp);
        if (d6 >= 0.0 && d5 <= d6) {
          type = 3;
          q = c;
        } else {
          const double vb = d5 * d2 - d1 * d6;
          if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
            type = 6;
            q = axpy(a, d2 / (d2 - d6), ac);
          } else {
            const double va = d3v * d6 - d5 * d4;
            const double e43 = d4 - d3v, e56 = d5 - d6;
            if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) {
              type = 5;
              q = axpy(b, e43 / (e43 + e56), sub(c, b));
            } else {
              type = 0;
              const double den = 1.0 / (va + vb + vc);
              q = axpy(axpy(a, vb * den, ab), vc * den, ac);
            }
          }
        }
      }
    }
  }
  const D3 d = sub(p, q);
  return dot(d, d);
}

// inclusion of a zero edge function: the edge (from -> to, counter-clockwise order in the xy projection) owns the
// points on it iff it points up, or exactly left.  Antisymmetric in the direction, so of two triangles that share an
// edge from opposite sides exactly one counts a point on it.
__device__ __forceinline__ bool edge_owns(double dx, double dy) { return dy > 0.0 || (dy == 0.0 && dx < 0.0); }

// Crossing of the ray p + t (0,0,1), t > 0, with triangle (a, b, c).  Returns t (> 0) or -1.  Watertight: edge
// functions in fp64 on fp32 inputs (exact whenever the coordinate differences fit in 26 bits), ties by edge_owns.
// oracle/mesh_port.py: check_sign is the same sequence of operations.
__device__ __forceinline__ double ray_z_crossing(D3 p, float4 fa, float4 fb, float4 fc) {
  const D3 a = sub(d3(fa), p), b = sub(d3(fb), p), c = sub(d3(fc), p);
  double U = b.x * c.y - b.y * c.x;     // edge b -> c
  double V = c.x * a.y - c.y * a.x;     // edge c -> a
  double W = a.x * b.y - a.y * b.x;     // edge a -> b
  const double den = U + V + W;
  if (den == 0.0) return -1.0;
  const double s = den > 0.0 ? 1.0 : -1.0;
  U *= s;
  V *= s;
  W *= s;
  if (U < 0.0 || V < 0.0 || W < 0.0) return -1.0;
  // counter-clockwise direction of each edge: as written when den > 0, reversed otherwise
  if (U == 0.0 && !edge_owns(s * (c.x - b.x), s * (c.y - b.y))) return -1.0;
  if (V == 0.0 && !edge_owns(s * (a.x - c.x), s * (a.y - c.y))) return -1.0;
  if (W == 0.0 && !edge_owns(s * (b.x - a.x), s * (b.y - a.y))) return -1.0;
  const double t = (U * a.z + V * b.z + W * c.z) / (s * den);
  return t > 0.0 ? t : -1.0;
}

// ---- queries -------------------------------------------------------------------------------------------------------

// Nearest face to p among faces with d2 <= cap2 (cap2 = +inf: exact query).  Rings of cells around the cell of p
// (clamped into the grid) are visited nearest first; ring r is visited only if the lower bound of the distance from p
// to any cell outside the block of rings < r can still beat min(best, cap2).  For p outside the grid, q = clamp(p):
// |p - x|^2 >= |p - q|^2 + |q - x|^2 for every x in the grid box.  Ties: lowest face index.
__device__ bool mesh_nearest(const Mesh& m, D3 p, double cap2, double& best, int& best_f, int& best_t) {
  const MeshGrid& g = m.g;
  double q[3] = {p.x, p.y, p.z}, out2 = 0.0;
  int c0[3];
  for (int k = 0; k < 3; ++k) {
    const double hi = g.lo[k] + g.dim[k] * g.h;
    double v = q[k] < g.lo[k] ? g.lo[k] : (q[k] > hi ? hi : q[k]);
    out2 += (q[k] - v) * (q[k] - v);
    q[k] = v;
    c0[k] = cell_of(g, k, v);
  }
  best = INFINITY;
  best_f = -1;
  best_t = 0;
  const D3 pd = p;
  int rmax = 0;
  for (int k = 0; k < 3; ++k) rmax = max(rmax, max(c0[k], g.dim[k] - 1 - c0[k]));
  for (int r = 0; r <= rmax; ++r) {
    const double bound = fmin(best, cap2);
    if (r > 0) {
      // distance from q to the outside of the block of rings < r (open sides only)
      double lb = INFINITY;
      for (int k = 0; k < 3; ++k) {
        if (c0[k] - (r - 1) > 0) lb = fmin(lb, q[k] - (g.lo[k] + (c0[k] - (r - 1)) * g.h));
        if (c0[k] + (r - 1) < g.dim[k] - 1) lb = fmin(lb, g.lo[k] + (c0[k] + r) * g.h - q[k]);
      }
      lb = fmax(lb, 0.0);
      if (out2 + lb * lb > bound) break;
    }
    const int z0 = max(c0[2] - r, 0), z1 = min(c0[2] + r, g.dim[2] - 1);
    const int y0 = max(c0[1] - r, 0), y1 = min(c0[1] + r, g.dim[1] - 1);
    for (int z = z0; z <= z1; ++z)
      for (int y = y0; y <= y1; ++y) {
        const bool face_row = (abs(z - c0[2]) == r) || (abs(y - c0[1]) == r);
        const int xs = face_row ? 1 : 2 * r;
        for (int x = c0[0] - r; x <= c0[0] + r; x += (xs > 0 ? xs : 1)) {
          if (x < 0 || x >= g.dim[0]) continue;
          // box distance of the cell from q
          const int cc[3] = {x, y, z};
          double bd = out2;
          for (int k = 0; k < 3; ++k) {
            const double l = g.lo[k] + cc[k] * g.h, u = l + g.h;
            const double e = q[k] < l ? l - q[k] : (q[k] > u ? q[k] - u : 0.0);
            bd += e * e;
          }
          if (bd > fmin(best, cap2)) continue;
          const int cell = (z * g.dim[1] + y) * g.dim[0] + x;
          const int e0 = __ldg(&m.cell_start[cell]), e1 = __ldg(&m.cell_start[cell + 1]);
          for (int e = e0; e < e1; ++e) {
            const int f = __ldg(&m.cell_faces[e]);
            const float4 a = __ldg(&m.tri[3 * (size_t)f]), b = __ldg(&m.tri[3 * (size_t)f + 1]),
                         c = __ldg(&m.tri[3 * (size_t)f + 2]);
            int t;
            const double d2 = point_triangle_d2(pd, d3(a), d3(b), d3(c), t);
            if (d2 <= cap2 && (d2 < best || (d2 == best && f < best_f))) {
              best = d2;
              best_f = f;
              best_t = t;
            }
          }
        }
      }
  }
  return best_f >= 0;
}

// inside = odd number of crossings of the ray p + t (0,0,1), t > 0.  The column of cells above p is walked; a face
// binned into several cells of the column counts only in the cell that holds its crossing point (the crossing's z
// clamped into the face's z-range, so that this cell is one the face is binned into).
__device__ bool mesh_inside(const Mesh& m, D3 p) {
  const MeshGrid& g = m.g;
  for (int k = 0; k < 2; ++k) {
    const double v = k == 0 ? p.x : p.y;
    if (v < g.lo[k] || v > g.lo[k] + g.dim[k] * g.h) return false;
  }
  if (p.z > g.lo[2] + g.dim[2] * g.h) return false;
  const int cx = cell_of(g, 0, p.x), cy = cell_of(g, 1, p.y), cz = cell_of(g, 2, p.z);
  int parity = 0;
  for (int z = cz; z < g.dim[2]; ++z) {
    const int cell = (z * g.dim[1] + cy) * g.dim[0] + cx;
    const int e0 = __ldg(&m.cell_start[cell]), e1 = __ldg(&m.cell_start[cell + 1]);
    for (int e = e0; e < e1; ++e) {
      const int f = __ldg(&m.cell_faces[e]);
      const float4 a = __ldg(&m.tri[3 * (size_t)f]), b = __ldg(&m.tri[3 * (size_t)f + 1]),
                   c = __ldg(&m.tri[3 * (size_t)f + 2]);
      const double t = ray_z_crossing(p, a, b, c);
      if (t < 0.0) continue;
      const double zmin = (double)fminf(fminf(a.z, b.z), c.z), zmax = (double)fmaxf(fmaxf(a.z, b.z), c.z);
      const double zh = fmin(fmax(p.z + t, zmin), zmax);
      if (cell_of(g, 2, zh) == z) parity ^= 1;
    }
  }
  return parity != 0;
}

__global__ void mesh_distance_kernel(Mesh m, const float* __restrict__ pts, int N, float* __restrict__ dist2,
                                     int64_t* __restrict__ face_idx, int* __restrict__ dist_type) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const D3 p = {(double)pts[3 * (size_t)i], (double)pts[3 * (size_t)i + 1], (double)pts[3 * (size_t)i + 2]};
  double best;
  int f, t;
  mesh_nearest(m, p, INFINITY, best, f, t);
  dist2[i] = (float)best;
  if (face_idx) face_idx[i] = f;
  if (dist_type) dist_type[i] = t;
}

__global__ void mesh_sign_kernel(Mesh m, const float* __restrict__ pts, int N, uint8_t* __restrict__ inside) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const D3 p = {(double)pts[3 * (size_t)i], (double)pts[3 * (size_t)i + 1], (double)pts[3 * (size_t)i + 2]};
  inside[i] = mesh_inside(m, p) ? 1 : 0;
}

// Per-ray flags of check_off_in_surface_points_cano_mesh (multiply.py:153-167): with signed distance
// s = (inside ? -1 : 1) * sqrtf(d2), off[row] = AND_s (s > thr), in[row] = OR_s (s <= 0) (= the reference's min tests).
// Inside samples set in; with thr >= 0 they also clear off (s <= 0 <= thr).  Otherwise the sample needs its distance
// only up to |thr|: the capped query is exact below cap2 = max((thr (1 + 1e-6))^2, 2^-120), beyond which
// sqrtf(float(d2)) > |thr| (the floor keeps float(d2) a normal float, so it cannot round to 0).  Past the cap an outside
// sample keeps off (s > |thr| >= thr) and an inside one clears it (s < -|thr| = thr).  thr must not be NaN (the entry
// points reject it).  off / in are initialised to 1 / 0 by the caller and only ever written 0 / 1, so the result does
// not depend on the order of the points.  Point i is sample slot[i] of row slot[i] / n (slot == NULL: slot = i); the
// number of points is *count_dev when given.
__global__ void mesh_flags_kernel(Mesh m, const float* __restrict__ xc, const int* __restrict__ slot,
                                  const int* __restrict__ count_dev, int cap, int n, float thr, double cap2,
                                  uint8_t* __restrict__ off, uint8_t* __restrict__ in) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = count_dev ? min(cap, *count_dev) : cap;
  if (i >= N) return;
  const int row = (slot ? slot[i] : i) / n;
  const D3 p = {(double)xc[3 * (size_t)i], (double)xc[3 * (size_t)i + 1], (double)xc[3 * (size_t)i + 2]};
  const bool inside = mesh_inside(m, p);
  if (inside) {
    in[row] = 1;
    if (thr >= 0.f) {
      off[row] = 0;
      return;
    }
  }
  double best;
  int f, t;
  if (!mesh_nearest(m, p, cap2, best, f, t)) {     // farther than |thr|
    if (inside) off[row] = 0;
    return;
  }
  const float d = sqrtf((float)best);
  const float s = inside ? -d : d;
  if (!(s > thr)) off[row] = 0;
  if (s <= 0.f) in[row] = 1;
}

int launch_surface_flags(const Mesh& m, const float* xc, const int* slot, const int* count_dev, int cap, int n,
                         float thr, uint8_t* off, uint8_t* in, cudaStream_t st) {
  if (cap <= 0) return 0;
  const double c = (double)thr * (1.0 + 1e-6);
  const double cap2 = fmax(c * c, 0x1p-120);
  mesh_flags_kernel<<<div_up(cap, 128), 128, 0, st>>>(m, xc, slot, count_dev, cap, n, thr, cap2, off, in);
  MP_LAUNCH_CHECK();
  return 0;
}

// multiply.py:549-560: off[R] = AND over rendered persons, in[R] = OR; a person's row k is ray hit_index[k].  Rays
// no person hits keep off = 1, in = 0.  Only 0 (off) / 1 (in) are written, so persons may scatter in any order.
__global__ void mesh_merge_flags_kernel(const int64_t* __restrict__ idx, int rows, const int* __restrict__ rows_dev,
                                        const uint8_t* __restrict__ off_p, const uint8_t* __restrict__ in_p,
                                        uint8_t* __restrict__ off, uint8_t* __restrict__ in) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (rows_dev) rows = min(rows, *rows_dev);
  if (k >= rows) return;
  const int64_t r = idx[k];
  if (!off_p[k]) off[r] = 0;
  if (in_p[k]) in[r] = 1;
}

int launch_merge_flags(const int64_t* idx, int rows, const int* rows_dev, const uint8_t* off_p, const uint8_t* in_p,
                       uint8_t* off, uint8_t* in, cudaStream_t st) {
  mesh_merge_flags_kernel<<<div_up(rows, 256), 256, 0, st>>>(idx, rows, rows_dev, off_p, in_p, off, in);
  MP_LAUNCH_CHECK();
  return 0;
}

const Mesh& mesh_of(const mp_mesh_t* h) { return h->m; }

// A mesh as its plan describes it, and the grid's buffers in the caller's storage.
static Mesh mesh_of_plan(const mp_mesh_plan_t& plan) {
  Mesh m{};
  m.V = plan.V;
  m.F = plan.F;
  for (int k = 0; k < 3; ++k) {
    m.g.lo[k] = plan.lo[k];
    m.g.dim[k] = plan.dim[k];
  }
  m.g.h = plan.h;
  m.g.inv_h = 1.0 / plan.h;
  m.g.ncell = plan.dim[0] * plan.dim[1] * plan.dim[2];
  m.n_refs = plan.n_refs;
  return m;
}
static void mesh_carve(Arena& a, Mesh& m) {
  m.cell_start = a.take<int>((size_t)m.g.ncell + 1);
  m.cell_cursor = a.take<int>((size_t)m.g.ncell);
  m.cell_faces = a.take<int>((size_t)m.n_refs);
  m.tri = a.take<float4>((size_t)m.F * 3);
}

}  // namespace mp

extern "C" {

int mp_mesh_plan(const float* verts, int V, const int64_t* faces, int F, float margin, void* scratch,
                 mp_mesh_plan_t* plan, void* stream) {
  MP_REQUIRE(verts && faces && scratch && plan, "mp_mesh_plan: null argument");
  MP_REQUIRE(V >= 3 && F >= 1, "mp_mesh_plan: need V >= 3 and F >= 1 (V = %d, F = %d)", V, F);
  MP_REQUIRE(margin >= 0.f, "mp_mesh_plan: margin must be >= 0");
  cudaStream_t st = (cudaStream_t)stream;
  mp::Arena a(scratch, MP_MESH_PLAN_SCRATCH_BYTES);
  mp::MeshGrid* g = a.take<mp::MeshGrid>(1);
  unsigned long long* total = a.take<unsigned long long>(1);
  int* bad = a.take<int>(1);
  MP_TRY(a.fits("mp_mesh_plan", "scratch"));
  MP_CHECK_CUDA(cudaMemsetAsync(total, 0, sizeof(unsigned long long), st));
  MP_CHECK_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
  mp::mesh_header_kernel<<<1, 1024, 0, st>>>(verts, V, F, margin, g);
  MP_LAUNCH_CHECK();
  mp::mesh_count_refs_kernel<<<mp::div_up(F, 256), 256, 0, st>>>(g, verts, V, faces, F, total, bad);
  MP_LAUNCH_CHECK();
  mp::MeshGrid hg;
  unsigned long long ht = 0;
  int hb = 0;
  MP_CHECK_CUDA(cudaMemcpyAsync(&hg, g, sizeof(hg), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaMemcpyAsync(&ht, total, sizeof(ht), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaMemcpyAsync(&hb, bad, sizeof(hb), cudaMemcpyDeviceToHost, st));
  MP_CHECK_CUDA(cudaStreamSynchronize(st));
  MP_REQUIRE(!hb, "mp_mesh_plan: a face index is outside [0, V)");
  MP_REQUIRE(ht < (1ull << 31), "mp_mesh_plan: %llu cell references (more than 2^31)", ht);
  memset(plan, 0, sizeof(*plan));
  plan->V = V;
  plan->F = F;
  for (int k = 0; k < 3; ++k) {
    plan->lo[k] = hg.lo[k];
    plan->dim[k] = hg.dim[k];
  }
  plan->h = hg.h;
  plan->n_refs = (long long)ht;
  mp::Arena s;
  mp::Mesh m = mp::mesh_of_plan(*plan);
  mp::mesh_carve(s, m);
  plan->storage_bytes = s.off;
  return 0;
}

int mp_mesh_create(const mp_mesh_plan_t* plan, const float* verts, const int64_t* faces, void* storage,
                   size_t storage_bytes, mp_mesh_t** out, void* stream) {
  MP_REQUIRE(plan && verts && faces && storage && out, "mp_mesh_create: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  mp::Mesh m = mp::mesh_of_plan(*plan);
  mp::Arena a(storage, storage_bytes);
  mp::mesh_carve(a, m);
  MP_TRY(a.fits("mp_mesh_create", "storage"));
  MP_CHECK_CUDA(cudaMemsetAsync(m.cell_cursor, 0, (size_t)m.g.ncell * sizeof(int), st));
  mp::mesh_count_kernel<<<mp::div_up(m.F, 256), 256, 0, st>>>(m.g, verts, faces, m.F, m.cell_cursor, m.tri);
  MP_LAUNCH_CHECK();
  mp::mesh_scan_kernel<<<1, 1024, 0, st>>>(m.cell_cursor, m.g.ncell, m.cell_start, m.cell_cursor);
  MP_LAUNCH_CHECK();
  mp::mesh_fill_kernel<<<mp::div_up(m.F, 256), 256, 0, st>>>(m.g, m.tri, m.F, m.cell_cursor, m.cell_faces);
  MP_LAUNCH_CHECK();
  mp_mesh* h = new mp_mesh();
  h->m = m;
  *out = h;
  return 0;
}

void mp_mesh_free(mp_mesh_t* m) { delete m; }

int mp_mesh_distance(const mp_mesh_t* mesh, const float* pts, int N, float* dist2, int64_t* face_idx, int* dist_type,
                     void* stream) {
  MP_REQUIRE(mesh && pts && dist2, "mp_mesh_distance: null argument");
  if (N <= 0) return 0;
  mp::mesh_distance_kernel<<<mp::div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(mesh->m, pts, N, dist2, face_idx,
                                                                                 dist_type);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_mesh_check_sign(const mp_mesh_t* mesh, const float* pts, int N, uint8_t* inside, void* stream) {
  MP_REQUIRE(mesh && pts && inside, "mp_mesh_check_sign: null argument");
  if (N <= 0) return 0;
  mp::mesh_sign_kernel<<<mp::div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(mesh->m, pts, N, inside);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_mesh_surface_flags(const mp_mesh_t* mesh, const float* x_c, int rows, int N_samples, float thr, uint8_t* off,
                          uint8_t* in, void* stream) {
  MP_REQUIRE(mesh && x_c && off && in, "mp_mesh_surface_flags: null argument");
  MP_REQUIRE(N_samples >= 1 && rows >= 0, "mp_mesh_surface_flags: bad sizes");
  MP_REQUIRE(!isnan(thr), "mp_mesh_surface_flags: thr is NaN");
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  MP_CHECK_CUDA(cudaMemsetAsync(off, 1, rows, st));
  MP_CHECK_CUDA(cudaMemsetAsync(in, 0, rows, st));
  return mp::launch_surface_flags(mesh->m, x_c, nullptr, nullptr, rows * N_samples, N_samples, thr, off, in, st);
}

}  // extern "C"
