// SMPLDeformer: nearest-SMPL-vertex skinning-weight lookup + closed-form (inverse) LBS.
//   reference: /root/reference/code/lib/model/deformer.py:19-50 (forward, forward_skinning,
//   query_skinning_weights_smpl_multi), :72-89 (skinning) and the pytorch3d knn_points call at :39.
//
// Design: the 6890 vertices are binned into a uniform grid (cell >= the 0.1 outlier
// radius of deformer.py:49) and stored cell-sorted as float4 (x,y,z,index) so that one warp of
// neighbouring sample points streams the same few cells with 128-bit loads out of L1.  The
// nearest vertex is EXACT: d2 = (dx*dx + dy*dy) + dz*dz with separately rounded operations and
// lowest-index tie-break — the definition the oracle uses (oracle/port.py:knn_points) — and
// points whose grid neighbourhood proves nothing fall back to a full scan when asked.
#include "common.cuh"

namespace mp {

// -------------------------------------------------------------------------------------------
// grid build: single CTA (V = 6890 is tiny); bbox -> cell size -> histogram -> scan -> scatter
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) grid_build_kernel(const float* __restrict__ verts, int V, float cell, int R0,
                                                          GridHeader* __restrict__ hdr,
                                                          int* __restrict__ cell_start, float4* __restrict__ sorted,
                                                          int* __restrict__ cursor) {
  __shared__ float s_lo[3][32], s_hi[3][32];
  __shared__ GridHeader g;
  __shared__ int s_part[1024];
  int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = tid; i < V; i += blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      float v = verts[3 * i + a];
      lo[a] = fminf(lo[a], v);
      hi[a] = fmaxf(hi[a], v);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
    if (lane == 0) {
      s_lo[a][wid] = lo[a];
      s_hi[a][wid] = hi[a];
    }
  }
  __syncthreads();
  if (tid == 0) {
    float ext = 0.f;
    for (int a = 0; a < 3; ++a) {
      float l = INFINITY, h = -INFINITY;
      for (int w = 0; w < 32; ++w) {
        l = fminf(l, s_lo[a][w]);
        h = fmaxf(h, s_hi[a][w]);
      }
      g.lo[a] = l;
      s_hi[a][0] = h;
      ext = fmaxf(ext, h - l);
    }
    float h = cell;
    // 2*R0 empty border cells on every side: a query within 2*R0*h of the vertex bounding box still has its
    // own cell inside the grid, which is what the optimality proof of nearest_vertex() needs.  Keep the grid
    // within kMaxCells (growing h only makes R0 cells cover more than the radius).
    const int pad = 2 * R0;
    for (;;) {
      long long n = 1;
      for (int a = 0; a < 3; ++a) {
        g.dim[a] = (int)floorf((s_hi[a][0] - g.lo[a]) / h) + 1 + 2 * pad;
        n *= g.dim[a];
      }
      if (n <= kMaxCells) {
        g.ncell = (int)n;
        break;
      }
      h *= 1.25f;
    }
    for (int a = 0; a < 3; ++a) g.lo[a] -= (float)pad * h;
    g.R0 = R0;
    g.h = h;
    g.inv_h = 1.0f / h;
    *hdr = g;
  }
  __syncthreads();
  int ncell = g.ncell;
  for (int c = tid; c <= ncell; c += blockDim.x) cursor[c] = 0;
  __syncthreads();
  for (int i = tid; i < V; i += blockDim.x) {
    int cx = min(g.dim[0] - 1, max(0, (int)floorf((verts[3 * i] - g.lo[0]) * g.inv_h)));
    int cy = min(g.dim[1] - 1, max(0, (int)floorf((verts[3 * i + 1] - g.lo[1]) * g.inv_h)));
    int cz = min(g.dim[2] - 1, max(0, (int)floorf((verts[3 * i + 2] - g.lo[2]) * g.inv_h)));
    atomicAdd(&cursor[(cz * g.dim[1] + cy) * g.dim[0] + cx], 1);
  }
  __syncthreads();
  // exclusive scan of cursor[0..ncell) into cell_start (block-wide, chunked)
  int per = (ncell + blockDim.x - 1) / blockDim.x;
  int b = tid * per, e = min(ncell, b + per);
  int s = 0;
  for (int c = b; c < e; ++c) s += cursor[c];
  s_part[tid] = s;
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int t = 0; t < (int)blockDim.x; ++t) {
      int v = s_part[t];
      s_part[t] = run;
      run += v;
    }
    cell_start[ncell] = run;
  }
  __syncthreads();
  int run = s_part[tid];
  for (int c = b; c < e; ++c) {
    int v = cursor[c];
    cell_start[c] = run;
    cursor[c] = run;
    run += v;
  }
  __syncthreads();
  for (int i = tid; i < V; i += blockDim.x) {
    float x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
    int cx = min(g.dim[0] - 1, max(0, (int)floorf((x - g.lo[0]) * g.inv_h)));
    int cy = min(g.dim[1] - 1, max(0, (int)floorf((y - g.lo[1]) * g.inv_h)));
    int cz = min(g.dim[2] - 1, max(0, (int)floorf((z - g.lo[2]) * g.inv_h)));
    int pos = atomicAdd(&cursor[(cz * g.dim[1] + cy) * g.dim[0] + cx], 1);
    sorted[pos] = make_float4(x, y, z, __int_as_float(i));
  }
}

// -------------------------------------------------------------------------------------------
// exact nearest vertex
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void nn_consider(const float4 v, float px, float py, float pz, float& best, int& bi) {
  float dx = __fsub_rn(px, v.x), dy = __fsub_rn(py, v.y), dz = __fsub_rn(pz, v.z);
  float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
  int idx = __float_as_int(v.w);
  if (d < best || (d == best && idx < bi)) {
    best = d;
    bi = idx;
  }
}

// Returns the nearest vertex index and squared distance.  `found_exact` is true when the grid
// neighbourhood proves the result is the global arg-min (best distance <= h); otherwise the
// caller may request a full scan.
// Scan the (2R+1)^3 block of cells around (cx,cy,cz), nearest cells first in z/y, skipping every cell whose
// box is provably farther than the best distance found so far (the box distance carries a safety margin so a
// cell holding an equally distant vertex is never skipped: ties must still resolve to the lowest index).
__device__ __forceinline__ void scan_block(const GridHeader& g, const int* __restrict__ cell_start,
                                           const float4* __restrict__ sorted, int cx, int cy, int cz, int R, float px,
                                           float py, float pz, float& best, int& bi) {
  const float qx = px - g.lo[0], qy = py - g.lo[1], qz = pz - g.lo[2];
  for (int dz = 0; dz <= 2 * R; ++dz) {
    // visiting order 0, -1, +1, -2, +2 ...
    int oz = (dz + 1) >> 1;
    int z = cz + ((dz & 1) ? -oz : oz);
    if (z < 0 || z >= g.dim[2]) continue;
    float ez = fmaxf(fmaxf(z * g.h - qz, qz - (z + 1) * g.h), 0.f);
    for (int dy = 0; dy <= 2 * R; ++dy) {
      int oy = (dy + 1) >> 1;
      int y = cy + ((dy & 1) ? -oy : oy);
      if (y < 0 || y >= g.dim[1]) continue;
      float ey = fmaxf(fmaxf(y * g.h - qy, qy - (y + 1) * g.h), 0.f);
      float dzy = ez * ez + ey * ey;
      if (dzy * 0.9999f - 1e-9f > best) continue;
      int base = (z * g.dim[1] + y) * g.dim[0];
      for (int dx = 0; dx <= 2 * R; ++dx) {
        int ox = (dx + 1) >> 1;
        int x = cx + ((dx & 1) ? -ox : ox);
        if (x < 0 || x >= g.dim[0]) continue;
        float ex = fmaxf(fmaxf(x * g.h - qx, qx - (x + 1) * g.h), 0.f);
        float dc = dzy + ex * ex;
        if (dc * 0.9999f - 1e-9f > best) continue;
        int b = cell_start[base + x], e = cell_start[base + x + 1];
        for (int j = b; j < e; ++j) nn_consider(__ldg(&sorted[j]), px, py, pz, best, bi);
      }
    }
  }
}

__device__ __forceinline__ void nearest_vertex(const GridHeader& g, const int* __restrict__ cell_start,
                                               const float4* __restrict__ sorted, int V, float px, float py,
                                               float pz, bool full_scan_if_unsure, float& best, int& bi) {
  best = INFINITY;
  bi = 0x7fffffff;
  float fx = (px - g.lo[0]) * g.inv_h, fy = (py - g.lo[1]) * g.inv_h, fz = (pz - g.lo[2]) * g.inv_h;
  // clamp before the int conversion so far-away points cannot overflow
  fx = fminf(fmaxf(fx, -4.f), (float)g.dim[0] + 4.f);
  fy = fminf(fmaxf(fy, -4.f), (float)g.dim[1] + 4.f);
  fz = fminf(fmaxf(fz, -4.f), (float)g.dim[2] + 4.f);
  int cx = (int)floorf(fx), cy = (int)floorf(fy), cz = (int)floorf(fz);
  // Everything outside the (2R+1)^3 block is farther than R*h from the query (when the query's own
  // cell lies inside the grid), so best <= (R*h)^2 proves global optimality.
  bool inside = cx >= 0 && cy >= 0 && cz >= 0 && cx < g.dim[0] && cy < g.dim[1] && cz < g.dim[2];
  float hh = g.h * 0.999f;
  if (!full_scan_if_unsure) {
    // outlier classification only: any vertex within the 0.1 radius lies in the (2 R0 + 1)^3 block (R0 h >= 0.1001).
    // The grid carries 2 R0 empty border cells, so a query whose cell is not in [R0, dim-1-R0] on some axis has
    // no vertex in its block at all: the common case for samples far from the body.
    const int R0 = g.R0;
    if (cx < R0 || cy < R0 || cz < R0 || cx > g.dim[0] - 1 - R0 || cy > g.dim[1] - 1 - R0 || cz > g.dim[2] - 1 - R0)
      return;
    scan_block(g, cell_start, sorted, cx, cy, cz, R0, px, py, pz, best, bi);
    return;
  }
  const int R0 = g.R0;
  scan_block(g, cell_start, sorted, cx, cy, cz, R0, px, py, pz, best, bi);
  float rr = (float)R0 * hh;
  bool proven = inside && best <= rr * rr;
  if (!proven && inside) {
    // the first block proved nothing: double the radius (the scan keeps `best`, so pruned cells stay pruned)
    scan_block(g, cell_start, sorted, cx, cy, cz, 2 * R0, px, py, pz, best, bi);
    proven = best <= 4.f * rr * rr;
  }
  if (!proven) {
    best = INFINITY;
    bi = 0x7fffffff;
    for (int j = 0; j < V; ++j) nn_consider(__ldg(&sorted[j]), px, py, pz, best, bi);
    // no finite distance (a non-finite coordinate, or every squared distance overflows): no nearest vertex, rather
    // than the lowest index of a tie at infinity
    if (!(best < INFINITY)) bi = 0x7fffffff;
  }
}

// T = sum_j w_j * tfs_j  (einsum 'bpn,bnij->bpij', deformer.py:85), rows 0..2 and the (3,3) entry
__device__ __forceinline__ void blend_tf(const float* __restrict__ w, const float* __restrict__ tfs, float T[12],
                                         float& s) {
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = 0.f;
  s = 0.f;
  const float4* w4 = reinterpret_cast<const float4*>(w);     // rows of 24 floats are 16-byte aligned
#pragma unroll
  for (int j4 = 0; j4 < MP_NUM_JOINTS / 4; ++j4) {
    float4 ww = __ldg(w4 + j4);
    float wv[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float wj = wv[u];
      if (wj == 0.f) continue;   // adding 0*finite leaves the fp32 sum unchanged
      const float* t = tfs + 16 * (4 * j4 + u);
#pragma unroll
      for (int k = 0; k < 12; ++k) T[k] = fmaf(wj, __ldg(&t[k]), T[k]);
      s = fmaf(wj, __ldg(&t[15]), s);
    }
  }
}

__device__ __forceinline__ void inv3(const float* A, int ld, float* I) {
  // adjugate / determinant of the 3x3 at A (row stride ld)
  float a = A[0], b = A[1], c = A[2], d = A[ld], e = A[ld + 1], f = A[ld + 2], g = A[2 * ld], h = A[2 * ld + 1],
        i = A[2 * ld + 2];
  float c00 = e * i - f * h, c01 = -(d * i - f * g), c02 = d * h - e * g;
  float det = a * c00 + b * c01 + c * c02;
  float r = 1.0f / det;
  I[0] = c00 * r;
  I[1] = -(b * i - c * h) * r;
  I[2] = (b * f - c * e) * r;
  I[3] = c01 * r;
  I[4] = (a * i - c * g) * r;
  I[5] = -(a * f - c * d) * r;
  I[6] = c02 * r;
  I[7] = -(a * h - b * g) * r;
  I[8] = (a * e - b * d) * r;
}

// Per-frame table: the blended transform only depends on the VERTEX whose weights are used (K = 1, weights
// detached, deformer.py:37-50), so T_v = sum_j W[v][j] tfs_j and its closed-form inverse are computed once per
// vertex (6890) instead of once per sample point (millions): x_c = I_v (x - t_v / s_v), J^-1 = I_v.
__global__ void vertex_tf_kernel(const float* __restrict__ weights, const float* __restrict__ tfs, int V,
                                 float4* __restrict__ vert_tf) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float T[12], s;
  blend_tf(weights + (size_t)v * MP_NUM_JOINTS, tfs, T, s);
  float I[9];
  inv3(T, 4, I);
  float is = 1.0f / s;
  vert_tf[3 * (size_t)v + 0] = make_float4(I[0], I[1], I[2], T[3] * is);
  vert_tf[3 * (size_t)v + 1] = make_float4(I[3], I[4], I[5], T[7] * is);
  vert_tf[3 * (size_t)v + 2] = make_float4(I[6], I[7], I[8], T[11] * is);
}

// ---- optional root finder (SURVEY.md §8 row f4) --------------------------------------------------------------
// The closed-form inverse picks the skinning weights of the nearest POSED vertex, the forward map
// (deformer.py:31-35, forward_skinning) those of the nearest CANONICAL vertex of x_c; where the two disagree
// forward_skinning(x_c) != x_d.  Broyden's method on g(x_c) = forward_skinning(x_c) - x_d, started from the
// closed-form inverse with J^-1 = the inverse blended 3x3 at the start point (the weights are detached, so that IS the
// Jacobian inside a Voronoi cell), rank-one "good Broyden" updates of J^-1 (Sherman-Morrison), lowest-residual
// iterate kept.  The reference has no such step (SURVEY.md fact 0-1); parity is against oracle/port.py:deform_broyden.
// Returns false, leaving f untouched, when x has no nearest vertex (a non-finite coordinate, or every fp32 squared
// distance overflows): such a point has no skinning weights.
__device__ __forceinline__ bool skin_forward_point(const Body& b, const GridHeader& gc, const float x[3], float f[3],
                                                   int& vi) {
  float d2;
  nearest_vertex(gc, b.cano_cell_start, b.cano_sorted, b.V, x[0], x[1], x[2], true, d2, vi);
  if (vi == 0x7fffffff) return false;
  float T[12], s;
  blend_tf(b.weights + (size_t)vi * MP_NUM_JOINTS, b.tfs, T, s);
  f[0] = fmaf(T[0], x[0], fmaf(T[1], x[1], fmaf(T[2], x[2], T[3])));
  f[1] = fmaf(T[4], x[0], fmaf(T[5], x[1], fmaf(T[6], x[2], T[7])));
  f[2] = fmaf(T[8], x[0], fmaf(T[9], x[1], fmaf(T[10], x[2], T[11])));
  return true;
}

// An iterate without a nearest vertex ends the iteration: the best iterate so far and its residual are returned and
// `steps` counts the steps taken.  A start without one is returned as it is, with a NaN residual and no step.
__device__ __noinline__ void broyden_refine(const Body& b, float px, float py, float pz, int max_steps, float thr,
                                            float xc[3], float& resid, int& steps) {
  const GridHeader gc = *b.cano_hdr;
  float x[3] = {xc[0], xc[1], xc[2]}, f[3], g[3];
  int vi;
  steps = 0;
  if (!skin_forward_point(b, gc, x, f, vi)) {
    resid = __int_as_float(0x7fffffff);
    return;
  }
  g[0] = f[0] - px;
  g[1] = f[1] - py;
  g[2] = f[2] - pz;
  float Ji[9];
  {
    const float4 r0 = __ldg(&b.vert_tf[3 * (size_t)vi]), r1 = __ldg(&b.vert_tf[3 * (size_t)vi + 1]),
                 r2 = __ldg(&b.vert_tf[3 * (size_t)vi + 2]);
    Ji[0] = r0.x; Ji[1] = r0.y; Ji[2] = r0.z; Ji[3] = r1.x; Ji[4] = r1.y; Ji[5] = r1.z; Ji[6] = r2.x; Ji[7] = r2.y;
    Ji[8] = r2.z;
  }
  float best = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  for (int k = 0; k < max_steps && best >= thr; ++k) {
    float dx[3], gn[3], dg[3], u[3], vt[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) dx[r] = -(Ji[3 * r] * g[0] + Ji[3 * r + 1] * g[1] + Ji[3 * r + 2] * g[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) x[r] += dx[r];
    if (!skin_forward_point(b, gc, x, f, vi)) {
      steps = k + 1;
      break;
    }
    gn[0] = f[0] - px;
    gn[1] = f[1] - py;
    gn[2] = f[2] - pz;
#pragma unroll
    for (int r = 0; r < 3; ++r) dg[r] = gn[r] - g[r];
#pragma unroll
    for (int r = 0; r < 3; ++r) u[r] = Ji[3 * r] * dg[0] + Ji[3 * r + 1] * dg[1] + Ji[3 * r + 2] * dg[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) vt[c] = dx[0] * Ji[c] + dx[1] * Ji[3 + c] + dx[2] * Ji[6 + c];
    float den = dx[0] * u[0] + dx[1] * u[1] + dx[2] * u[2];
    if (fabsf(den) > 1e-20f) {
      float id = 1.0f / den;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) Ji[3 * r + c] += (dx[r] - u[r]) * vt[c] * id;
    }
    g[0] = gn[0];
    g[1] = gn[1];
    g[2] = gn[2];
    float rn = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
    steps = k + 1;
    if (rn < best) {
      best = rn;
      xc[0] = x[0];
      xc[1] = x[1];
      xc[2] = x[2];
    }
  }
  resid = best;
}

// Shared per-point routine of the inverse deformer.  ROOT = false is the reference's path; the ROOT = true
// instantiations exist so that the optional refinement costs the default kernels neither registers nor stack.
// Returns the vertex whose weights were used (0x7fffffff: none within reach, x_c = x).
template <bool ROOT = false>
__device__ __forceinline__ int deform_inverse_point(const Body& b, const GridHeader& g, float px, float py, float pz,
                                                     bool exact_far, float xc[3], bool& outlier) {
  float d2;
  int vi;
  nearest_vertex(g, b.posed_cell_start, b.posed_sorted, b.V, px, py, pz, exact_far, d2, vi);
  // deformer.py:41-49: d2 = clamp(d2, max=4); outlier = sqrt(d2) > 0.1
  float dc = fminf(d2, 4.f);
  outlier = sqrtf(dc) > 0.1f;
  if (vi == 0x7fffffff) {   // nothing within reach of the grid (and no full scan requested)
    outlier = true;
    xc[0] = px;
    xc[1] = py;
    xc[2] = pz;
    return vi;
  }
  // [A t; 0 s]^-1 [x;1] = A^-1 (x - t/s), from the per-vertex table
  const float4 r0 = __ldg(&b.vert_tf[3 * (size_t)vi]), r1 = __ldg(&b.vert_tf[3 * (size_t)vi + 1]),
               r2 = __ldg(&b.vert_tf[3 * (size_t)vi + 2]);
  float qx = px - r0.w, qy = py - r1.w, qz = pz - r2.w;
  xc[0] = r0.x * qx + r0.y * qy + r0.z * qz;
  xc[1] = r1.x * qx + r1.y * qy + r1.z * qz;
  xc[2] = r2.x * qx + r2.y * qy + r2.z * qz;
  if (ROOT && b.root_steps > 0 && !outlier) {   // non-default (row f4); outliers keep the closed form (their SDF is forced to 4)
    float resid;
    int steps;
    broyden_refine(b, px, py, pz, b.root_steps, b.root_thr, xc, resid, steps);
  }
  return vi;
}

__global__ void deform_broyden_kernel(Body b, const float* __restrict__ x, int N, int max_steps, float thr,
                                      float* __restrict__ x_c, float* __restrict__ residual,
                                      uint8_t* __restrict__ converged, uint8_t* __restrict__ outlier,
                                      int* __restrict__ steps_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  GridHeader g = *b.posed_hdr;
  float xc[3];
  bool o;
  float px = x[3 * i], py = x[3 * i + 1], pz = x[3 * i + 2];
  deform_inverse_point<false>(b, g, px, py, pz, true, xc, o);
  float resid;
  int steps;
  broyden_refine(b, px, py, pz, max_steps, thr, xc, resid, steps);
  x_c[3 * i] = xc[0];
  x_c[3 * i + 1] = xc[1];
  x_c[3 * i + 2] = xc[2];
  if (residual) residual[i] = resid;
  if (converged) converged[i] = resid < thr ? 1 : 0;
  if (outlier) outlier[i] = o ? 1 : 0;
  if (steps_out) steps_out[i] = steps;
}

template <bool ROOT>
__global__ void deform_inverse_kernel(Body b, const float* __restrict__ x, int N, float* __restrict__ x_c,
                                      uint8_t* __restrict__ outlier, int exact_far) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  GridHeader g = *b.posed_hdr;
  float xc[3];
  bool o;
  deform_inverse_point<ROOT>(b, g, x[3 * i], x[3 * i + 1], x[3 * i + 2], exact_far != 0, xc, o);
  x_c[3 * i] = xc[0];
  x_c[3 * i + 1] = xc[1];
  x_c[3 * i + 2] = xc[2];
  if (outlier) outlier[i] = o ? 1 : 0;
}

// Sampler / main-pass variant: points are generated from rays on the fly
//   points = cam_loc + z * ray_dirs        (ray_sampler.py:82, multiply.py:295)
// `slot[i]` gives where the SDF of point i has to land; outliers get sdf = 4 right here
// (multiply.py:142-143) and everything else is appended to the compact work list of the MLP.
template <bool ROOT>
__global__ void deform_rays_kernel(Body b, const float* __restrict__ dirs, const float* __restrict__ cam,
                                   const float* __restrict__ z, int z_stride, const int* __restrict__ zpos,
                                   int zpos_stride, int n_per_ray, int R, int prune, float* __restrict__ sdf_out,
                                   int sdf_stride, float* __restrict__ xc_list, int* __restrict__ slot_list,
                                   int* __restrict__ count, uint8_t* __restrict__ outlier_out,
                                   const int* __restrict__ active, const int* __restrict__ R_dev) {
  if (active && *active == 0) return;
  if (R_dev) R = min(R, *R_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = R * n_per_ray;
  bool valid = i < total;
  bool keep = false;
  float xc[3] = {0.f, 0.f, 0.f};
  int slot = 0;
  if (valid) {
    int r = i / n_per_ray, j = i - r * n_per_ray;
    int col = zpos ? zpos[(size_t)r * zpos_stride + j] : j;
    float zz = z[(size_t)r * z_stride + col];
    float px = __fadd_rn(cam[3 * r], __fmul_rn(zz, dirs[3 * r]));
    float py = __fadd_rn(cam[3 * r + 1], __fmul_rn(zz, dirs[3 * r + 1]));
    float pz = __fadd_rn(cam[3 * r + 2], __fmul_rn(zz, dirs[3 * r + 2]));
    GridHeader g = *b.posed_hdr;
    bool o;
    deform_inverse_point<ROOT>(b, g, px, py, pz, prune == 0, xc, o);
    slot = r * sdf_stride + col;
    if (outlier_out) outlier_out[slot] = o ? 1 : 0;
    if (o && prune) {
      sdf_out[slot] = 4.0f;
    } else {
      keep = true;
    }
  }
  // warp-aggregated append
  unsigned m = __ballot_sync(0xffffffffu, keep);
  int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && m) base = atomicAdd(count, __popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (keep) {
    int p = base + __popc(m & ((1u << lane) - 1));
    xc_list[3 * p] = xc[0];
    xc_list[3 * p + 1] = xc[1];
    xc_list[3 * p + 2] = xc[2];
    slot_list[p] = slot;
  }
}

// forward skinning Jacobian: weights from the nearest CANONICAL vertex (deformer.py:31-35);
// J = (sum_j w_j tfs_j)[:3,:3] because the weights are detached (deformer.py:47).
__global__ void deform_forward_jac_kernel(Body b, const float* __restrict__ x_c, int N, const int* __restrict__ n_dev,
                                          float* __restrict__ x_d, float* __restrict__ Jinv, int jstride) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? *n_dev : N;
  if (i >= n) return;
  GridHeader g = *b.cano_hdr;
  float px = x_c[3 * i], py = x_c[3 * i + 1], pz = x_c[3 * i + 2];
  float d2;
  int vi;
  nearest_vertex(g, b.cano_cell_start, b.cano_sorted, b.V, px, py, pz, true, d2, vi);
  const bool none = vi == 0x7fffffff;   // no nearest vertex (non-finite or overflowing x_c): x_d and J^-1 are NaN
  const float nan = __int_as_float(0x7fffffff);
  if (x_d) {
    if (none) {
      x_d[3 * i] = x_d[3 * i + 1] = x_d[3 * i + 2] = nan;
    } else {
      float T[12], s;
      blend_tf(b.weights + (size_t)vi * MP_NUM_JOINTS, b.tfs, T, s);
      x_d[3 * i] = T[0] * px + T[1] * py + T[2] * pz + T[3];
      x_d[3 * i + 1] = T[4] * px + T[5] * py + T[6] * pz + T[7];
      x_d[3 * i + 2] = T[8] * px + T[9] * py + T[10] * pz + T[11];
    }
  }
  if (Jinv) {
    const float4 nan4 = make_float4(nan, nan, nan, nan);
    const float4 r0 = none ? nan4 : __ldg(&b.vert_tf[3 * (size_t)vi]),
                 r1 = none ? nan4 : __ldg(&b.vert_tf[3 * (size_t)vi + 1]),
                 r2 = none ? nan4 : __ldg(&b.vert_tf[3 * (size_t)vi + 2]);
    if (jstride == 12) {   // padded rows: three 128-bit stores
      float4* o = reinterpret_cast<float4*>(Jinv + 12 * (size_t)i);
      o[0] = make_float4(r0.x, r0.y, r0.z, r1.x);
      o[1] = make_float4(r1.y, r1.z, r2.x, r2.y);
      o[2] = make_float4(r2.z, 0.f, 0.f, 0.f);
    } else {
      float* o = Jinv + 9 * (size_t)i;
      o[0] = r0.x; o[1] = r0.y; o[2] = r0.z; o[3] = r1.x; o[4] = r1.y; o[5] = r1.z; o[6] = r2.x; o[7] = r2.y; o[8] = r2.z;
    }
  }
}

// ---- backward (VJPs of mp_deform_inverse and mp_deform_forward_jac) ------------------------------------------------
// Every point's dL/d(blended transform) goes to the bones with its (detached) vertex weights: d_tfs_j = sum_i w_ij dA_i.
// A fixed grid of CTAs walks the points in a fixed order; per warp the 32 points' terms are added by shuffles and lane 0
// accumulates them in fp64 shared memory; each CTA leaves one partial [24,16] and bone_grad_final_kernel adds the
// partials in CTA order.  No atomics: reruns are bit-identical.
constexpr int kBgThreads = 256, kBgMaxBlocks = 1024, kBoneGrad = MP_NUM_JOINTS * 16;

static int bone_grad_blocks(int N) { return N > 0 ? std::min(div_up(N, kBgThreads), kBgMaxBlocks) : 0; }

// acc[16 j + 4 r + c] += sum over the warp's lanes of w_j dA[4 r + c], rows r < NROW; w == nullptr: the lane adds nothing.
// Every lane of the warp must call it.
template <int NROW>
__device__ __forceinline__ void bone_grad_warp(const float* __restrict__ w, const float dA[16], double* acc, int lane) {
  const float4* w4 = reinterpret_cast<const float4*>(w);
#pragma unroll 1
  for (int j4 = 0; j4 < MP_NUM_JOINTS / 4; ++j4) {
    float4 ww = w ? __ldg(w4 + j4) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float wv[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float wj = wv[u];
      if (!__any_sync(0xffffffffu, wj != 0.f)) continue;
      double* a = acc + 16 * (4 * j4 + u);
#pragma unroll
      for (int k = 0; k < 4 * NROW; ++k) {
        const float t = warp_sum(wj * dA[k]);
        if (lane == 0) a[k] += (double)t;
      }
    }
  }
}

__device__ __forceinline__ void bone_grad_zero(double (*acc)[kBoneGrad]) {
  for (int i = threadIdx.x; i < (kBgThreads / 32) * kBoneGrad; i += blockDim.x) acc[i / kBoneGrad][i % kBoneGrad] = 0.0;
  __syncthreads();
}

__device__ __forceinline__ void bone_grad_store(double (*acc)[kBoneGrad], double* __restrict__ partials) {
  __syncthreads();
  for (int i = threadIdx.x; i < kBoneGrad; i += blockDim.x) {
    double t = acc[0][i];
    for (int q = 1; q < kBgThreads / 32; ++q) t += acc[q][i];
    partials[(size_t)blockIdx.x * kBoneGrad + i] = t;
  }
}

__global__ void __launch_bounds__(kBoneGrad) bone_grad_final_kernel(const double* __restrict__ partials, int nblk,
                                                                    float* __restrict__ d_tfs) {
  const int i = threadIdx.x;
  double t = 0.0;
  for (int q = 0; q < nblk; ++q) t += partials[(size_t)q * kBoneGrad + i];
  d_tfs[i] = (float)t;
}

// x_c = (A^-1 [x;1])[:3] with A = sum_j w_j tfs_j = [M t; 0 s]: with u = M^-T g and tau = t / s (the forward's table),
// dL/dA = -[u ; -tau.u] [x_c ; 1]^T and dL/dx = u.  All four rows go to the bones, as torch's inverse backward gives them.
__global__ void __launch_bounds__(kBgThreads) deform_inverse_backward_kernel(Body b, const float* __restrict__ x, int N,
                                                                             int exact_far, const float* __restrict__ d_xc,
                                                                             float* __restrict__ d_x,
                                                                             float* __restrict__ x_c_out,
                                                                             double* __restrict__ partials) {
  __shared__ double acc[kBgThreads / 32][kBoneGrad];
  bone_grad_zero(acc);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const GridHeader g = *b.posed_hdr;
  for (int base = blockIdx.x * kBgThreads; base < N; base += gridDim.x * kBgThreads) {
    const int i = base + threadIdx.x;
    float dA[16];                       // zero for lanes without a point or a vertex: bone_grad_warp multiplies by w = 0
#pragma unroll
    for (int k = 0; k < 16; ++k) dA[k] = 0.f;
    const float* w = nullptr;
    if (i < N) {
      const float px = x[3 * i], py = x[3 * i + 1], pz = x[3 * i + 2];
      float xc[3];
      bool o;
      const int vi = deform_inverse_point<false>(b, g, px, py, pz, exact_far != 0, xc, o);
      const float gx = d_xc[3 * i], gy = d_xc[3 * i + 1], gz = d_xc[3 * i + 2];
      float u[3] = {gx, gy, gz};        // no vertex within reach: x_c = x
      if (vi != 0x7fffffff) {
        const float4 r0 = __ldg(&b.vert_tf[3 * (size_t)vi]), r1 = __ldg(&b.vert_tf[3 * (size_t)vi + 1]),
                     r2 = __ldg(&b.vert_tf[3 * (size_t)vi + 2]);
        u[0] = r0.x * gx + r1.x * gy + r2.x * gz;
        u[1] = r0.y * gx + r1.y * gy + r2.y * gz;
        u[2] = r0.z * gx + r1.z * gy + r2.z * gz;
        const float tu = r0.w * u[0] + r1.w * u[1] + r2.w * u[2];
        const float a[4] = {-u[0], -u[1], -u[2], tu}, bb[4] = {xc[0], xc[1], xc[2], 1.f};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) dA[4 * r + c] = a[r] * bb[c];
        w = b.weights + (size_t)vi * MP_NUM_JOINTS;
      }
      if (d_x) {
        d_x[3 * i] = u[0];
        d_x[3 * i + 1] = u[1];
        d_x[3 * i + 2] = u[2];
      }
      if (x_c_out) {
        x_c_out[3 * i] = xc[0];
        x_c_out[3 * i + 1] = xc[1];
        x_c_out[3 * i + 2] = xc[2];
      }
    }
    bone_grad_warp<4>(w, dA, acc[warp], lane);
  }
  bone_grad_store(acc, partials);
}

// x_d = M x_c + t and Jinv = M^-1 with M, t blended with the weights of the nearest CANONICAL vertex (the forward's
// search and table): dL/dM = -Jinv^T d_Jinv Jinv^T, dL/dT[:3,:] += d_x_d [x_c;1]^T, dL/dx_c = M^T d_x_d (the weights are
// piecewise constant, so Jinv contributes nothing to it).  The bottom row of d_tfs is 0.
__global__ void __launch_bounds__(kBgThreads) deform_forward_jac_backward_kernel(
    Body b, const float* __restrict__ x_c, int N, const float* __restrict__ d_xd, const float* __restrict__ d_Jinv,
    float* __restrict__ d_xc, double* __restrict__ partials) {
  __shared__ double acc[kBgThreads / 32][kBoneGrad];
  bone_grad_zero(acc);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const GridHeader g = *b.cano_hdr;
  for (int base = blockIdx.x * kBgThreads; base < N; base += gridDim.x * kBgThreads) {
    const int i = base + threadIdx.x;
    float dA[16];                       // zero for lanes without a point or a vertex: bone_grad_warp multiplies by w = 0
#pragma unroll
    for (int k = 0; k < 16; ++k) dA[k] = 0.f;
    const float* w = nullptr;
    if (i < N) {
      const float px = x_c[3 * i], py = x_c[3 * i + 1], pz = x_c[3 * i + 2];
      float d2;
      int vi;
      nearest_vertex(g, b.cano_cell_start, b.cano_sorted, b.V, px, py, pz, true, d2, vi);
      if (vi == 0x7fffffff) {   // no nearest vertex: d_x_c is NaN and nothing goes to the bones (w stays null)
        if (d_xc) d_xc[3 * i] = d_xc[3 * i + 1] = d_xc[3 * i + 2] = __int_as_float(0x7fffffff);
      } else {
        w = b.weights + (size_t)vi * MP_NUM_JOINTS;
        float dxc[3] = {0.f, 0.f, 0.f};
        if (d_xd) {
          const float gx = d_xd[3 * i], gy = d_xd[3 * i + 1], gz = d_xd[3 * i + 2];
          const float gg[3] = {gx, gy, gz}, xh[4] = {px, py, pz, 1.f};
          float T[12], s;
          blend_tf(w, b.tfs, T, s);
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) dA[4 * r + c] = gg[r] * xh[c];
#pragma unroll
          for (int c = 0; c < 3; ++c) dxc[c] = T[c] * gx + T[4 + c] * gy + T[8 + c] * gz;
        }
        if (d_Jinv) {
          const float4 r0 = __ldg(&b.vert_tf[3 * (size_t)vi]), r1 = __ldg(&b.vert_tf[3 * (size_t)vi + 1]),
                       r2 = __ldg(&b.vert_tf[3 * (size_t)vi + 2]);
          const float I[9] = {r0.x, r0.y, r0.z, r1.x, r1.y, r1.z, r2.x, r2.y, r2.z};
          const float* dJ = d_Jinv + 9 * (size_t)i;
          float H[9];   // d_Jinv Jinv^T
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) H[3 * r + c] = dJ[3 * r] * I[3 * c] + dJ[3 * r + 1] * I[3 * c + 1] + dJ[3 * r + 2] * I[3 * c + 2];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) dA[4 * r + c] -= I[r] * H[c] + I[3 + r] * H[3 + c] + I[6 + r] * H[6 + c];
        }
        if (d_xc) {
          d_xc[3 * i] = dxc[0];
          d_xc[3 * i + 1] = dxc[1];
          d_xc[3 * i + 2] = dxc[2];
        }
      }
    }
    bone_grad_warp<3>(w, dA, acc[warp], lane);
  }
  bone_grad_store(acc, partials);
}

int body_build_grid(const float* verts, int V, float cell, int R0, GridHeader* hdr, int* cell_start, float4* sorted,
                    int* scratch, cudaStream_t st) {
  grid_build_kernel<<<1, 1024, 0, st>>>(verts, V, cell, R0, hdr, cell_start, sorted, scratch);
  MP_LAUNCH_CHECK();
  return 0;
}

int launch_deform_rays(const Body& b, const float* dirs, const float* cam, const float* z, int z_stride,
                       const int* zpos, int zpos_stride, int n_per_ray, int R, int prune, float* sdf_out,
                       int sdf_stride, float* xc_list, int* slot_list, int* count, uint8_t* outlier_out,
                       const int* active, cudaStream_t st, const int* R_dev) {
  int total = R * n_per_ray;
  if (total <= 0) return 0;
  if (b.root_steps > 0)
    deform_rays_kernel<true><<<div_up(total, 128), 128, 0, st>>>(b, dirs, cam, z, z_stride, zpos, zpos_stride,
                                                               n_per_ray, R, prune, sdf_out, sdf_stride, xc_list,
                                                               slot_list, count, outlier_out, active, R_dev);
  else
    deform_rays_kernel<false><<<div_up(total, 128), 128, 0, st>>>(b, dirs, cam, z, z_stride, zpos, zpos_stride,
                                                                n_per_ray, R, prune, sdf_out, sdf_stride, xc_list,
                                                                slot_list, count, outlier_out, active, R_dev);
  MP_LAUNCH_CHECK();
  return 0;
}

int launch_forward_jac(const Body& b, const float* x_c, int N, const int* n_dev, float* x_d, float* Jinv,
                       int jstride, cudaStream_t st) {
  if (N <= 0) return 0;
  deform_forward_jac_kernel<<<div_up(N, 128), 128, 0, st>>>(b, x_c, N, n_dev, x_d, Jinv, jstride);
  MP_LAUNCH_CHECK();
  return 0;
}

// The body's two vertex grids and per-vertex transforms, in its caller's storage.
static void body_carve(Arena& a, int V, Body& b) {
  b.cano_hdr = a.take<GridHeader>(1);
  b.posed_hdr = a.take<GridHeader>(1);
  b.cano_cell_start = a.take<int>(kMaxCells + 1);
  b.posed_cell_start = a.take<int>(kMaxCells + 1);
  b.cano_sorted = a.take<float4>(V);
  b.posed_sorted = a.take<float4>(V);
  b.scratch = a.take<int>(kMaxCells + 8);
  b.vert_tf = a.take<float4>((size_t)V * 3);
}

// per-CTA fp64 partials of the bone gradient
static double* deform_backward_carve(Arena& a, int N) {
  return a.take<double>((size_t)bone_grad_blocks(N) * kBoneGrad);
}

}  // namespace mp

extern "C" {

size_t mp_body_bytes(int V) {
  mp::Arena a;
  mp::Body b{};
  mp::body_carve(a, V > 0 ? V : 0, b);
  return a.off;
}

int mp_body_create(const float* verts_cano, const float* weights, int V, float cano_cell, void* storage,
                   size_t storage_bytes, mp_body_t** out, void* stream) {
  MP_REQUIRE(verts_cano && weights && storage && out, "mp_body_create: null argument");
  MP_REQUIRE(V > 0, "mp_body_create: V must be positive");
  mp::Arena a(storage, storage_bytes);
  mp::Body b{};
  mp::body_carve(a, V, b);
  MP_TRY(a.fits("mp_body_create", "storage"));
  b.V = V;
  b.weights = weights;
  b.verts_cano = verts_cano;
  b.verts_posed = nullptr;
  b.tfs = nullptr;
  b.root_steps = 0;
  b.root_thr = 1e-5f;
  b.cano_cell = cano_cell;
  mp_body* h = new mp_body();
  h->b = b;
  int r = mp::body_build_grid(verts_cano, V, cano_cell * 0.5f, 2, b.cano_hdr, b.cano_cell_start, b.cano_sorted, b.scratch,
                              (cudaStream_t)stream);
  if (r) {
    delete h;
    return r;
  }
  *out = h;
  return 0;
}

void mp_body_free(mp_body_t* b) { delete b; }

int mp_body_set_pose(mp_body_t* h, const float* verts_posed, const float* tfs, void* stream) {
  MP_REQUIRE(h && verts_posed && tfs, "mp_body_set_pose: null argument");
  mp::Body& b = h->b;
  b.verts_posed = verts_posed;
  b.tfs = tfs;
  mp::vertex_tf_kernel<<<mp::div_up(b.V, 128), 128, 0, (cudaStream_t)stream>>>(b.weights, tfs, b.V, b.vert_tf);
  MP_LAUNCH_CHECK();
  // two cells of 0.05005 cover the 0.1 outlier radius of deformer.py:49 (see nearest_vertex); the finer cells let
  // the distance pruning of scan_block skip most of the block
  return mp::body_build_grid(verts_posed, b.V, 0.05005f, 2, b.posed_hdr, b.posed_cell_start, b.posed_sorted, b.scratch,
                             (cudaStream_t)stream);
}

int mp_deform_inverse(mp_body_t* h, const float* x, int N, float* x_c, uint8_t* outlier, int exact_far,
                      void* stream) {
  MP_REQUIRE(h && h->b.tfs, "mp_deform_inverse: body has no pose (call mp_body_set_pose)");
  if (N <= 0) return 0;   // deformer.py:20
  if (h->b.root_steps > 0)
    mp::deform_inverse_kernel<true><<<mp::div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(h->b, x, N, x_c, outlier,
                                                                                           exact_far);
  else
    mp::deform_inverse_kernel<false><<<mp::div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(h->b, x, N, x_c, outlier,
                                                                                            exact_far);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_body_set_root_finder(mp_body_t* h, int max_steps, float cvg_threshold) {
  MP_REQUIRE(h, "mp_body_set_root_finder: null body");
  MP_REQUIRE(max_steps >= 0 && max_steps <= 64, "mp_body_set_root_finder: max_steps %d outside [0, 64]", max_steps);
  MP_REQUIRE(cvg_threshold > 0.f, "mp_body_set_root_finder: threshold must be positive");
  h->b.root_steps = max_steps;
  h->b.root_thr = cvg_threshold;
  return 0;
}

int mp_deform_broyden(mp_body_t* h, const float* x, int N, int max_steps, float cvg_threshold, float* x_c,
                      float* residual, uint8_t* converged, uint8_t* outlier, int* steps, void* stream) {
  MP_REQUIRE(h && h->b.tfs, "mp_deform_broyden: body has no pose (call mp_body_set_pose)");
  MP_REQUIRE(max_steps >= 0 && max_steps <= 64 && cvg_threshold > 0.f, "mp_deform_broyden: bad iteration limits");
  if (N <= 0) return 0;   // nothing is read or written: every buffer may be null
  MP_REQUIRE(x && x_c, "mp_deform_broyden: null input or output");
  mp::deform_broyden_kernel<<<mp::div_up(N, 128), 128, 0, (cudaStream_t)stream>>>(
      h->b, x, N, max_steps, cvg_threshold, x_c, residual, converged, outlier, steps);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_deform_forward_jac(mp_body_t* h, const float* x_c, int N, float* x_d, float* Jinv, void* stream) {
  MP_REQUIRE(h && h->b.tfs, "mp_deform_forward_jac: body has no pose (call mp_body_set_pose)");
  return mp::launch_forward_jac(h->b, x_c, N, nullptr, x_d, Jinv, 9, (cudaStream_t)stream);
}

size_t mp_deform_backward_workspace_bytes(int N) {
  mp::Arena a;
  mp::deform_backward_carve(a, N);
  return a.off;
}

int mp_deform_inverse_backward(mp_body_t* h, const float* x, int N, int exact_far, const float* d_x_c, float* d_tfs,
                               float* d_x, float* x_c, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(h && h->b.tfs, "mp_deform_inverse_backward: body has no pose (call mp_body_set_pose)");
  MP_REQUIRE(h->b.root_steps == 0,
             "mp_deform_inverse_backward: the body's root finder is on; only the closed-form inverse has a backward");
  MP_REQUIRE(d_tfs && N >= 0 && (N == 0 || (x && d_x_c)), "mp_deform_inverse_backward: null argument");
  mp::Arena a(workspace, workspace_bytes);
  double* partials = mp::deform_backward_carve(a, N);
  MP_TRY(a.fits("mp_deform_inverse_backward"));
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = mp::bone_grad_blocks(N);
  if (nblk) {
    mp::deform_inverse_backward_kernel<<<nblk, mp::kBgThreads, 0, st>>>(h->b, x, N, exact_far, d_x_c, d_x, x_c,
                                                                       partials);
    MP_LAUNCH_CHECK();
  }
  mp::bone_grad_final_kernel<<<1, mp::kBoneGrad, 0, st>>>(partials, nblk, d_tfs);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_deform_forward_jac_backward(mp_body_t* h, const float* x_c, int N, const float* d_x_d, const float* d_Jinv,
                                   float* d_tfs, float* d_x_c, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(h && h->b.tfs, "mp_deform_forward_jac_backward: body has no pose (call mp_body_set_pose)");
  MP_REQUIRE(d_tfs && N >= 0 && (N == 0 || x_c), "mp_deform_forward_jac_backward: null argument");
  mp::Arena a(workspace, workspace_bytes);
  double* partials = mp::deform_backward_carve(a, N);
  MP_TRY(a.fits("mp_deform_forward_jac_backward"));
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = mp::bone_grad_blocks(N);
  if (nblk) {
    mp::deform_forward_jac_backward_kernel<<<nblk, mp::kBgThreads, 0, st>>>(h->b, x_c, N, d_x_d, d_Jinv, d_x_c, partials);
    MP_LAUNCH_CHECK();
  }
  mp::bone_grad_final_kernel<<<1, mp::kBoneGrad, 0, st>>>(partials, nblk, d_tfs);
  MP_LAUNCH_CHECK();
  return 0;
}
}
