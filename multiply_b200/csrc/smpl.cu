// SMPL body model server: shape/pose blend shapes, forward kinematics, linear blend skinning.
//   reference: /root/reference/code/lib/model/smpl.py:50-95 (SMPLServer.forward)
//              -> lib/smpl/body_models.py:278-364 (SMPL.forward) -> lib/smpl/lbs.py:136-229 (lbs),
//              :276-307 (batch_rodrigues), :323-378 (batch_rigid_transform)
// The reference issues ~100 tiny ATen kernels per person per forward (launch-bound, SURVEY §8a-3); here it is two
// launches: one CTA does the 10-coefficient shape blend, the joint regression, Rodrigues and the 24-joint
// kinematic chain (plus SMPLServer's scale / translation / canonical-inverse), then a grid-wide kernel does the
// 207-term pose blend and the skinning per vertex with coalesced reads of `posedirs`.
#include "common.cuh"

namespace mp {

struct Smpl {
  int V;
  const float* v_template;   // [V,3]
  const float* shapedirs;    // [V,3,10]
  const float* posedirs;     // [207, V*3]
  const float* J_regressor;  // [24,V]
  const float* lbs_weights;  // [V,24]
  int parents[MP_NUM_JOINTS];
  // storage
  float* v_shaped;           // [V,3]
  float* pose_feature;       // [207]
  float* A_abs;              // [24,16] scaled/translated bone transforms w.r.t. theta = 0
  float* tfs_c_inv;          // [24,16]
  float* verts_c;            // [V,3]
  float* tmp_tfs;            // [24,16]
  float* J_t;                // [24,3]     J_regressor @ v_template           (precomputed at creation)
  float* J_s;                // [24,3,10]  J_regressor @ shapedirs: J(betas) = J_t + J_s . betas
};

__device__ __forceinline__ void mat4_mul(const float* a, const float* b, float* c) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) s = fmaf(a[4 * i + k], b[4 * k + j], s);
      c[4 * i + j] = s;
    }
}

// Joint regression is linear in the shape coefficients: J = Jr @ (v_template + shapedirs . betas) (lbs.py:184-188) =
// Jr @ v_template + (Jr @ shapedirs) . betas.  The two regressed tensors are computed once per model (one warp per joint),
// which takes the 24 x V regression -- 58 of the SMPL server's 90 us per call -- out of the per-frame path.
__global__ void __launch_bounds__(1024) smpl_jreg_kernel(Smpl m) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp >= MP_NUM_JOINTS) return;
  const float* jr = m.J_regressor + (size_t)warp * m.V;
  float acc[33];
#pragma unroll
  for (int k = 0; k < 33; ++k) acc[k] = 0.f;
  for (int v = lane; v < m.V; v += 32) {
    const float w = jr[v];
    if (w == 0.f) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      acc[a] = fmaf(w, m.v_template[3 * v + a], acc[a]);
      const float* sd = m.shapedirs + ((size_t)3 * v + a) * 10;
#pragma unroll
      for (int l = 0; l < 10; ++l) acc[3 + a * 10 + l] = fmaf(w, sd[l], acc[3 + a * 10 + l]);
    }
  }
#pragma unroll
  for (int k = 0; k < 33; ++k) acc[k] = warp_sum(acc[k]);
  if (lane == 0) {
    for (int a = 0; a < 3; ++a) {
      m.J_t[warp * 3 + a] = acc[a];
      for (int l = 0; l < 10; ++l) m.J_s[(warp * 3 + a) * 10 + l] = acc[3 + a * 10 + l];
    }
  }
}

// one CTA of 1024 threads
__global__ void __launch_bounds__(1024) smpl_pose_kernel(Smpl m, const float* __restrict__ scale_p,
                                                         const float* __restrict__ transl, const float* __restrict__ thetas,
                                                         const float* __restrict__ betas, int absolute,
                                                         float* __restrict__ tfs_out) {
  __shared__ float sJ[MP_NUM_JOINTS][3];
  __shared__ float sR[MP_NUM_JOINTS][9];
  __shared__ float sG[MP_NUM_JOINTS][16];
  __shared__ float sb[10];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 10) sb[tid] = betas[tid];
  __syncthreads();
  // J = J_regressor @ v_shaped (lbs.py:188, :232-249) through the precomputed regressions (smpl_jreg_kernel)
  if (tid < MP_NUM_JOINTS * 3) {
    float j = m.J_t[tid];
#pragma unroll
    for (int l = 0; l < 10; ++l) j = fmaf(sb[l], m.J_s[tid * 10 + l], j);
    sJ[tid / 3][tid % 3] = j;
  }
  // Rodrigues      lbs.py:276-307
  if (tid < MP_NUM_JOINTS) {
    float rx = thetas[3 * tid], ry = thetas[3 * tid + 1], rz = thetas[3 * tid + 2];
    float ax = rx + 1e-8f, ay = ry + 1e-8f, az = rz + 1e-8f;
    float angle = sqrtf(ax * ax + ay * ay + az * az);
    float dx = rx / angle, dy = ry / angle, dz = rz / angle;
    float c = cosf(angle), s = sinf(angle);
    float K[9] = {0.f, -dz, dy, dz, 0.f, -dx, -dy, dx, 0.f};
    float KK[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        float t = 0.f;
        for (int k = 0; k < 3; ++k) t = fmaf(K[3 * i + k], K[3 * k + j], t);
        KK[3 * i + j] = t;
      }
    for (int i = 0; i < 9; ++i) {
      float ident = (i == 0 || i == 4 || i == 8) ? 1.f : 0.f;
      float r = ident + s * K[i] + (1.f - c) * KK[i];
      sR[tid][i] = r;
      // pose_feature = (rot_mats[1:] - I)      lbs.py:199
      if (tid >= 1) m.pose_feature[(tid - 1) * 9 + i] = r - ident;
    }
  }
  __syncthreads();
  // kinematic chain      lbs.py:323-378 ; then SMPLServer's scale / translation / canonical inverse  smpl.py:86-91
  if (tid == 0) {
    for (int i = 0; i < MP_NUM_JOINTS; ++i) {
      float T[16];
      int p = m.parents[i];
      for (int r = 0; r < 3; ++r) {
        for (int c2 = 0; c2 < 3; ++c2) T[4 * r + c2] = sR[i][3 * r + c2];
        T[4 * r + 3] = (i == 0) ? sJ[0][r] : (sJ[i][r] - sJ[p][r]);
      }
      T[12] = T[13] = T[14] = 0.f;
      T[15] = 1.f;
      if (i == 0) {
        for (int k = 0; k < 16; ++k) sG[0][k] = T[k];
      } else {
        mat4_mul(sG[p], T, sG[i]);
      }
    }
  }
  __syncthreads();
  if (tid < MP_NUM_JOINTS) {
    // rel_transforms = G - pad(G @ [J;0])      lbs.py:371-376
    float A[16];
    for (int k = 0; k < 16; ++k) A[k] = sG[tid][k];
    for (int r = 0; r < 4; ++r) {
      float t = sG[tid][4 * r] * sJ[tid][0] + sG[tid][4 * r + 1] * sJ[tid][1] + sG[tid][4 * r + 2] * sJ[tid][2];
      A[4 * r + 3] -= t;
    }
    const float sc = scale_p[0];
    // tf_mats[:, :, :3, :] *= scale ; tf_mats[:, :, :3, 3] += transl * scale      smpl.py:86-88
    for (int r = 0; r < 3; ++r) {
      for (int c2 = 0; c2 < 4; ++c2) A[4 * r + c2] *= sc;
      A[4 * r + 3] += transl[r] * sc;
    }
    for (int k = 0; k < 16; ++k) m.A_abs[tid * 16 + k] = A[k];
    float O[16];
    if (absolute) {
      for (int k = 0; k < 16; ++k) O[k] = A[k];
    } else {
      mat4_mul(A, m.tfs_c_inv + tid * 16, O);      // einsum('bnij,njk->bnik')  smpl.py:91
    }
    for (int k = 0; k < 16; ++k) tfs_out[tid * 16 + k] = O[k];
  }
}

// per vertex: pose blend shapes + skinning + SMPLServer's scale/translation
//   v_posed = v_shaped + pose_feature @ posedirs ; T = W @ A ; verts = T v_posed      lbs.py:201-227, smpl.py:78
// A_abs already carries the scale and translation: (s*A_rot) v + (s*A_t + t*s) = s*(A v) + t*s.
// smpl_vertex is the per-vertex part, shared with the backward so that both see the same x = v_posed and T.
__device__ __forceinline__ void smpl_vertex(const Smpl& m, const float* spf, const float* sA, const float* sb, int v,
                                            float xo[3], float T[12]) {
  const size_t ld = (size_t)m.V * 3;
  float p0 = 0.f, p1 = 0.f, p2 = 0.f;
  for (int k = 0; k < 207; ++k) {
    const float* pd = m.posedirs + (size_t)k * ld + 3 * (size_t)v;
    float f = spf[k];
    p0 = fmaf(f, pd[0], p0);
    p1 = fmaf(f, pd[1], p1);
    p2 = fmaf(f, pd[2], p2);
  }
  // v_shaped = v_template + blend_shapes(betas, shapedirs)      lbs.py:184, :252-273
  float vs[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float* sd = m.shapedirs + ((size_t)3 * v + a) * 10;
    float sacc = 0.f;
#pragma unroll
    for (int l = 0; l < 10; ++l) sacc = fmaf(sb[l], sd[l], sacc);
    vs[a] = m.v_template[3 * v + a] + sacc;
  }
  xo[0] = vs[0] + p0;
  xo[1] = vs[1] + p1;
  xo[2] = vs[2] + p2;
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = 0.f;
  const float* w = m.lbs_weights + (size_t)v * MP_NUM_JOINTS;
  for (int j = 0; j < MP_NUM_JOINTS; ++j) {
    float wj = w[j];
    if (wj == 0.f) continue;
#pragma unroll
    for (int k = 0; k < 12; ++k) T[k] = fmaf(wj, sA[16 * j + k], T[k]);
  }
}

__device__ __forceinline__ void smpl_load_shared(const Smpl& m, const float* betas, float* spf, float* sA, float* sb) {
  if (threadIdx.x < 10) sb[threadIdx.x] = betas[threadIdx.x];
  for (int i = threadIdx.x; i < 207; i += blockDim.x) spf[i] = m.pose_feature[i];
  for (int i = threadIdx.x; i < MP_NUM_JOINTS * 16; i += blockDim.x) sA[i] = m.A_abs[i];
}

__global__ void smpl_skin_kernel(Smpl m, const float* __restrict__ betas, float* __restrict__ verts_out) {
  __shared__ float spf[207];
  __shared__ float sA[MP_NUM_JOINTS * 16];
  __shared__ float sb[10];
  smpl_load_shared(m, betas, spf, sA, sb);
  __syncthreads();
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= m.V) return;
  float x[3], T[12];
  smpl_vertex(m, spf, sA, sb, v, x, T);
  verts_out[3 * v] = T[0] * x[0] + T[1] * x[1] + T[2] * x[2] + T[3];
  verts_out[3 * v + 1] = T[4] * x[0] + T[5] * x[1] + T[6] * x[2] + T[7];
  verts_out[3 * v + 2] = T[8] * x[0] + T[9] * x[1] + T[10] * x[2] + T[11];
}

// tfs_c_inv = inverse of 24 affine 4x4 matrices (bottom row 0 0 0 1)      smpl.py:47
__global__ void affine_inverse_kernel(const float* __restrict__ T, float* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* A = T + 16 * i;
  float a = A[0], b = A[1], c = A[2], d = A[4], e = A[5], f = A[6], g = A[8], h = A[9], k = A[10];
  float c00 = e * k - f * h, c01 = -(d * k - f * g), c02 = d * h - e * g;
  float det = a * c00 + b * c01 + c * c02;
  float r = 1.0f / det;
  float I[9] = {c00 * r, -(b * k - c * h) * r, (b * f - c * e) * r, c01 * r, (a * k - c * g) * r, -(a * f - c * d) * r,
                c02 * r, -(a * h - b * g) * r, (a * e - b * d) * r};
  float* o = out + 16 * i;
  for (int rr = 0; rr < 3; ++rr) {
    for (int cc = 0; cc < 3; ++cc) o[4 * rr + cc] = I[3 * rr + cc];
    o[4 * rr + 3] = -(I[3 * rr] * A[3] + I[3 * rr + 1] * A[7] + I[3 * rr + 2] * A[11]);
  }
  o[12] = o[13] = o[14] = 0.f;
  o[15] = 1.f;
}

// ---- backward (VJP of mp_smpl_forward) ----------------------------------------------------------------------------
// The per-vertex pass reverses the skinning, the pose blend and the shape blend of every vertex and leaves per-block
// partial sums of dL/dA_j (rows 0..2), dL/dpose_feature and dL/dbetas; one CTA adds them in block order and reverses the
// 24-joint part in fp64.  pose_feature / A_abs are recomputed into the workspace by smpl_pose_kernel itself, so the
// handle's per-call scratch (which a later forward overwrites) is never read.
constexpr int kSmplBwdThreads = 128;
constexpr int kSmplNA = MP_NUM_JOINTS * 12, kSmplNP = kSmplNA + 207 + 10;   // dA rows 0..2 | d pose_feature | d betas

__global__ void __launch_bounds__(kSmplBwdThreads) smpl_skin_backward_kernel(Smpl m, const float* __restrict__ betas,
                                                                             const float* __restrict__ d_verts,
                                                                             float* __restrict__ partials) {
  __shared__ float spf[207];
  __shared__ float sA[MP_NUM_JOINTS * 16];
  __shared__ float sb[10];
  __shared__ float red[kSmplBwdThreads / 32][kSmplNP];
  smpl_load_shared(m, betas, spf, sA, sb);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = v < m.V;
  float x[3] = {0.f, 0.f, 0.f}, T[12], g[3] = {0.f, 0.f, 0.f};
  if (valid) {
    smpl_vertex(m, spf, sA, sb, v, x, T);
    g[0] = d_verts[3 * v];
    g[1] = d_verts[3 * v + 1];
    g[2] = d_verts[3 * v + 2];
  } else {
#pragma unroll
    for (int k = 0; k < 12; ++k) T[k] = 0.f;
  }
  const float xh[4] = {x[0], x[1], x[2], 1.f};
  // verts = T[:3,:] [x;1]:  dT = g [x;1]^T (dA_j = w_j dT), dx = T[:3,:3]^T g
  float dx[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) dx[c] = T[c] * g[0] + T[4 + c] * g[1] + T[8 + c] * g[2];
  const float* w = m.lbs_weights + (size_t)(valid ? v : 0) * MP_NUM_JOINTS;
  for (int j = 0; j < MP_NUM_JOINTS; ++j) {
    const float wj = valid ? w[j] : 0.f;
    const bool any = __any_sync(0xffffffffu, wj != 0.f);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float t = any ? warp_sum(wj * g[r] * xh[c]) : 0.f;
        if (lane == 0) red[warp][12 * j + 4 * r + c] = t;
      }
  }
  // v_posed = v_shaped + pose_feature @ posedirs:  d pose_feature[k] = sum_v posedirs[k, v] . dx_v
  const size_t ld = (size_t)m.V * 3;
  for (int k = 0; k < 207; ++k) {
    float t = 0.f;
    if (valid) {
      const float* pd = m.posedirs + (size_t)k * ld + 3 * (size_t)v;
      t = pd[0] * dx[0] + pd[1] * dx[1] + pd[2] * dx[2];
    }
    t = warp_sum(t);
    if (lane == 0) red[warp][kSmplNA + k] = t;
  }
  // v_shaped = v_template + shapedirs . betas:  d betas[l] = sum_v shapedirs[v, :, l] . dx_v
  for (int l = 0; l < 10; ++l) {
    float t = 0.f;
    if (valid) {
      const float* sd = m.shapedirs + (size_t)3 * v * 10 + l;
      t = sd[0] * dx[0] + sd[10] * dx[1] + sd[20] * dx[2];
    }
    t = warp_sum(t);
    if (lane == 0) red[warp][kSmplNA + 207 + l] = t;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSmplNP; i += blockDim.x) {
    float t = red[0][i];
    for (int q = 1; q < kSmplBwdThreads / 32; ++q) t += red[q][i];
    partials[(size_t)blockIdx.x * kSmplNP + i] = t;
  }
}

// Rodrigues exactly as lbs.py:276-307 writes it (angle = |theta + 1e-8|, axis = theta / angle), in fp64:
// R = I + sin(a) K + (1 - cos(a)) K K with K = skew(axis).  At theta = 0 the axis is 0 and sin(a) / a -> 1, so dR
// reaches theta through the skew basis, as torch autograd's derivative of the same expression does.
__device__ void rodrigues64(const float* th, double R[9], double K[9], double& ang, double a[3], double& c, double& s) {
  double t2 = 0.0;
  for (int q = 0; q < 3; ++q) {
    a[q] = (double)th[q] + 1e-8;
    t2 += a[q] * a[q];
  }
  ang = sqrt(t2);
  const double dx = th[0] / ang, dy = th[1] / ang, dz = th[2] / ang;
  c = cos(ang);
  s = sin(ang);
  const double Kv[9] = {0.0, -dz, dy, dz, 0.0, -dx, -dy, dx, 0.0};
  for (int i = 0; i < 9; ++i) K[i] = Kv[i];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double kk = 0.0;
      for (int k = 0; k < 3; ++k) kk += K[3 * i + k] * K[3 * k + j];
      R[3 * i + j] = (i == j ? 1.0 : 0.0) + s * K[3 * i + j] + (1.0 - c) * kk;
    }
}

__global__ void __launch_bounds__(512) smpl_backward_final_kernel(
    Smpl m, const float* __restrict__ scale_p, const float* __restrict__ transl, const float* __restrict__ thetas,
    const float* __restrict__ betas, int absolute, const float* __restrict__ partials, int nblk,
    const float* __restrict__ d_tfs, float* __restrict__ d_scale, float* __restrict__ d_transl,
    float* __restrict__ d_thetas, float* __restrict__ d_betas) {
  __shared__ double sP[kSmplNP];
  __shared__ double sJ[MP_NUM_JOINTS][3], sR[MP_NUM_JOINTS][9], sG[MP_NUM_JOINTS][16];
  __shared__ double sdG[MP_NUM_JOINTS][12], sdJ[MP_NUM_JOINTS][3], sdR[MP_NUM_JOINTS][9];
  __shared__ double sds[MP_NUM_JOINTS], sdt[MP_NUM_JOINTS][3];
  const int tid = threadIdx.x;
  // fixed-order sum of the per-block partials
  for (int i = tid; i < kSmplNP; i += blockDim.x) {
    double t = 0.0;
    for (int q = 0; q < nblk; ++q) t += (double)partials[(size_t)q * kSmplNP + i];
    sP[i] = t;
  }
  // J = J_t + J_s . betas (lbs.py:188) and Rodrigues, recomputed in fp64
  if (tid < MP_NUM_JOINTS * 3) {
    double j = m.J_t[tid];
    for (int l = 0; l < 10; ++l) j += (double)betas[l] * (double)m.J_s[tid * 10 + l];
    sJ[tid / 3][tid % 3] = j;
  }
  if (tid < MP_NUM_JOINTS) {
    double K[9], ang, a[3], c, s;
    rodrigues64(thetas + 3 * tid, sR[tid], K, ang, a, c, s);
  }
  __syncthreads();
  // kinematic chain G_i = G_parent T_i (lbs.py:323-370)
  if (tid == 0) {
    for (int i = 0; i < MP_NUM_JOINTS; ++i) {
      double T[16];
      const int p = m.parents[i];
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[4 * r + c] = sR[i][3 * r + c];
        T[4 * r + 3] = i == 0 ? sJ[0][r] : sJ[i][r] - sJ[p][r];
      }
      T[12] = T[13] = T[14] = 0.0;
      T[15] = 1.0;
      for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
          if (i == 0) {
            sG[0][4 * r + c] = T[4 * r + c];
          } else {
            double t = 0.0;
            for (int k = 0; k < 4; ++k) t += sG[p][4 * r + k] * T[4 * k + c];
            sG[i][4 * r + c] = t;
          }
        }
    }
  }
  __syncthreads();
  if (tid < MP_NUM_JOINTS) {
    const int j = tid;
    const double sc = scale_p[0];
    // dA (rows 0..2) from the vertices and from smpl_tfs = A (absolute) or A @ tfs_c_inv (smpl.py:91); the bottom row of
    // d_tfs reaches nothing (row 3 of A is constant)
    double dA[12];
    for (int k = 0; k < 12; ++k) dA[k] = sP[12 * j + k];
    if (d_tfs) {
      const float* dt = d_tfs + 16 * j;
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) {
          if (absolute) {
            dA[4 * r + c] += dt[4 * r + c];
          } else {
            const float* ci = m.tfs_c_inv + 16 * j;
            double t = 0.0;
            for (int k = 0; k < 4; ++k) t += (double)dt[4 * r + k] * (double)ci[4 * c + k];
            dA[4 * r + c] += t;
          }
        }
    }
    // A0 = G - pad(G [J;0]) (lbs.py:371-376); A[:3] = s A0[:3] + [0 | t s] (smpl.py:86-88)
    double A0[12];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 4; ++c) A0[4 * r + c] = sG[j][4 * r + c];
      A0[4 * r + 3] -= sG[j][4 * r] * sJ[j][0] + sG[j][4 * r + 1] * sJ[j][1] + sG[j][4 * r + 2] * sJ[j][2];
    }
    double ds = 0.0;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 4; ++c) ds += dA[4 * r + c] * A0[4 * r + c];
      ds += dA[4 * r + 3] * (double)transl[r];
      sdt[j][r] = sc * dA[4 * r + 3];
    }
    sds[j] = ds;
    double dJ[3] = {0.0, 0.0, 0.0};
    for (int r = 0; r < 3; ++r) {
      const double d3 = sc * dA[4 * r + 3];
      for (int c = 0; c < 4; ++c) sdG[j][4 * r + c] = sc * dA[4 * r + c];
      for (int c = 0; c < 3; ++c) {
        sdG[j][4 * r + c] -= d3 * sJ[j][c];
        dJ[c] -= d3 * sG[j][4 * r + c];
      }
    }
    for (int c = 0; c < 3; ++c) sdJ[j][c] = dJ[c];
  }
  __syncthreads();
  // the chain in reverse: children (higher indices) first
  if (tid == 0) {
    for (int j = MP_NUM_JOINTS - 1; j >= 0; --j) {
      const double* dG = sdG[j];
      if (j == 0) {
        for (int r = 0; r < 3; ++r) {
          for (int c = 0; c < 3; ++c) sdR[0][3 * r + c] = dG[4 * r + c];
          sdJ[0][r] += dG[4 * r + 3];
        }
        continue;
      }
      const int p = m.parents[j];
      // dT_j = G_p^T dG_j (row 3 of dG_j is 0)
      for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 4; ++b) {
          double t = 0.0;
          for (int r = 0; r < 3; ++r) t += sG[p][4 * r + a] * dG[4 * r + b];
          if (b < 3) {
            sdR[j][3 * a + b] = t;
          } else {
            sdJ[j][a] += t;
            sdJ[p][a] -= t;
          }
        }
      }
      // dG_p += dG_j T_j^T
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) {
          double t = 0.0;
          for (int k = 0; k < 3; ++k) t += dG[4 * r + k] * sR[j][3 * c + k];
          t += dG[4 * r + 3] * (sJ[j][c] - sJ[p][c]);
          sdG[p][4 * r + c] += t;
        }
        sdG[p][4 * r + 3] += dG[4 * r + 3];
      }
    }
    double ds = 0.0, dt[3] = {0.0, 0.0, 0.0};
    for (int j = 0; j < MP_NUM_JOINTS; ++j) {
      ds += sds[j];
      for (int r = 0; r < 3; ++r) dt[r] += sdt[j][r];
    }
    d_scale[0] = (float)ds;
    for (int r = 0; r < 3; ++r) d_transl[r] = (float)dt[r];
  }
  __syncthreads();
  if (tid < MP_NUM_JOINTS) {
    const int j = tid;
    double dR[9];
    for (int i = 0; i < 9; ++i) dR[i] = sdR[j][i] + (j >= 1 ? sP[kSmplNA + 9 * (j - 1) + i] : 0.0);  // lbs.py:199
    double R[9], K[9], ang, a[3], c, s;
    rodrigues64(thetas + 3 * j, R, K, ang, a, c, s);
    // R = I + s K + (1 - c) K K
    double dang = 0.0, dK[9];
    for (int p = 0; p < 3; ++p)
      for (int q = 0; q < 3; ++q) {
        double kk = 0.0, dkk = 0.0;
        for (int k = 0; k < 3; ++k) {
          kk += K[3 * p + k] * K[3 * k + q];
          dkk += dR[3 * p + k] * K[3 * q + k] + K[3 * k + p] * dR[3 * k + q];   // dL/dK of K K: dR K^T + K^T dR
        }
        dang += dR[3 * p + q] * (c * K[3 * p + q] + s * kk);
        dK[3 * p + q] = s * dR[3 * p + q] + (1.0 - c) * dkk;
      }
    // K = skew(axis), axis = theta / angle, angle = |theta + 1e-8|
    const double dd[3] = {dK[7] - dK[5], dK[2] - dK[6], dK[3] - dK[1]};
    double dth[3];
    for (int q = 0; q < 3; ++q) {
      dth[q] = dd[q] / ang;
      dang -= dd[q] * (double)thetas[3 * j + q] / (ang * ang);
    }
    for (int q = 0; q < 3; ++q) d_thetas[3 * j + q] = (float)(dth[q] + dang * a[q] / ang);
  }
  if (tid < 10) {
    double t = sP[kSmplNA + 207 + tid];
    for (int k = 0; k < MP_NUM_JOINTS * 3; ++k) t += sdJ[k / 3][k % 3] * (double)m.J_s[k * 10 + tid];
    d_betas[tid] = (float)t;
  }
}

static int smpl_backward_blocks(int V) { return div_up(V, kSmplBwdThreads); }

static int smpl_run(const Smpl& m, const float* scale, const float* transl, const float* thetas, const float* betas,
                    int absolute, float* verts, float* tfs, cudaStream_t st) {
  smpl_pose_kernel<<<1, 1024, 0, st>>>(m, scale, transl, thetas, betas, absolute, tfs);
  MP_LAUNCH_CHECK();
  smpl_skin_kernel<<<div_up(m.V, 128), 128, 0, st>>>(m, betas, verts);
  MP_LAUNCH_CHECK();
  return 0;
}

// The model's per-handle buffers, in its caller's storage; `canon` holds the canonical pose's 86 parameters.
static void smpl_carve(Arena& a, int V, Smpl& m, float*& canon) {
  m.v_shaped = a.take<float>((size_t)V * 3);
  m.verts_c = a.take<float>((size_t)V * 3);
  m.pose_feature = a.take<float>(207);
  m.A_abs = a.take<float>(24 * 16);
  m.tfs_c_inv = a.take<float>(24 * 16);
  m.tmp_tfs = a.take<float>(24 * 16);
  m.J_t = a.take<float>(24 * 3);
  m.J_s = a.take<float>(24 * 3 * 10);
  canon = a.take<float>(86);
}

// The backward's per-call scratch: its own pose features, absolute and posed transforms, and per-CTA partials.
struct SmplBackwardWs {
  float *pose_feature, *A_abs, *tfs, *partials;
};
static void smpl_backward_carve(Arena& a, int V, SmplBackwardWs& w) {
  w.pose_feature = a.take<float>(207);
  w.A_abs = a.take<float>(24 * 16);
  w.tfs = a.take<float>(24 * 16);
  w.partials = a.take<float>((size_t)smpl_backward_blocks(V) * kSmplNP);
}

}  // namespace mp

struct mp_smpl {
  mp::Smpl m;
};

extern "C" {

size_t mp_smpl_bytes(int V) {
  mp::Arena a;
  mp::Smpl m{};
  float* canon;
  mp::smpl_carve(a, V > 0 ? V : 0, m, canon);
  return a.off;
}

int mp_smpl_create(const float* v_template, const float* shapedirs, const float* posedirs, const float* J_regressor,
                   const int* parents_host, const float* lbs_weights, int V, const float* betas_canonical, void* storage,
                   size_t storage_bytes, mp_smpl_t** out, void* stream) {
  using namespace mp;
  MP_REQUIRE(v_template && shapedirs && posedirs && J_regressor && parents_host && lbs_weights && storage && out,
             "mp_smpl_create: null argument");
  Arena a(storage, storage_bytes);
  Smpl m{};
  float* canon;
  smpl_carve(a, V, m, canon);
  MP_TRY(a.fits("mp_smpl_create", "storage"));
  cudaStream_t st = (cudaStream_t)stream;
  m.V = V;
  m.v_template = v_template;
  m.shapedirs = shapedirs;
  m.posedirs = posedirs;
  m.J_regressor = J_regressor;
  m.lbs_weights = lbs_weights;
  for (int i = 0; i < MP_NUM_JOINTS; ++i) m.parents[i] = parents_host[i];
  mp_smpl* h = new mp_smpl();
  h->m = m;
  // canonical pose (smpl.py:35-47): scale 1, no translation, hips +-pi/6 about z, the person's betas; absolute
  // transforms, inverted once
  float host[86];
  memset(host, 0, sizeof(host));
  host[0] = 1.f;
  host[4 + 5] = (float)(M_PI / 6.0);
  host[4 + 8] = (float)(-M_PI / 6.0);
  cudaError_t e = cudaMemcpyAsync(canon, host, sizeof(host), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // host[] is a stack buffer
  if (e != cudaSuccess) {
    delete h;
    set_error("mp_smpl_create: %s", cudaGetErrorString(e));
    return -2;
  }
  const float* betas = betas_canonical ? betas_canonical : canon + 76;
  smpl_jreg_kernel<<<1, 1024, 0, st>>>(m);
  g_launches++;
  int rc = smpl_run(m, canon, canon + 1, canon + 4, betas, 1, m.verts_c, m.tmp_tfs, st);
  if (rc == 0) {
    affine_inverse_kernel<<<1, 32, 0, st>>>(m.tmp_tfs, m.tfs_c_inv, 24);
    g_launches++;
  }
  if (rc) {
    delete h;
    return rc;
  }
  *out = h;
  return 0;
}

void mp_smpl_free(mp_smpl_t* h) { delete h; }

int mp_smpl_canonical(mp_smpl_t* h, float* verts_c, float* tfs_c_inv, void* stream) {
  MP_REQUIRE(h, "mp_smpl_canonical: null handle");
  cudaStream_t st = (cudaStream_t)stream;
  if (verts_c)
    MP_CHECK_CUDA(cudaMemcpyAsync(verts_c, h->m.verts_c, (size_t)h->m.V * 3 * 4, cudaMemcpyDeviceToDevice, st));
  if (tfs_c_inv)
    MP_CHECK_CUDA(cudaMemcpyAsync(tfs_c_inv, h->m.tfs_c_inv, 24 * 16 * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int mp_smpl_forward(mp_smpl_t* h, const float* scale, const float* transl, const float* thetas, const float* betas,
                    int absolute, float* smpl_verts, float* smpl_tfs, void* stream) {
  MP_REQUIRE(h && scale && transl && thetas && betas && smpl_verts && smpl_tfs, "mp_smpl_forward: null argument");
  return mp::smpl_run(h->m, scale, transl, thetas, betas, absolute, smpl_verts, smpl_tfs, (cudaStream_t)stream);
}

size_t mp_smpl_backward_workspace_bytes(int V) {
  mp::Arena a;
  mp::SmplBackwardWs w;
  mp::smpl_backward_carve(a, V > 0 ? V : 0, w);
  return a.off;
}

int mp_smpl_backward(mp_smpl_t* h, const float* scale, const float* transl, const float* thetas, const float* betas,
                     int absolute, const float* d_verts, const float* d_tfs, float* d_scale, float* d_transl,
                     float* d_thetas, float* d_betas, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(h && scale && transl && thetas && betas && d_scale && d_transl && d_thetas && d_betas,
             "mp_smpl_backward: null argument");
  Arena a(workspace, workspace_bytes);
  SmplBackwardWs w;
  smpl_backward_carve(a, h->m.V, w);
  MP_TRY(a.fits("mp_smpl_backward"));
  cudaStream_t st = (cudaStream_t)stream;
  Smpl m = h->m;   // a copy whose per-call scratch lives in the workspace
  m.pose_feature = w.pose_feature;
  m.A_abs = w.A_abs;
  float* tfs_scratch = w.tfs;
  float* partials = w.partials;
  int nblk = d_verts ? smpl_backward_blocks(m.V) : 0;
  if (nblk) {
    smpl_pose_kernel<<<1, 1024, 0, st>>>(m, scale, transl, thetas, betas, absolute, tfs_scratch);
    MP_LAUNCH_CHECK();
    smpl_skin_backward_kernel<<<nblk, kSmplBwdThreads, 0, st>>>(m, betas, d_verts, partials);
    MP_LAUNCH_CHECK();
  }
  smpl_backward_final_kernel<<<1, 512, 0, st>>>(m, scale, transl, thetas, betas, absolute, partials, nblk, d_tfs, d_scale,
                                                d_transl, d_thetas, d_betas);
  MP_LAUNCH_CHECK();
  return 0;
}
}
