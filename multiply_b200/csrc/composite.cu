// Multi-person compositing along each ray.
//   reference: /root/reference/code/lib/model/multiply.py:427-480 — flatten all persons' samples
//   into one table, sort by t_end (:443), stable-sort by ray (:445), nerfacc
//   render_weight_from_density / pack_info / accumulate_along_rays (:455-478), and the
//   background transmittance taken at the START of each ray's last sample (:457-463).
//
// Design: no global sort.  Each person's per-ray list is already sorted, so one warp per
// ray merges the P lists by rank (binary searches in shared memory), scans sigma*delta with a
// warp scan and reduces the weighted sums in registers — one kernel, one pass over the samples.
// Tie order on equal t_end: (person, sample) ascending — the order oracle/port.py uses.
#include "common.cuh"

namespace mp {

__global__ void fill_int_kernel(int* p, int n, int v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void row_of_ray_kernel(const int64_t* __restrict__ idx, int n_rows, int* __restrict__ row_of_ray,
                                  const int* __restrict__ n_dev) {
  if (n_dev) n_rows = min(n_rows, *n_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_rows) row_of_ray[idx[i]] = i;
}

// The ray's row in each person's hit list (-1: the person does not cover it); returns K, its samples over all persons.
__device__ __forceinline__ int ray_rows(const CompositePersons& cp, int P, int ray, int n, int* row) {
  int K = 0;
  for (int p = 0; p < P; ++p) {
    row[p] = cp.row_of_ray[p][ray];
    if (row[p] >= 0) K += n;
  }
  return K;
}

// Rank of every sample of the ray in the merged (t_end, person, sample) order; scatters sigma * delta into ssd[rank]
// and the rank into srank.  ste receives the t_end lists ([P][n]) and is free again when this returns.
__device__ __forceinline__ void merge_ranks(const CompositePersons& cp, const int* row, int n, float beta, float* ste,
                                            float* ssd, int* srank, int lane) {
  const int P = cp.P;
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    for (int i = lane; i < n; i += 32) ste[p * n + i] = z[i + 1];
  }
  __syncwarp();
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    const float* s = cp.sdf[p] + (size_t)row[p] * n;
    for (int i = lane; i < n; i += 32) {
      float te = ste[p * n + i];
      int r = i;
      for (int q = 0; q < P; ++q) {
        if (q == p || row[q] < 0) continue;
        r += (q < p) ? upper_bound(ste + q * n, n, te) : lower_bound(ste + q * n, n, te);
      }
      float ts = z[i];
      float sigma = laplace_density(s[i], beta);       // multiply.py:450
      ssd[r] = sigma * (te - ts);
      srank[p * n + i] = r;
    }
  }
  __syncwarp();
}

// In-place exclusive scan of ssd[0, K) (lane-owned chunks of ceil(K / 32)); returns the exclusive prefix of the ray's
// last merged sample, i.e. the exponent of bg_T, in every lane.
__device__ __forceinline__ float scan_excl_chunks(float* ssd, int K, int lane) {
  int C = (K + 31) >> 5;
  int b = lane * C, e = min(K, b + C);
  float s1 = 0.f;
  for (int k = b; k < e; ++k) s1 += ssd[k];
  float run = warp_scan_excl(s1, lane);
  float last_excl = 0.f;
  for (int k = b; k < e; ++k) {
    float v = ssd[k];
    ssd[k] = run;          // exclusive prefix
    if (k == K - 1) last_excl = run;
    run += v;
  }
  __syncwarp();
  return warp_max(((K - 1) >= b && (K - 1) < e) ? last_excl : -INFINITY);
}

__global__ void composite_kernel(CompositePersons cp, int R, int n, float beta, float* __restrict__ fg_rgb,
                                 float* __restrict__ normal, float* __restrict__ acc, float* __restrict__ acc_person,
                                 float* __restrict__ bg_T) {
  extern __shared__ float smem[];
  const int P = cp.P;
  int wpc = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ray = blockIdx.x * wpc + wid;
  if (ray >= R) return;
  float* ste = smem + (size_t)wid * 3 * P * n;   // t_end lists, [P][n]
  float* ssd = ste + P * n;                      // sigma*delta in merged order
  int* srank = (int*)(ssd + P * n);              // merged rank of (p,i)
  int row[MP_MAX_PERSONS];
  const int K = ray_rows(cp, P, ray, n, row);
  if (K == 0) {
    if (lane == 0) {
      fg_rgb[3 * ray] = fg_rgb[3 * ray + 1] = fg_rgb[3 * ray + 2] = 0.f;
      normal[3 * ray] = normal[3 * ray + 1] = normal[3 * ray + 2] = 0.f;
      acc[ray] = 0.f;
      bg_T[ray] = 1.f;                             // multiply.py:461
      for (int p = 0; p < P; ++p) acc_person[(size_t)ray * P + p] = 0.f;
    }
    return;
  }
  merge_ranks(cp, row, n, beta, ste, ssd, srank, lane);
  // exclusive scan of sigma*delta -> transmittance exponent, in place
  float last_excl = scan_excl_chunks(ssd, K, lane);
  float a_rgb[3] = {0.f, 0.f, 0.f}, a_n[3] = {0.f, 0.f, 0.f}, a_w = 0.f;
  float a_p[MP_MAX_PERSONS];
  for (int p = 0; p < MP_MAX_PERSONS; ++p) a_p[p] = 0.f;
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    const float* s = cp.sdf[p] + (size_t)row[p] * n;
    const float* c = cp.rgb[p] + (size_t)row[p] * n * 3;
    const float* nm = cp.nrm[p] + (size_t)row[p] * n * 3;
    for (int i = lane; i < n; i += 32) {
      float sigma = laplace_density(s[i], beta);
      float sd = sigma * (z[i + 1] - z[i]);
      float alpha = 1.f - expf(-sd);
      float T = expf(-ssd[srank[p * n + i]]);
      float w = T * alpha;
      a_rgb[0] += w * c[3 * i];
      a_rgb[1] += w * c[3 * i + 1];
      a_rgb[2] += w * c[3 * i + 2];
      a_n[0] += w * nm[3 * i];
      a_n[1] += w * nm[3 * i + 1];
      a_n[2] += w * nm[3 * i + 2];
      a_w += w;
      a_p[p] += w;
    }
  }
  for (int k = 0; k < 3; ++k) {
    a_rgb[k] = warp_sum(a_rgb[k]);
    a_n[k] = warp_sum(a_n[k]);
  }
  a_w = warp_sum(a_w);
  for (int p = 0; p < P; ++p) a_p[p] = warp_sum(a_p[p]);
  if (lane == 0) {
    for (int k = 0; k < 3; ++k) {
      fg_rgb[3 * ray + k] = a_rgb[k];
      normal[3 * ray + k] = a_n[k];
    }
    acc[ray] = a_w;
    for (int p = 0; p < P; ++p) acc_person[(size_t)ray * P + p] = a_p[p];
    bg_T[ray] = expf(-last_excl);     // transmittance at the start of the ray's last sample
  }
}

// Upstream gradients of the compositor (any may be NULL = zero) and the per-person sample gradients it produces.
struct CompositeGrads {
  const float* d_fg;      // [R,3]
  const float* d_nrm;     // [R,3]
  const float* d_acc;     // [R]
  const float* d_accp;    // [R,P]
  const float* d_bgT;     // [R]
  float* d_sdf[MP_MAX_PERSONS];   // [R_p,n]
  float* d_rgb[MP_MAX_PERSONS];   // [R_p,n,3]
  float* d_nrm_s[MP_MAX_PERSONS]; // [R_p,n,3]
};

// Backward of composite_kernel, one warp per ray.  With x_k = sigma_k delta_k in merged order, T_k = exp(-sum_{j<k} x_j),
// w_k = T_k (1 - exp(-x_k)) and g_k = <dfg, rgb_k> + <dnormal, n_k> + dacc + dacc_person[person(k)]:
//   dL/dx_k = T_{k+1} g_k - S_{k+1} - [k < K-1] bg_T dbg_T,      S_{k+1} = sum_{j>k} w_j g_j
// (bg_T is the transmittance at the START of the last sample, so it does not depend on x_{K-1}).  The merged order and
// the prefix scan are the forward's own (merge_ranks, scan_excl_chunks); the suffix sums are a reverse chunked scan.
// dL/dbeta of the ray goes to dbeta_ray[ray], reduced over rays in a fixed order by reduce_dbeta_kernel.
__global__ void composite_backward_kernel(CompositePersons cp, CompositeGrads g, int R, int n, float beta,
                                          float* __restrict__ dbeta_ray) {
  extern __shared__ float smem[];
  const int P = cp.P;
  int wpc = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ray = blockIdx.x * wpc + wid;
  if (ray >= R) return;
  float* ste = smem + (size_t)wid * 3 * P * n;   // t_end lists; then w_k g_k, then S_{k+1}, in merged order
  float* ssd = ste + P * n;                      // sigma*delta -> exclusive prefix, in merged order
  int* srank = (int*)(ssd + P * n);
  int row[MP_MAX_PERSONS];
  const int K = ray_rows(cp, P, ray, n, row);
  if (K == 0) {                                  // bg_T = 1 is a constant: nothing depends on a sample
    if (lane == 0) dbeta_ray[ray] = 0.f;
    return;
  }
  merge_ranks(cp, row, n, beta, ste, ssd, srank, lane);
  float last_excl = scan_excl_chunks(ssd, K, lane);
  const float dfg[3] = {g.d_fg ? g.d_fg[3 * ray] : 0.f, g.d_fg ? g.d_fg[3 * ray + 1] : 0.f,
                        g.d_fg ? g.d_fg[3 * ray + 2] : 0.f};
  const float dn[3] = {g.d_nrm ? g.d_nrm[3 * ray] : 0.f, g.d_nrm ? g.d_nrm[3 * ray + 1] : 0.f,
                       g.d_nrm ? g.d_nrm[3 * ray + 2] : 0.f};
  const float dacc = g.d_acc ? g.d_acc[ray] : 0.f;
  const float dbgT = g.d_bgT ? g.d_bgT[ray] : 0.f;
  float* wg = ste;
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    const float* s = cp.sdf[p] + (size_t)row[p] * n;
    const float* c = cp.rgb[p] + (size_t)row[p] * n * 3;
    const float* nm = cp.nrm[p] + (size_t)row[p] * n * 3;
    const float dap = (g.d_accp ? g.d_accp[(size_t)ray * P + p] : 0.f) + dacc;
    for (int i = lane; i < n; i += 32) {
      int r = srank[p * n + i];
      float sd = laplace_density(s[i], beta) * (z[i + 1] - z[i]);
      float w = expf(-ssd[r]) * (1.f - expf(-sd));
      float gk = dfg[0] * c[3 * i] + dfg[1] * c[3 * i + 1] + dfg[2] * c[3 * i + 2] + dn[0] * nm[3 * i] +
                 dn[1] * nm[3 * i + 1] + dn[2] * nm[3 * i + 2] + dap;
      wg[r] = w * gk;
    }
  }
  __syncwarp();
  // exclusive suffix sums of w_k g_k, in place: lane chunks walked backwards after a reverse warp scan of chunk sums
  {
    int C = (K + 31) >> 5;
    int b = lane * C, e = min(K, b + C);
    float s1 = 0.f;
    for (int k = e - 1; k >= b; --k) s1 += wg[k];
    float incl = s1;                               // inclusive reverse scan over lanes
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_down_sync(0xffffffffu, incl, o);
      if (lane + o < 32) incl += t;
    }
    float run = __shfl_down_sync(0xffffffffu, incl, 1);
    if (lane == 31) run = 0.f;
    for (int k = e - 1; k >= b; --k) {
      float v = wg[k];
      wg[k] = run;                                 // S_{k+1}
      run += v;
    }
  }
  __syncwarp();
  const float bgT_term = expf(-last_excl) * dbgT;
  const float inv_b = __fdiv_rn(1.0f, beta);
  float a_beta = 0.f;
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    const float* s = cp.sdf[p] + (size_t)row[p] * n;
    const float* c = cp.rgb[p] + (size_t)row[p] * n * 3;
    const float* nm = cp.nrm[p] + (size_t)row[p] * n * 3;
    const float dap = (g.d_accp ? g.d_accp[(size_t)ray * P + p] : 0.f) + dacc;
    float* o_sdf = g.d_sdf[p] + (size_t)row[p] * n;
    float* o_rgb = g.d_rgb[p] + (size_t)row[p] * n * 3;
    float* o_nrm = g.d_nrm_s[p] + (size_t)row[p] * n * 3;
    for (int i = lane; i < n; i += 32) {
      int r = srank[p * n + i];
      float sdf = s[i];
      float sigma = laplace_density(sdf, beta);
      float delta = z[i + 1] - z[i];
      float sd = sigma * delta;
      float T = expf(-ssd[r]);
      float ex = expf(-sd);
      float w = T * (1.f - ex);
      float gk = dfg[0] * c[3 * i] + dfg[1] * c[3 * i + 1] + dfg[2] * c[3 * i + 2] + dn[0] * nm[3 * i] +
                 dn[1] * nm[3 * i + 1] + dn[2] * nm[3 * i + 2] + dap;
      float dx = (T * ex) * gk - wg[r] - ((r < K - 1) ? bgT_term : 0.f);
      // torch's kinks: sign(0) = 0 and d|s|/ds = sign(s), so both derivatives carry sign(s)^2 resp. sign(s)
      float sg = (sdf > 0.f) ? 1.f : ((sdf < 0.f) ? -1.f : 0.f);
      float as = fabsf(sdf);
      // e2 = exp(-|s|/beta) / (2 beta^2) as one exponential, so that it stays a normal float where exp(-|s|/beta)
      // alone would be subnormal (beta = 1e-4)
      float e2 = 0.5f * expf(2.f * logf(inv_b) - as * inv_b);
      float dsig_ds = -(sg * sg) * e2;
      // -sigma/beta + sign(s) e |s| / (2 beta^3); for s > 0, sigma = e / (2 beta) and the two terms share e2
      float dsig_db = (sg > 0.f) ? e2 * (as * inv_b - 1.f) : -sigma * inv_b + sg * e2 * as * inv_b;
      float dxd = dx * delta;
      o_sdf[i] = dxd * dsig_ds;
      a_beta += dxd * dsig_db;
      for (int k = 0; k < 3; ++k) {
        o_rgb[3 * i + k] = w * dfg[k];
        o_nrm[3 * i + k] = w * dn[k];
      }
    }
  }
  a_beta = warp_sum(a_beta);
  if (lane == 0) dbeta_ray[ray] = a_beta;
}

// d_beta = sum over rays of dbeta_ray, in a fixed order (one block: strided partial sums, then a fixed tree)
__global__ void reduce_dbeta_kernel(const float* __restrict__ dbeta_ray, int R, float* __restrict__ d_beta) {
  __shared__ float part[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < R; i += 256) s += dbeta_ray[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *d_beta = part[0];
}

// rgb = fg + bg_T * bg ; fg_rgb_values = fg + bg_T * 1     (multiply.py:544-545, :590)
__global__ void final_compose_kernel(const float* __restrict__ fg, const float* __restrict__ bgT,
                                     const float* __restrict__ bg, int R, float* __restrict__ rgb,
                                     float* __restrict__ fg_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * R) return;
  int r = i / 3;
  float b = bg ? bg[i] : 1.0f;
  rgb[i] = fg[i] + bgT[r] * b;
  if (fg_out) fg_out[i] = fg[i] + bgT[r] * 1.0f;
}

// Dynamic shared memory per warp (one ray) of both compositor kernels: the t_end lists, sigma*delta and merged ranks of
// its P*n samples; *wpc is set to the warps per CTA that fit in 200 KB.
static size_t composite_smem(int P, int n, int* wpc) {
  const size_t per_warp = (size_t)3 * P * n * sizeof(float);
  *wpc = clamp_wpc((size_t)(200 * 1024) / per_warp);
  return per_warp;
}

int launch_composite(const CompositePersons& cp, int R, int n, float beta, float* fg_rgb, float* normal, float* acc,
                     float* acc_person, float* bg_T, cudaStream_t st) {
  int wpc;
  const size_t per_warp = composite_smem(cp.P, n, &wpc);
  MP_REQUIRE(per_warp <= 200 * 1024, "composite: P*n too large for shared memory");
  MP_CHECK_CUDA(cudaFuncSetAttribute(composite_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(wpc * per_warp)));
  composite_kernel<<<div_up(R, wpc), wpc * 32, wpc * per_warp, st>>>(cp, R, n, beta, fg_rgb, normal, acc, acc_person,
                                                                      bg_T);
  MP_LAUNCH_CHECK();
  return 0;
}

int launch_composite_backward(const CompositePersons& cp, const CompositeGrads& g, int R, int n, float beta,
                              float* dbeta_ray, float* d_beta, cudaStream_t st) {
  int wpc;
  const size_t per_warp = composite_smem(cp.P, n, &wpc);
  MP_REQUIRE(per_warp <= 200 * 1024, "composite backward: P*n too large for shared memory");
  MP_CHECK_CUDA(cudaFuncSetAttribute(composite_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(wpc * per_warp)));
  composite_backward_kernel<<<div_up(R, wpc), wpc * 32, wpc * per_warp, st>>>(cp, g, R, n, beta, dbeta_ray);
  MP_LAUNCH_CHECK();
  reduce_dbeta_kernel<<<1, 256, 0, st>>>(dbeta_ray, R, d_beta);
  MP_LAUNCH_CHECK();
  return 0;
}

// backward of final_compose_kernel, one thread per ray:
//   d fg = d rgb + d fg_values ; d bg_T = sum_c (d rgb_c * bg_c + d fg_values_c) ; d bg = bg_T * d rgb
__global__ void final_compose_backward_kernel(const float* __restrict__ bgT, const float* __restrict__ bg, int R,
                                              const float* __restrict__ d_rgb, const float* __restrict__ d_fgv,
                                              float* __restrict__ d_fg, float* __restrict__ d_bgT,
                                              float* __restrict__ d_bg) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float t = bgT[r];
  float acc = 0.f;
  for (int c = 0; c < 3; ++c) {
    int i = 3 * r + c;
    float dr = d_rgb[i];
    float dv = d_fgv ? d_fgv[i] : 0.f;
    float b = bg ? bg[i] : 1.0f;
    d_fg[i] = dr + dv;
    acc += dr * b + dv;
    if (d_bg) d_bg[i] = t * dr;
  }
  d_bgT[r] = acc;
}

int launch_row_of_ray(const int64_t* idx, int n_rows, int R, int* row_of_ray, cudaStream_t st, const int* n_dev) {
  fill_int_kernel<<<div_up(R, 256), 256, 0, st>>>(row_of_ray, R, -1);
  MP_LAUNCH_CHECK();
  if (n_rows > 0) {
    row_of_ray_kernel<<<div_up(n_rows, 256), 256, 0, st>>>(idx, n_rows, row_of_ray, n_dev);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

// The backward's per-ray d beta terms, then each person's row_of_ray map.
struct CompositeWs {
  float* dbeta_ray;
  int* row_of_ray[MP_MAX_PERSONS];
};
static void composite_carve(Arena& a, int R, int P, bool backward, CompositeWs& w) {
  w.dbeta_ray = backward ? a.take<float>(R) : nullptr;
  for (int p = 0; p < P; ++p) w.row_of_ray[p] = a.take<int>(R);
}

// cp from the caller's person records: each person's row_of_ray map is filled from its hit list on st.
static int composite_persons(const CompositeWs& w, const mp_person_samples_t* persons, int P, int R,
                             CompositePersons& cp, cudaStream_t st) {
  cp.P = P;
  for (int p = 0; p < P; ++p) {
    MP_TRY(launch_row_of_ray(persons[p].ray_index, persons[p].n_rows, R, w.row_of_ray[p], st, nullptr));
    set_person(cp, p, persons[p], w.row_of_ray[p]);
  }
  return 0;
}

static size_t composite_ws_bytes(int R, int P, bool backward) {
  if (P < 1 || P > MP_MAX_PERSONS) return 0;
  Arena a;
  CompositeWs w;
  composite_carve(a, R > 0 ? R : 0, P, backward, w);
  return a.off;
}

int launch_final_compose(const float* fg, const float* bgT, const float* bg, int R, float* rgb, float* fg_out,
                         cudaStream_t st) {
  final_compose_kernel<<<div_up(3 * R, 256), 256, 0, st>>>(fg, bgT, bg, R, rgb, fg_out);
  MP_LAUNCH_CHECK();
  return 0;
}

}  // namespace mp

extern "C" {

size_t mp_composite_workspace_bytes(int R, int P) { return mp::composite_ws_bytes(R, P, false); }

int mp_composite(const mp_person_samples_t* persons, int P, int R, int n, float beta, float* fg_rgb, float* normal,
                 float* acc, float* acc_person, float* bg_T, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(persons && P >= 1 && P <= MP_MAX_PERSONS, "mp_composite: bad person list");
  mp::Arena a(workspace, workspace_bytes);
  mp::CompositeWs w;
  mp::composite_carve(a, R, P, false, w);
  MP_TRY(a.fits("mp_composite"));
  mp::CompositePersons cp;
  cudaStream_t st = (cudaStream_t)stream;
  MP_TRY(mp::composite_persons(w, persons, P, R, cp, st));
  return mp::launch_composite(cp, R, n, beta, fg_rgb, normal, acc, acc_person, bg_T, st);
}

size_t mp_composite_backward_workspace_bytes(int R, int P) { return mp::composite_ws_bytes(R, P, true); }

int mp_composite_backward(const mp_person_samples_t* persons, int P, int R, int n, float beta, const float* d_fg_rgb,
                          const float* d_normal, const float* d_acc, const float* d_acc_person, const float* d_bg_T,
                          const mp_person_sample_grads_t* grads, float* d_beta, void* workspace,
                          size_t workspace_bytes, void* stream) {
  MP_REQUIRE(persons && grads && P >= 1 && P <= MP_MAX_PERSONS, "mp_composite_backward: bad person list");
  MP_REQUIRE(d_beta && R >= 1 && n >= 1, "mp_composite_backward: null d_beta or empty problem");
  for (int p = 0; p < P; ++p)
    MP_REQUIRE(persons[p].n_rows == 0 || (grads[p].d_sdf && grads[p].d_rgb && grads[p].d_normal && persons[p].z_vals &&
                                          persons[p].sdf && persons[p].rgb && persons[p].normal && persons[p].ray_index),
               "mp_composite_backward: null argument for person %d", p);
  int wpc;
  MP_REQUIRE(mp::composite_smem(P, n, &wpc) <= 200 * 1024, "mp_composite_backward: P*n too large for shared memory");
  mp::Arena a(workspace, workspace_bytes);
  mp::CompositeWs w;
  mp::composite_carve(a, R, P, true, w);
  MP_TRY(a.fits("mp_composite_backward"));
  mp::CompositePersons cp;
  mp::CompositeGrads g;
  g.d_fg = d_fg_rgb;
  g.d_nrm = d_normal;
  g.d_acc = d_acc;
  g.d_accp = d_acc_person;
  g.d_bgT = d_bg_T;
  cudaStream_t st = (cudaStream_t)stream;
  MP_TRY(mp::composite_persons(w, persons, P, R, cp, st));
  for (int p = 0; p < P; ++p) {
    g.d_sdf[p] = grads[p].d_sdf;
    g.d_rgb[p] = grads[p].d_rgb;
    g.d_nrm_s[p] = grads[p].d_normal;
  }
  return mp::launch_composite_backward(cp, g, R, n, beta, w.dbeta_ray, d_beta, st);
}

int mp_final_compose_backward(const float* bg_T, const float* bg_rgb, int R, const float* d_rgb_values,
                              const float* d_fg_rgb_values, float* d_fg_rgb, float* d_bg_T, float* d_bg_rgb,
                              void* stream) {
  MP_REQUIRE(bg_T && d_rgb_values && d_fg_rgb && d_bg_T, "mp_final_compose_backward: null argument");
  if (R <= 0) return 0;
  mp::final_compose_backward_kernel<<<mp::div_up(R, 256), 256, 0, (cudaStream_t)stream>>>(
      bg_T, bg_rgb, R, d_rgb_values, d_fg_rgb_values, d_fg_rgb, d_bg_T, d_bg_rgb);
  MP_LAUNCH_CHECK();
  return 0;
}

int mp_final_compose(const float* fg_rgb, const float* bg_T, const float* bg_rgb, int R, float* rgb_values,
                     float* fg_rgb_values, void* stream) {
  MP_REQUIRE(fg_rgb && bg_T && rgb_values, "mp_final_compose: null argument");
  if (R <= 0) return 0;
  return mp::launch_final_compose(fg_rgb, bg_T, bg_rgb, R, rgb_values, fg_rgb_values, (cudaStream_t)stream);
}
}
