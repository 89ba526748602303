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

struct CompositePersons {
  int P;
  int n_rows[MP_MAX_PERSONS];
  const int* row_of_ray[MP_MAX_PERSONS];   // [R] -> row in the person's hit list or -1
  const float* z[MP_MAX_PERSONS];          // [R_p, n+1]
  const float* sdf[MP_MAX_PERSONS];        // [R_p, n]
  const float* rgb[MP_MAX_PERSONS];        // [R_p, n, 3]
  const float* nrm[MP_MAX_PERSONS];        // [R_p, n, 3]
};

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

__device__ __forceinline__ int count_le(const float* a, int n, float v) {   // #elements <= v
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] > v) hi = mid; else lo = mid + 1;
  }
  return lo;
}
__device__ __forceinline__ int count_lt(const float* a, int n, float v) {   // #elements < v
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] >= v) hi = mid; else lo = mid + 1;
  }
  return lo;
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
  int K = 0;
  for (int p = 0; p < P; ++p) {
    row[p] = cp.row_of_ray[p][ray];
    if (row[p] >= 0) K += n;
  }
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
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    for (int i = lane; i < n; i += 32) ste[p * n + i] = z[i + 1];
  }
  __syncwarp();
  // rank of every sample in the merged (t_end, person, sample) order; scatter sigma*delta
  for (int p = 0; p < P; ++p) {
    if (row[p] < 0) continue;
    const float* z = cp.z[p] + (size_t)row[p] * (n + 1);
    const float* s = cp.sdf[p] + (size_t)row[p] * n;
    for (int i = lane; i < n; i += 32) {
      float te = ste[p * n + i];
      int r = i;
      for (int q = 0; q < P; ++q) {
        if (q == p || row[q] < 0) continue;
        r += (q < p) ? count_le(ste + q * n, n, te) : count_lt(ste + q * n, n, te);
      }
      float ts = z[i];
      float sigma = laplace_density(s[i], beta);       // multiply.py:450
      ssd[r] = sigma * (te - ts);
      srank[p * n + i] = r;
    }
  }
  __syncwarp();
  // exclusive scan of sigma*delta -> transmittance exponent, in place
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
  last_excl = warp_max(((K - 1) >= b && (K - 1) < e) ? last_excl : -INFINITY);
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

int launch_composite(const CompositePersons& cp, int R, int n, float beta, float* fg_rgb, float* normal, float* acc,
                     float* acc_person, float* bg_T, cudaStream_t st) {
  size_t per_warp = (size_t)3 * cp.P * n * sizeof(float);
  MP_REQUIRE(per_warp <= 200 * 1024, "composite: P*n too large for shared memory");
  int wpc = clamp_wpc((size_t)(200 * 1024) / per_warp);
  MP_CHECK_CUDA(cudaFuncSetAttribute(composite_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(wpc * per_warp)));
  composite_kernel<<<div_up(R, wpc), wpc * 32, wpc * per_warp, st>>>(cp, R, n, beta, fg_rgb, normal, acc, acc_person,
                                                                      bg_T);
  MP_LAUNCH_CHECK();
  return 0;
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

int launch_final_compose(const float* fg, const float* bgT, const float* bg, int R, float* rgb, float* fg_out,
                         cudaStream_t st) {
  final_compose_kernel<<<div_up(3 * R, 256), 256, 0, st>>>(fg, bgT, bg, R, rgb, fg_out);
  MP_LAUNCH_CHECK();
  return 0;
}

}  // namespace mp

extern "C" {

size_t mp_composite_workspace_bytes(int R, int P) { return (size_t)P * (mp::align_up((size_t)R * 4, 256)) + 4096; }

int mp_composite(const mp_person_samples_t* persons, int P, int R, int n, float beta, float* fg_rgb, float* normal,
                 float* acc, float* acc_person, float* bg_T, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(persons && P >= 1 && P <= MP_MAX_PERSONS, "mp_composite: bad person list");
  MP_REQUIRE(workspace_bytes >= mp_composite_workspace_bytes(R, P), "mp_composite: workspace too small");
  mp::Arena a(workspace, workspace_bytes);
  mp::CompositePersons cp;
  cp.P = P;
  cudaStream_t st = (cudaStream_t)stream;
  for (int p = 0; p < P; ++p) {
    int* ror = a.take<int>(R);
    MP_REQUIRE(a.ok, "mp_composite: workspace too small");
    MP_TRY(mp::launch_row_of_ray(persons[p].ray_index, persons[p].n_rows, R, ror, st, nullptr));
    cp.n_rows[p] = persons[p].n_rows;
    cp.row_of_ray[p] = ror;
    cp.z[p] = persons[p].z_vals;
    cp.sdf[p] = persons[p].sdf;
    cp.rgb[p] = persons[p].rgb;
    cp.nrm[p] = persons[p].normal;
  }
  return mp::launch_composite(cp, R, n, beta, fg_rgb, normal, acc, acc_person, bg_T, st);
}

int mp_final_compose(const float* fg_rgb, const float* bg_T, const float* bg_rgb, int R, float* rgb_values,
                     float* fg_rgb_values, void* stream) {
  MP_REQUIRE(fg_rgb && bg_T && rgb_values, "mp_final_compose: null argument");
  if (R <= 0) return 0;
  return mp::launch_final_compose(fg_rgb, bg_T, bg_rgb, R, rgb_values, fg_rgb_values, (cudaStream_t)stream);
}
}
