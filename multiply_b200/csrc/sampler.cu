// VolSDF error-bound ray sampler (Algorithm 1), eval mode.
//   reference: /root/reference/code/lib/model/ray_sampler.py
//     UniformSampler.get_z_vals          :21-42
//     ErrorBoundSampler.get_z_vals       :66-220
//     ErrorBoundSampler.get_error_bound  :222-230
//
// Design: one warp per ray, the ray's sorted sample list (<= max_total_iters * E values)
// staged in shared memory; prefix sums are warp scans over per-lane contiguous chunks; the
// resampled points are merged (stable two-way merge by rank) instead of re-sorted.  The
// batch-global convergence test `beta.max() > beta0` (:137) is an atomicOr into a per-trip
// flag that the NEXT kernels read, so the whole loop runs without any host synchronisation:
// the host enqueues max_total_iters trips and the kernels of trips after convergence exit
// immediately.  This file is compiled with -fmad=false so that comparisons see the same
// separately-rounded a*a + b*b the reference computes.
#include "common.cuh"

namespace mp {

struct SamplerState {
  int not_converge[8];   // per trip: any ray with beta > beta0
  int active[8];         // per trip: loop still running at the start of trip t (active[0] = 1)
  int count[8];          // per trip: compact work-list length
  int final_trip;        // trip whose resample produced the final samples
};

struct SamplerTables {
  float* u_E;      // linspace(0,1,E)   ray_sampler.py:167 (non-final trips), :29 (uniform t_vals)
  float* u_S;      // linspace(0,1,S)   ray_sampler.py:167 (final, eval)
  int* extra_idx;  // [max_iters][X] : linspace(0, M-1, X).long() for M = (k+1)E   ray_sampler.py:204
  float* z_bg;     // [32] : linspace(0,1,32) * (1/bound)   ray_sampler.py:215-218
};

// torch.linspace element (ATen CPU kernel; see mp_linspace_host)
__device__ __forceinline__ float linspace_at(float start, float end, int n, int i) {
  if (n == 1) return start;
  float step = (end - start) / (float)(n - 1);
  return (i < n / 2) ? fmaf(step, (float)i, start) : fmaf(-step, (float)(n - 1 - i), end);
}

__global__ void tables_kernel(SamplerTables t, int E, int S, int X, int max_iters, float inv_bound,
                              SamplerState* st) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < E) t.u_E[i] = linspace_at(0.f, 1.f, E, i);
  if (i < S) t.u_S[i] = linspace_at(0.f, 1.f, S, i);
  if (i < 32) t.z_bg[i] = linspace_at(0.f, 1.f, 32, i) * inv_bound;
  if (i < max_iters * X) {
    int k = i / X, j = i - k * X;
    int M = (k + 1) * E;
    t.extra_idx[i] = (int)linspace_at(0.f, (float)(M - 1), X, j);
  }
  if (i == 0) {
    for (int k = 0; k < 8; ++k) {
      st->not_converge[k] = 0;
      st->active[k] = (k == 0) ? 1 : 0;
      st->count[k] = 0;
    }
    st->final_trip = -1;
  }
}

// uniform initial samples + Lemma-2 beta bound     ray_sampler.py:21-42, :70-76
// One warp per ray: lane l owns samples l, l+32, ... (coalesced stores of the ray's row; the one-thread-per-ray version
// wrote 256 values at a 5 KB stride each: 38 us for 2300 rays).
__global__ void sampler_init_kernel(const float* __restrict__ dirs, const float* __restrict__ cam, int R, float r,
                                    float near, int E, const float* __restrict__ tvals, float bound_coef,
                                    float* __restrict__ z, int zcap, float* __restrict__ beta,
                                    float* __restrict__ far_out, SamplerState* st, const int* __restrict__ R_dev,
                                    const float* __restrict__ t_rand) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (R_dev) R = min(R, *R_dev);     // device-side row count (hit list culled on the GPU, no host sync)
  if (ray >= R) return;
  const float* o = cam + 3 * ray;
  const float* d = dirs + 3 * ray;
  // rend_util.get_sphere_intersections, :131-147 (a miss is reported by mp_render_rays' sphere_status_kernel)
  float dot = d[0] * o[0] + d[1] * o[1] + d[2] * o[2];
  float nrm = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
  float under = dot * dot - (nrm * nrm - r * r);
  float far = fmaxf(sqrtf(under) * 1.f - dot, 0.f);
  if (lane == 0) far_out[ray] = far;
  float* zr = z + (size_t)ray * zcap;
  auto zu = [&](int j) { float t = tvals[j]; return near * (1.f - t) + far * t; };
  // sample j (training mode, model.training: stratified in the interval between the midpoints, ray_sampler.py:32-40)
  auto zs = [&](int j) {
    float zj = zu(j);
    if (t_rand) {
      float lower = (j == 0) ? zj : .5f * (zj + zu(j - 1));
      float upper = (j == E - 1) ? zj : .5f * (zu(j + 1) + zj);
      zj = lower + (upper - lower) * t_rand[(size_t)ray * E + j];
    }
    return zj;
  };
  float sum = 0.f;
  for (int j = lane; j < E; j += 32) {
    float zj = zs(j);
    zr[j] = zj;
    if (j > 0) {
      float dd = zj - zs(j - 1);
      sum += dd * dd;
    }
  }
  sum = warp_sum(sum);
  if (lane == 0) beta[ray] = sqrtf(bound_coef * sum);
}

// ---- per-ray warp routines -------------------------------------------------------------------

// d* of Theorem 1 for interval i     ray_sampler.py:98-110
__device__ __forceinline__ float dstar_interval(float z0, float z1, float s0, float s1) {
  float a = z1 - z0, b = fabsf(s0), c = fabsf(s1);
  float aa = a * a, bb = b * b, cc = c * c;
  bool first = (aa + bb) <= cc;
  bool second = (aa + cc) <= bb;
  float ds = 0.f;
  if (first) ds = b;
  if (second) ds = c;
  float s = (a + b + c) / 2.0f;
  float area = s * (s - a) * (s - b) * (s - c);
  if (!first && !second && ((b + c - a) > 0.f)) ds = (2.0f * sqrtf(area)) / a;
  float sg0 = (s0 > 0.f) ? 1.f : ((s0 < 0.f) ? -1.f : 0.f);
  float sg1 = (s1 > 0.f) ? 1.f : ((s1 < 0.f) ? -1.f : 0.f);
  float m = ((sg1 * sg0) == 1.f) ? 1.f : 0.f;
  return m * ds;
}

// get_error_bound for one ray     ray_sampler.py:222-230
__device__ float error_bound_warp(const float* sz, const float* ss, const float* sd, int M, float beta, int lane) {
  int n = M - 1;
  int C = (n + 31) >> 5;
  int b = lane * C, e = min(n, b + C);
  float fb2 = 4.f * (beta * beta);
  float s1 = 0.f, s2 = 0.f;
  for (int i = b; i < e; ++i) {
    float dist = sz[i + 1] - sz[i];
    float dens = laplace_density(ss[i], beta);
    s1 += dist * dens;
    s2 += (expf(-sd[i] / beta) * (dist * dist)) / fb2;
  }
  float run1 = warp_scan_excl(s1, lane);
  float run2 = warp_scan_excl(s2, lane);
  float mx = -INFINITY;
  bool has_nan = false;
  for (int i = b; i < e; ++i) {
    float dist = sz[i + 1] - sz[i];
    float dens = laplace_density(ss[i], beta);
    run2 += (expf(-sd[i] / beta) * (dist * dist)) / fb2;
    float ex = expf(run2);
    float cl = (ex > 1.e6f) ? 1.e6f : ex;
    float bound = (cl - 1.0f) * expf(-run1);
    run1 += dist * dens;
    if (bound != bound) has_nan = true;
    mx = fmaxf(mx, bound);
  }
  mx = warp_max(mx);
  unsigned any = __ballot_sync(0xffffffffu, has_nan);
  return any ? NAN : mx;
}

// Beta line search of one trip     ray_sampler.py:94-122, :137
__global__ void sampler_beta_kernel(const float* __restrict__ z, const float* __restrict__ sdf, int zcap, int M,
                                    int R, float beta0, float eps, int beta_iters, int trip,
                                    float* __restrict__ beta_state, SamplerState* st, int mmax,
                                    const int* __restrict__ R_dev) {
  if (st->active[trip] == 0) return;
  extern __shared__ float smem[];
  int wpc = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ray = blockIdx.x * wpc + wid;
  if (R_dev) R = min(R, *R_dev);
  if (ray >= R) return;
  float* sz = smem + (size_t)wid * 3 * mmax;
  float* ss = sz + mmax;
  float* sd = ss + mmax;
  const float* zr = z + (size_t)ray * zcap;
  const float* sr = sdf + (size_t)ray * zcap;
  for (int i = lane; i < M; i += 32) {
    sz[i] = zr[i];
    ss[i] = sr[i];
  }
  __syncwarp();
  for (int i = lane; i < M - 1; i += 32) sd[i] = dstar_interval(sz[i], sz[i + 1], ss[i], ss[i + 1]);
  __syncwarp();
  float beta = beta_state[ray];
  float err = error_bound_warp(sz, ss, sd, M, beta0, lane);
  if (err <= eps) beta = beta0;
  float bmin = beta0, bmax = beta;
  // a ray whose error at beta0 is already within eps has bmin == bmax == beta0: every bisection step would evaluate
  // mid = beta0 again and leave the bracket unchanged (ray_sampler.py:116-121), so the loop is skipped — bit-identical
  const int iters = (bmin == bmax) ? 0 : beta_iters;
  for (int j = 0; j < iters; ++j) {
    float mid = (bmin + bmax) / 2.f;
    err = error_bound_warp(sz, ss, sd, M, mid, lane);
    if (err <= eps) bmax = mid;
    if (err > eps) bmin = mid;
  }
  if (lane == 0) {
    beta_state[ray] = bmax;
    if (bmax > beta0) atomicOr(&st->not_converge[trip], 1);
  }
}

// Resampling of one trip: weights / error-bound pdf -> cdf -> inverse-CDF samples -> merge, or the
// final sample set     ray_sampler.py:124-220
__global__ void sampler_resample_kernel(const float* __restrict__ z, const float* __restrict__ sdf, int zcap, int M,
                                        int R, int E, int S, int X, int max_iters, float add_tiny, float near,
                                        int trip, const float* __restrict__ beta_state,
                                        const float* __restrict__ far, SamplerTables tab,
                                        float* __restrict__ z_out, float* __restrict__ sdf_out,
                                        int* __restrict__ pos_new, float* __restrict__ z_final,
                                        SamplerState* st, int mmax, const int* __restrict__ R_dev,
                                        mp_sampler_rng_t rng, float* __restrict__ z_eik) {
  if (st->active[trip] == 0) return;
  if (R_dev) R = min(R, *R_dev);
  const bool cont = (st->not_converge[trip] != 0) && (trip + 1 < max_iters);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (trip + 1 < 8) st->active[trip + 1] = cont ? 1 : 0;
    if (!cont) st->final_trip = trip;
  }
  extern __shared__ float smem[];
  int wpc = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ray = blockIdx.x * wpc + wid;
  if (ray >= R) return;
  float* sz = smem + (size_t)wid * (4 * mmax + E);
  float* ss = sz + mmax;
  float* sp = ss + mmax;      // pdf
  float* sc = sp + mmax;      // cdf
  float* sn = sc + mmax;      // new samples [E]
  const float* zr = z + (size_t)ray * zcap;
  const float* sr = sdf + (size_t)ray * zcap;
  for (int i = lane; i < M; i += 32) {
    sz[i] = zr[i];
    ss[i] = sr[i];
  }
  __syncwarp();
  const float beta = beta_state[ray];
  const float fb2 = 4.f * (beta * beta);
  // pass 1: per-lane chunk sums of the free energy and the error sections
  int C = (M + 31) >> 5;
  int b = lane * C, e = min(M, b + C);
  float s1 = 0.f, s2 = 0.f;
  for (int i = b; i < e; ++i) {
    float dist = (i < M - 1) ? (sz[i + 1] - sz[i]) : 1e10f;
    float dens = laplace_density(ss[i], beta);
    if (i < M - 1) s1 += dist * dens;      // the 1e10 tail interval follows every prefix that is used
    if (cont && i < M - 1) {
      float ds = dstar_interval(sz[i], sz[i + 1], ss[i], ss[i + 1]);
      s2 += (expf(-ds / beta) * (dist * dist)) / fb2;
    }
  }
  float run1 = warp_scan_excl(s1, lane);
  float run2 = warp_scan_excl(s2, lane);
  float psum = 0.f;
  for (int i = b; i < e; ++i) {
    float dist = (i < M - 1) ? (sz[i + 1] - sz[i]) : 1e10f;
    float dens = laplace_density(ss[i], beta);
    float fe = dist * dens;
    float T = expf(-run1);                 // transmittance (exclusive cumsum), :131-132
    float pdf;
    if (cont) {
      float ds = (i < M - 1) ? dstar_interval(sz[i], sz[i + 1], ss[i], ss[i + 1]) : 0.f;
      if (i < M - 1) run2 += (expf(-ds / beta) * (dist * dist)) / fb2;
      float ex = expf(run2);
      float cl = (ex > 1.e6f) ? 1.e6f : ex;
      pdf = (cl - 1.0f) * T + add_tiny;    // :146-148
    } else {
      float alpha = 1.f - expf(-fe);
      pdf = alpha * T + 1e-5f;             // :158-160
    }
    run1 += fe;
    if (i < M - 1) {
      sp[i] = pdf;
      psum += pdf;
    }
  }
  psum = warp_sum(psum);
  __syncwarp();
  // normalise + cdf (M entries: 0, cumsum)
  int n = M - 1;
  int C2 = (n + 31) >> 5;
  int b2 = lane * C2, e2 = min(n, b2 + C2);
  float cs = 0.f;
  for (int i = b2; i < e2; ++i) {
    float p = sp[i] / psum;
    sp[i] = p;
    cs += p;
  }
  float crun = warp_scan_excl(cs, lane);
  for (int i = b2; i < e2; ++i) {
    crun += sp[i];
    sc[i + 1] = crun;
  }
  if (lane == 0) sc[0] = 0.f;
  __syncwarp();
  // inverse CDF     :166-186
  const int N = cont ? E : S;
  // training mode draws the abscissae of the FINAL set at random (ray_sampler.py:171); every other set is linspace
  const bool rnd = !cont && rng.u_final != nullptr;
  const float* u_tab = cont ? tab.u_E : (rnd ? rng.u_final + (size_t)ray * S : tab.u_S);
  for (int j = lane; j < N; j += 32) {
    float u = u_tab[j];
    int inds = upper_bound(sc, M, u);          // searchsorted(right=True)
    int below = max(0, inds - 1);
    int above = min(M - 1, inds);
    float c0 = sc[below], c1 = sc[above];
    float b0 = sz[below], b1 = sz[above];
    float denom = c1 - c0;
    if (denom < 1e-5f) denom = 1.f;
    float t = (u - c0) / denom;
    sn[j] = b0 + t * (b1 - b0);
  }
  __syncwarp();
  // the inverse CDF is monotone up to rounding; repair the (rare) 1-ulp inversions so that the
  // rank merge below equals torch.sort (:189, :209)
  if (rnd) {
    // final set, training mode: sort(cat([z_samples, near, far, z_vals[:, randperm(M)[:X]]]))   :194-209 — nothing is
    // ordered (random abscissae, random extras), so the S+X+2 values are rank-sorted: rank = #smaller + #equal before
    const int T = M / E - 1;                                   // trips before this one = row of the per-trip draws
    const int* perm = rng.extra_perm + (size_t)T * max_iters * E;
    const int n = S + X + 2;
    float* vals = sp;                                          // sp | sc are contiguous: 2 * mmax >= S + X + 2 floats
    for (int k = lane; k < n; k += 32)
      vals[k] = (k < S) ? sn[k] : ((k == S) ? near : ((k == S + 1) ? far[ray] : sz[perm[k - S - 2]]));
    __syncwarp();
    float* zf = z_final + (size_t)ray * n;
    for (int k = lane; k < n; k += 32) {
      const float v = vals[k];
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const float w = vals[j];
        rank += (w < v || (w == v && j < k)) ? 1 : 0;
      }
      zf[rank] = v;
    }
    __syncwarp();
    if (lane == 0 && z_eik) z_eik[ray] = zf[rng.eik_idx[(size_t)T * R + ray]];       // :212-213
    return;
  }
  bool inv = false;
  for (int j = lane + 1; j < N; j += 32) inv |= (sn[j] < sn[j - 1]);
  if (__ballot_sync(0xffffffffu, inv)) {
    if (lane == 0) {
      for (int j = 1; j < N; ++j) {
        float v = sn[j];
        int k = j - 1;
        while (k >= 0 && sn[k] > v) {
          sn[k + 1] = sn[k];
          --k;
        }
        sn[k + 1] = v;
      }
    }
    __syncwarp();
  }
  if (cont) {
    // z_vals, samples_idx = sort(cat([z_vals, samples]))     :189-191  (stable two-way merge)
    float* zo = z_out + (size_t)ray * zcap;
    float* so = sdf_out + (size_t)ray * zcap;
    int* pn = pos_new + (size_t)ray * E;
    for (int i = lane; i < M; i += 32) {
      int p = i + lower_bound(sn, N, sz[i]);
      zo[p] = sz[i];
      so[p] = ss[i];
    }
    for (int j = lane; j < N; j += 32) {
      int p = j + upper_bound(sz, M, sn[j]);
      zo[p] = sn[j];
      pn[j] = p;
    }
  } else {
    // final: sort(cat([z_samples, near, far, z_vals[:, sampling_idx]]))     :194-209
    const int* idx = tab.extra_idx + (size_t)(M / E - 1) * X;
    float* zf = z_final + (size_t)ray * (S + X + 2);
    const float farv = far[ray];
    // list B (sorted): [near, z[idx[0..X)], far]  -> staged in sp
    int NB = X + 2;
    for (int k = lane; k < NB; k += 32) sp[k] = (k == 0) ? near : ((k == NB - 1) ? farv : sz[idx[k - 1]]);
    __syncwarp();
    for (int j = lane; j < N; j += 32) zf[j + lower_bound(sp, NB, sn[j])] = sn[j];
    for (int k = lane; k < NB; k += 32) zf[k + upper_bound(sn, N, sp[k])] = sp[k];
  }
}

__global__ void trips_kernel(const SamplerState* st, int* trips_out) {
  *trips_out = st->final_trip + 1;
}

// inverse-sphere depths: linspace(0,1,32) / bound (ray_sampler.py:215-218); in training mode the UniformSampler
// jitters them too (:32-40), with the draws of the trip count the loop ended on
__global__ void zbg_kernel(const float* tab, int R, float inv_bound, const float* __restrict__ t_rand_bg,
                           const SamplerState* st, float* z_bg) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * 32) return;
  if (!t_rand_bg) {
    z_bg[i] = tab[i & 31];
    return;
  }
  const int j = i & 31;
  auto zu = [&](int k) { return linspace_at(0.f, 1.f, 32, k); };
  const float zj = zu(j);
  const float lower = (j == 0) ? zj : .5f * (zj + zu(j - 1));
  const float upper = (j == 31) ? zj : .5f * (zu(j + 1) + zj);
  const int T = st->final_trip < 0 ? 0 : st->final_trip;
  z_bg[i] = (lower + (upper - lower) * t_rand_bg[(size_t)T * R * 32 + i]) * inv_bound;
}

struct SamplerWs {
  float *zA, *zB, *sA, *sB, *beta, *far, *xc_list;
  int *pos_new, *slot_list;
  SamplerState* st;
  SamplerTables tab;
  void* mlp_ws;
  size_t mlp_ws_bytes;
};

static void sampler_carve(Arena& a, const mp_sampler_cfg_t& c, int R, SamplerWs& w) {
  int E = c.N_samples_eval, S = c.N_samples, X = c.N_samples_extra;
  size_t zcap = (size_t)c.max_total_iters * E;
  w.zA = a.take<float>((size_t)R * zcap);
  w.zB = a.take<float>((size_t)R * zcap);
  w.sA = a.take<float>((size_t)R * zcap);
  w.sB = a.take<float>((size_t)R * zcap);
  w.beta = a.take<float>(R);
  w.far = a.take<float>(R);
  w.pos_new = a.take<int>((size_t)R * E);
  w.xc_list = a.take<float>((size_t)R * E * 3);
  w.slot_list = a.take<int>((size_t)R * E);
  w.st = a.take<SamplerState>(1);
  w.tab.u_E = a.take<float>(E);
  w.tab.u_S = a.take<float>(S);
  w.tab.extra_idx = a.take<int>((size_t)c.max_total_iters * (X > 0 ? X : 1));
  w.tab.z_bg = a.take<float>(32);
  w.mlp_ws_bytes = field_ws_bytes(R * E);
  w.mlp_ws = a.take<char>(w.mlp_ws_bytes);
}

// The whole Algorithm-1 loop for one person.  z_final [R, S+X+2].
int sample_rays(const mp_sampler_cfg_t& c, const Body& body, const Field& field, const float* dirs,
                const float* cam, int R, float* z_final, float* z_bg, int* trips_out, void* ws, size_t ws_bytes,
                cudaStream_t st, const int* R_dev, const mp_sampler_rng_t* rng_in, float* z_eik) {
  mp_sampler_rng_t rng;
  memset(&rng, 0, sizeof(rng));
  if (rng_in) rng = *rng_in;
  const bool training = rng_in != nullptr;
  const int E = c.N_samples_eval, S = c.N_samples, X = c.N_samples_extra;
  MP_REQUIRE(E >= 2 && S >= 1 && X >= 0 && c.max_total_iters >= 1 && c.max_total_iters <= 8,
             "sampler: unsupported configuration (E=%d S=%d X=%d iters=%d)", E, S, X, c.max_total_iters);
  MP_REQUIRE(S <= E, "sampler: N_samples (%d) must not exceed N_samples_eval (%d)", S, E);
  // training mode takes the extras from randperm(M)[:X] (ray_sampler.py:202), which has only min(X, M) entries when the
  // loop ends after one trip (M = E); the row of S+X+2 samples would be padded with whatever the permutation row holds
  MP_REQUIRE(!training || X <= E, "sampler: training mode needs N_samples_extra (%d) <= N_samples_eval (%d)", X, E);
  if (R <= 0) return 0;
  Arena a(ws, ws_bytes);
  SamplerWs w;
  sampler_carve(a, c, R, w);
  MP_TRY(a.fits("sampler"));
  const int zcap = c.max_total_iters * E;
  const float beta0 = sampler_beta(c);
  const float bound_coef = 1.0f / (4.0f * logf((float)(c.eps + 1.0)));     // ray_sampler.py:75
  int tn = max(max(E, S), max(32, c.max_total_iters * max(X, 1)));
  tables_kernel<<<div_up(tn, 128), 128, 0, st>>>(w.tab, E, S, X, c.max_total_iters,
                                                 (float)(1.0 / c.scene_bounding_sphere), w.st);
  MP_LAUNCH_CHECK();
  sampler_init_kernel<<<div_up(R * 32, 128), 128, 0, st>>>(dirs, cam, R, c.scene_bounding_sphere, c.near, E, w.tab.u_E,
                                                      bound_coef, w.zA, zcap, w.beta, w.far, w.st, R_dev, rng.t_rand);
  MP_LAUNCH_CHECK();
  float *zc = w.zA, *zn = w.zB, *sc = w.sA, *sn = w.sB;
  const int mmax = zcap;
  size_t per_warp_beta = (size_t)3 * mmax * sizeof(float);
  size_t per_warp_res = (size_t)(4 * mmax + E) * sizeof(float);
  int wpc_b = clamp_wpc((size_t)(200 * 1024) / per_warp_beta);
  int wpc_r = clamp_wpc((size_t)(200 * 1024) / per_warp_res);
  MP_REQUIRE(per_warp_res <= 220 * 1024, "sampler: N_samples_eval too large for shared memory");
  // every trip's launch asks for warps * per-warp bytes <= 200 KB (or one warp of the longest list)
  const size_t smem_cap = (size_t)200 * 1024;
  MP_CHECK_CUDA(cudaFuncSetAttribute(sampler_beta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)max(smem_cap, (size_t)wpc_b * per_warp_beta)));
  MP_CHECK_CUDA(cudaFuncSetAttribute(sampler_resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)max(smem_cap, (size_t)wpc_r * per_warp_res)));
  const int wpc_for_trip = 8;      // warps (= rays) per block: small blocks spread a 4096-ray batch over all SMs
  for (int t = 0; t < c.max_total_iters; ++t) {
    const int M = (t + 1) * E;
    // SDF of the E new samples of every ray (multiply.py:137-151 under no_grad, ray_sampler.py:82-88)
    // (training mode: the SDF callback does not clamp outliers, multiply.py:142 is eval-only -> exact far search)
    MP_TRY(launch_deform_rays(body, dirs, cam, zc, zcap, t == 0 ? nullptr : w.pos_new, E, E, R, /*prune=*/training ? 0 : 1, sc,
                              zcap, w.xc_list, w.slot_list, &w.st->count[t], nullptr, &w.st->active[t], st, R_dev));
    MlpCall mlp{};
    mlp.x = w.xc_list;
    mlp.slot = w.slot_list;
    mlp.count = &w.st->count[t];
    mlp.cap = R * E;
    mlp.sdf = sc;
    MP_TRY(field_run(field, mlp, w.mlp_ws, w.mlp_ws_bytes, st));
    // shared memory per ray sized for THIS trip's list (M = (t+1) E entries; the final-set staging needs X + 2):
    // trip 0 -- usually the only active one -- then keeps every ray of the batch resident at once instead of
    // 13 warps per SM sized for the longest possible list
    const int stride = max(M, X + 2);
    const size_t pw_b = (size_t)3 * stride * sizeof(float), pw_r = (size_t)(4 * stride + E) * sizeof(float);
    const int wb = min(wpc_for_trip, clamp_wpc((size_t)(200 * 1024) / pw_b));
    const int wr = min(wpc_for_trip, clamp_wpc((size_t)(200 * 1024) / pw_r));
    sampler_beta_kernel<<<div_up(R, wb), wb * 32, wb * pw_b, st>>>(
        zc, sc, zcap, M, R, beta0, c.eps, c.beta_iters, t, w.beta, w.st, stride, R_dev);
    MP_LAUNCH_CHECK();
    sampler_resample_kernel<<<div_up(R, wr), wr * 32, wr * pw_r, st>>>(
        zc, sc, zcap, M, R, E, S, X, c.max_total_iters, c.add_tiny, c.near, t, w.beta, w.far, w.tab, zn, sn,
        w.pos_new, z_final, w.st, stride, R_dev, rng, z_eik);
    MP_LAUNCH_CHECK();
    float* tz = zc; zc = zn; zn = tz;
    float* ts = sc; sc = sn; sn = ts;
  }
  if (trips_out) {
    trips_kernel<<<1, 1, 0, st>>>(w.st, trips_out);
    MP_LAUNCH_CHECK();
  }
  if (z_bg) {
    zbg_kernel<<<div_up(R * 32, 256), 256, 0, st>>>(w.tab.z_bg, R, (float)(1.0 / c.scene_bounding_sphere), rng.t_rand_bg,
                                                    w.st, z_bg);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

size_t sampler_ws_bytes(const mp_sampler_cfg_t& c, int R) {
  Arena a;
  SamplerWs w;
  sampler_carve(a, c, R > 0 ? R : 0, w);
  return a.off;
}

}  // namespace mp

extern "C" {

size_t mp_sampler_workspace_bytes(const mp_sampler_cfg_t* cfg, int R) {
  if (!cfg) return 0;
  return mp::sampler_ws_bytes(*cfg, R);
}

int mp_sample_rays(const mp_sampler_cfg_t* cfg, mp_body_t* body, mp_net_t* field, const float* ray_dirs,
                   const float* cam_loc, int R, float* z_vals, float* z_bg, int* trips_out, void* workspace,
                   size_t workspace_bytes, void* stream) {
  MP_REQUIRE(cfg && body && field && ray_dirs && cam_loc && z_vals, "mp_sample_rays: null argument");
  MP_REQUIRE(body->b.tfs, "mp_sample_rays: body has no pose (call mp_body_set_pose)");
  return mp::sample_rays(*cfg, body->b, field->f, ray_dirs, cam_loc, R, z_vals, z_bg, trips_out, workspace,
                         workspace_bytes, (cudaStream_t)stream, nullptr, nullptr, nullptr);
}

int mp_sample_rays_train(const mp_sampler_cfg_t* cfg, mp_body_t* body, mp_net_t* field, const float* ray_dirs,
                         const float* cam_loc, int R, const mp_sampler_rng_t* rng, float* z_vals, float* z_bg,
                         float* z_eik, int* trips_out, void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(cfg && body && field && ray_dirs && cam_loc && z_vals && rng, "mp_sample_rays_train: null argument");
  MP_REQUIRE(rng->t_rand && rng->u_final && rng->eik_idx && (cfg->N_samples_extra == 0 || rng->extra_perm),
             "mp_sample_rays_train: incomplete random draws");
  MP_REQUIRE(body->b.tfs, "mp_sample_rays_train: body has no pose (call mp_body_set_pose)");
  return mp::sample_rays(*cfg, body->b, field->f, ray_dirs, cam_loc, R, z_vals, z_bg, trips_out, workspace,
                         workspace_bytes, (cudaStream_t)stream, nullptr, rng, z_eik);
}
}
