// NeRF++ inverted-sphere background.
//   reference: /root/reference/code/lib/model/multiply.py
//     background rendering block   :514-539
//     bg_volume_rendering          :682-696  (AbsDensity, lib/model/density.py:32-34)
//     depth2pts_outside            :698-726
//   and the inverse-sphere sample depths of ray_sampler.py:215-218 / multiply.py:482-484.
#include "common.cuh"

namespace mp {

__device__ __forceinline__ float bg_linspace32(int i) {
  float step = 1.0f / 31.0f;
  return (i < 16) ? fmaf(step, (float)i, 0.f) : fmaf(-step, (float)(31 - i), 1.0f);
}

// one thread per (ray, sample): depth = flip(linspace(0,1,32) / bound)[j] ; pts = depth2pts_outside(o, d, depth)
// inverse-sphere depth k of ray r: linspace(0,1,32)[k] / bound (ray_sampler.py:215-218); with t_rand (training mode:
// the UniformSampler of the inverse sphere sees model.training, ray_sampler.py:32-40) stratified between the midpoints
__device__ __forceinline__ float bg_depth(int r, int k, float inv_bound, const float* __restrict__ t_rand) {
  float zk = bg_linspace32(k);
  if (t_rand) {
    float lower = (k == 0) ? zk : .5f * (zk + bg_linspace32(k - 1));
    float upper = (k == 31) ? zk : .5f * (bg_linspace32(k + 1) + zk);
    zk = lower + (upper - lower) * t_rand[(size_t)r * 32 + k];
  }
  return zk * inv_bound;
}

__global__ void bg_points_kernel(const float* __restrict__ dirs, const float* __restrict__ cam, int R, float bound,
                                 float inv_bound, float* __restrict__ pts, float* __restrict__ dirs_out,
                                 const float* __restrict__ t_rand) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * 32) return;
  int r = idx >> 5, j = idx & 31;
  float depth = bg_depth(r, 31 - j, inv_bound, t_rand);     // torch.flip(z_vals_bg)   multiply.py:516
  const float* o = cam + 3 * r;
  const float* d = dirs + 3 * r;
  float odd = d[0] * o[0] + d[1] * o[1] + d[2] * o[2];
  float oo = o[0] * o[0] + o[1] * o[1] + o[2] * o[2];
  float under = odd * odd - (oo - bound * bound);
  float dsph = sqrtf(under) - odd;
  float ps[3], pm[3];
  for (int k = 0; k < 3; ++k) {
    ps[k] = o[k] + dsph * d[k];
    pm[k] = o[k] - odd * d[k];
  }
  float pmn = sqrtf(pm[0] * pm[0] + pm[1] * pm[1] + pm[2] * pm[2]);
  float ax[3] = {o[1] * ps[2] - o[2] * ps[1], o[2] * ps[0] - o[0] * ps[2], o[0] * ps[1] - o[1] * ps[0]};
  float an = sqrtf(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
  // a ray through the sphere's centre has o x p_sphere = 0 and a rotation angle of exactly 0: a zero axis gives the
  // limit p_sphere / |p_sphere| (the reference divides 0 by 0 here and returns NaN)
  for (int k = 0; k < 3; ++k) ax[k] = (an > 0.f) ? ax[k] / an : 0.f;
  float phi = asinf(pmn / bound);
  float theta = asinf(pmn * depth);
  float ang = phi - theta;
  float ca = cosf(ang), sa = sinf(ang);
  float cr[3] = {ax[1] * ps[2] - ax[2] * ps[1], ax[2] * ps[0] - ax[0] * ps[2], ax[0] * ps[1] - ax[1] * ps[0]};
  float dt = ax[0] * ps[0] + ax[1] * ps[1] + ax[2] * ps[2];
  float pn[3];
  for (int k = 0; k < 3; ++k) pn[k] = ps[k] * ca + cr[k] * sa + ax[k] * dt * (1.f - ca);
  float nn = sqrtf(pn[0] * pn[0] + pn[1] * pn[1] + pn[2] * pn[2]);
  float* q = pts + 4 * (size_t)idx;
  q[0] = pn[0] / nn;
  q[1] = pn[1] / nn;
  q[2] = pn[2] / nn;
  q[3] = depth;
  dirs_out[3 * (size_t)idx] = d[0];
  dirs_out[3 * (size_t)idx + 1] = d[1];
  dirs_out[3 * (size_t)idx + 2] = d[2];
}

// one warp per ray, lane = sample     multiply.py:682-696, :539
__global__ void bg_composite_kernel(const float* __restrict__ sdf, const float* __restrict__ rgb, int R,
                                    float inv_bound, float* __restrict__ out, const float* __restrict__ t_rand) {
  int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= R) return;
  size_t i = (size_t)w * 32 + lane;
  float dens = fabsf(sdf[i]);
  float zc = bg_depth(w, 31 - lane, inv_bound, t_rand);
  float zn = (lane < 31) ? bg_depth(w, 30 - lane, inv_bound, t_rand) : 0.f;
  float dist = (lane < 31) ? (zc - zn) : 1e10f;
  float fe = dist * dens;
  float T = expf(-warp_scan_excl(fe, lane));
  float wgt = (1.f - expf(-fe)) * T;
  for (int k = 0; k < 3; ++k) {
    float v = warp_sum(wgt * rgb[3 * i + k]);
    if (lane == 0) out[3 * (size_t)w + k] = v;
  }
}

// Backward of bg_composite_kernel, one warp per ray, lane = sample.  With fe_j = dist_j |s_j|, T_j = exp(-sum_{k<j} fe_k),
// w_j = T_j (1 - exp(-fe_j)) and h_j = <d bg_rgb, rgb_j>:
//   dL/dfe_j = T_{j+1} h_j - sum_{k>j} w_k h_k ;  dL/ds_j = dL/dfe_j dist_j sign(s_j) ;  dL/drgb_j = w_j d bg_rgb
// (sign(0) = 0: AbsDensity's autograd kink).  The last interval is 1e10 long, as in the forward.
__global__ void bg_composite_backward_kernel(const float* __restrict__ sdf, const float* __restrict__ rgb, int R,
                                             float inv_bound, const float* __restrict__ t_rand,
                                             const float* __restrict__ d_out, float* __restrict__ d_sdf,
                                             float* __restrict__ d_rgb) {
  int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= R) return;
  size_t i = (size_t)w * 32 + lane;
  float s = sdf[i];
  float dens = fabsf(s);
  float zc = bg_depth(w, 31 - lane, inv_bound, t_rand);
  float zn = (lane < 31) ? bg_depth(w, 30 - lane, inv_bound, t_rand) : 0.f;
  float dist = (lane < 31) ? (zc - zn) : 1e10f;
  float fe = dist * dens;
  float T = expf(-warp_scan_excl(fe, lane));
  float ex = expf(-fe);
  float wgt = (1.f - ex) * T;
  const float d0 = d_out[3 * (size_t)w], d1 = d_out[3 * (size_t)w + 1], d2 = d_out[3 * (size_t)w + 2];
  float h = d0 * rgb[3 * i] + d1 * rgb[3 * i + 1] + d2 * rgb[3 * i + 2];
  // exclusive suffix sum of w h over the lanes above
  float incl = wgt * h;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += t;
  }
  float suf = __shfl_down_sync(0xffffffffu, incl, 1);
  if (lane == 31) suf = 0.f;
  float dfe = (T * ex) * h - suf;
  float sg = (s > 0.f) ? 1.f : ((s < 0.f) ? -1.f : 0.f);
  d_sdf[i] = dfe * dist * sg;
  d_rgb[3 * i] = wgt * d0;
  d_rgb[3 * i + 1] = wgt * d1;
  d_rgb[3 * i + 2] = wgt * d2;
}

// 32 samples per ray: points, view directions, colour, SDF, then the MLP's workspace
struct BgWs {
  float *pts, *dexp, *rgb, *sdf;
  void* mlp;
  size_t mlp_bytes;
};
static void bg_carve(Arena& a, int R, BgWs& w) {
  const int N = R * 32;
  w.pts = a.take<float>((size_t)N * 4);
  w.dexp = a.take<float>((size_t)N * 3);
  w.rgb = a.take<float>((size_t)N * 3);
  w.sdf = a.take<float>(N);
  w.mlp_bytes = field_ws_bytes(N);
  w.mlp = a.take<char>(w.mlp_bytes);
}

size_t bg_ws_bytes(int R) {
  Arena a;
  BgWs w;
  bg_carve(a, R > 0 ? R : 0, w);
  return a.off;
}

int render_background(const Field& f, const float* dirs, const float* cam, int R, float bound, float* bg_rgb,
                      void* ws, size_t ws_bytes, cudaStream_t st, const float* t_rand, float* tap_sdf, float* tap_rgb) {
  if (R <= 0) return 0;
  Arena a(ws, ws_bytes);
  BgWs w;
  bg_carve(a, R, w);
  MP_TRY(a.fits("background"));
  const int N = R * 32;
  float inv_bound = (float)(1.0 / bound);
  bg_points_kernel<<<div_up(N, 256), 256, 0, st>>>(dirs, cam, R, bound, inv_bound, w.pts, w.dexp, t_rand);
  MP_LAUNCH_CHECK();
  MlpCall c{};
  c.x = w.pts;
  c.cap = N;
  c.dirs = w.dexp;
  c.sdf = w.sdf;
  c.rgb = w.rgb;
  MP_TRY(field_run(f, c, w.mlp, w.mlp_bytes, st));
  if (tap_sdf) MP_CHECK_CUDA(cudaMemcpyAsync(tap_sdf, w.sdf, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (tap_rgb)
    MP_CHECK_CUDA(cudaMemcpyAsync(tap_rgb, w.rgb, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  bg_composite_kernel<<<div_up(N, 256), 256, 0, st>>>(w.sdf, w.rgb, R, inv_bound, bg_rgb, t_rand);
  MP_LAUNCH_CHECK();
  return 0;
}

}  // namespace mp

extern "C" {
size_t mp_background_workspace_bytes(int R) { return mp::bg_ws_bytes(R); }

int mp_background(mp_net_t* bg_field, const float* ray_dirs, const float* cam_loc, int R, float bound_r, float* bg_rgb,
                  void* workspace, size_t workspace_bytes, void* stream) {
  MP_REQUIRE(bg_field && ray_dirs && cam_loc && bg_rgb, "mp_background: null argument");
  return mp::render_background(bg_field->f, ray_dirs, cam_loc, R, bound_r, bg_rgb, workspace, workspace_bytes,
                               (cudaStream_t)stream, nullptr, nullptr, nullptr);
}

int mp_bg_composite_backward(const float* bg_sdf, const float* bg_rgb_samples, int R, float bound_r,
                             const float* t_rand_bg, const float* d_bg_rgb, float* d_bg_sdf, float* d_bg_rgb_samples,
                             void* stream) {
  MP_REQUIRE(bg_sdf && bg_rgb_samples && d_bg_rgb && d_bg_sdf && d_bg_rgb_samples,
             "mp_bg_composite_backward: null argument");
  if (R <= 0) return 0;
  float inv_bound = (float)(1.0 / bound_r);
  mp::bg_composite_backward_kernel<<<mp::div_up(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      bg_sdf, bg_rgb_samples, R, inv_bound, t_rand_bg, d_bg_rgb, d_bg_sdf, d_bg_rgb_samples);
  MP_LAUNCH_CHECK();
  return 0;
}
}
