// Packing of ImplicitNet / RenderingNet parameters into kernel layouts.
//   reference: /root/reference/code/lib/model/networks.py
//     weight norm      W = g * v / ||v||_row                      (:82-83, :257-258)
//     cond concat      layer 0 input = [embed(x), cond]            (:163-164)  -> folded into the bias per call
//     skip             layer 4 input = [h3, embed(x)] / sqrt(2)    (:166-167)  -> 1/sqrt(2) folded into W4
//     lin_pose         colour input [x, n, lin_pose(pose), feat]   (:277-281)  -> folded into the bias per call
#include "common.cuh"
#include <memory>

namespace mp {

// W_nat[o][i] = (g ? g[o] * v[o][i] / ||v[o]|| : v[o][i]) * scale ; one warp per output row
__global__ void fold_kernel(const float* __restrict__ v, const float* __restrict__ g, int out, int in, float scale,
                            float* __restrict__ W) {
  int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (o >= out) return;
  const float* row = v + (size_t)o * in;
  float f = 1.f;
  if (g) {
    float s = 0.f;
    for (int i = lane; i < in; i += 32) s = fmaf(row[i], row[i], s);
    s = warp_sum(s);
    f = g[o] / sqrtf(s);
  }
  for (int i = lane; i < in; i += 32) W[(size_t)o * in + i] = (row[i] * f) * scale;
}

// Wt[k][o] = W[o][col_off + k]  for k < ncols   (Wt row stride = ldt)
__global__ void transpose_cols_kernel(const float* __restrict__ W, int out, int in, int col_off, int ncols,
                                      float* __restrict__ Wt, int ldt) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ncols * out) return;
  int k = idx / out, o = idx - k * out;
  Wt[(size_t)k * ldt + o] = W[(size_t)o * in + col_off + k];
}

// out[o] = base[o] + sum_k M[k][o] * c[k]      (M is [K][out], i.e. transposed)
__global__ void bias_fold_kernel(const float* __restrict__ base, const float* __restrict__ Mt, const float* __restrict__ c,
                                 int K, int out, float* __restrict__ dst) {
  int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= out) return;
  float s = base[o];
  for (int k = 0; k < K; ++k) s = fmaf(Mt[(size_t)k * out + o], c[k], s);
  dst[o] = s;
}

// colour mode 0: M[k][o] = sum_j W0[o][6+j] * Wp[j][k]  (69 x out), base[o] = b0[o] + sum_j W0[o][6+j]*bp[j]
__global__ void pose_fold_kernel(const float* __restrict__ W0, int in0, int out0, const float* __restrict__ b0,
                                 const float* __restrict__ Wp, const float* __restrict__ bp, int pdim, int cdim,
                                 int col_off, float* __restrict__ Mt, float* __restrict__ base) {
  int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= out0) return;
  const float* w = W0 + (size_t)o * in0 + col_off;
  float s = b0[o];
  for (int j = 0; j < pdim; ++j) s = fmaf(w[j], bp[j], s);
  base[o] = s;
  for (int k = 0; k < cdim; ++k) {
    float m = 0.f;
    for (int j = 0; j < pdim; ++j) m = fmaf(w[j], Wp[j * cdim + k], m);
    Mt[(size_t)k * out0 + o] = m;
  }
}

__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, float* __restrict__ d) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = a[i] + b[i];
}

static int fold(const float* v, const float* g, int out, int in, float scale, float* W, cudaStream_t st) {
  fold_kernel<<<div_up(out, 8), 256, 0, st>>>(v, g, out, in, scale, W);
  MP_LAUNCH_CHECK();
  return 0;
}
static int tcols(const float* W, int out, int in, int off, int n, float* Wt, int ldt, cudaStream_t st) {
  transpose_cols_kernel<<<div_up(n * out, 256), 256, 0, st>>>(W, out, in, off, n, Wt, ldt);
  MP_LAUNCH_CHECK();
  return 0;
}
static int copy(float* dst, const float* src, int n, cudaStream_t st) {
  MP_CHECK_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// Every condition the pack sets on the two networks, checked on the host from the descriptors' dimensions and whether
// lin_pose is there: fills the field's dimensions and decides whether the tensor-core engine gets a full program for it
// (the fused foreground shade chain or the background chain).
static int field_check(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background, Field& f) {
  MP_REQUIRE(imp->lin.n_layers == 9, "mp_field_pack: ImplicitNet must have 9 linear layers (got %d)",
             imp->lin.n_layers);
  MP_REQUIRE(imp->skip_layer == 4, "mp_field_pack: skip_in must be [4]");
  MP_REQUIRE(ren->lin.n_layers >= 1 && ren->lin.n_layers <= MP_MAX_LAYERS,
             "mp_field_pack: RenderingNet must have 1 to %d linear layers (got %d)", MP_MAX_LAYERS, ren->lin.n_layers);
  f.is_bg = is_background;
  f.d_in = imp->d_in;
  f.multires = imp->multires;
  f.emb_dim = imp->d_in * (1 + 2 * imp->multires);
  f.cond_dim = imp->cond_dim;
  f.skip_layer = imp->skip_layer;
  f.n_imp = imp->lin.n_layers;
  const int E = f.emb_dim;
  for (int l = 0; l < f.n_imp; ++l) {
    const int in = imp->lin.in_dim[l], o = imp->lin.out_dim[l];
    bool ok;
    if (l == 0) ok = (in == E + f.cond_dim) && o == kHidden;
    else if (l == f.skip_layer - 1) ok = (in == kHidden) && (o == kHidden - E);
    else if (l == f.n_imp - 1) ok = (in == kHidden) && (o == kHidden + 1);
    else ok = (in == kHidden) && (o == kHidden);
    MP_REQUIRE(ok, "mp_field_pack: implicit layer %d has unsupported shape %dx%d", l, o, in);
    f.imp_in[l] = in;
    f.imp_out[l] = o;
  }
  f.n_ren = ren->lin.n_layers;
  f.ren_mode = ren->mode;
  f.multires_view = ren->multires_view;
  for (int l = 0; l < f.n_ren; ++l) {
    f.ren_in[l] = ren->lin.in_dim[l];
    f.ren_out[l] = ren->lin.out_dim[l];
  }
  if (ren->mode == 0) {
    f.ren_extra = 6;
    f.ren_cond_dim = 69;
    MP_REQUIRE(f.ren_in[0] == 6 + 8 + kHidden && ren->lin_pose_weight && ren->lin_pose_bias,
               "mp_field_pack: pose_no_view colour net must take 270 inputs and carry lin_pose");
  } else {
    f.ren_extra = 3 * (1 + 2 * ren->multires_view);
    f.ren_cond_dim = 32;
    MP_REQUIRE(f.ren_in[0] == f.ren_extra + 32 + kHidden,
               "mp_field_pack: nerf_frame_encoding colour net has unsupported input width %d", f.ren_in[0]);
  }
  const bool fg_chain = (f.ren_mode == 0) && (f.n_ren == 5) && f.ren_out[0] == kHidden;
  const bool bg_chain = (f.ren_mode == 1) && (f.n_ren == 2) && f.ren_out[0] <= kHidden && f.ren_extra <= 27;
  MP_REQUIRE(!fg_chain || (f.d_in <= 4 && 1 + 2 * f.multires <= 14),
             "tc_pack: the final-gradient step keeps 1 + 2 * multires <= 14 embedding columns per axis");
  f.tc_full = fg_chain || bg_chain;
  return 0;
}

// The whole storage of a packed field, one take per buffer: the fp32 layers (natural and transposed weights, biases
// padded to 264 because the tensor-core epilogue reads 256 columns), the per-call folded biases and conditioning
// columns, then the tensor-core share (tc_pack_carve).  On a sizing Arena it only measures.
static void field_carve(Arena& a, Field& f) {
  for (int l = 0; l < f.n_imp; ++l) {
    const int in = f.imp_in[l], o = f.imp_out[l];
    f.imp_W[l] = a.take<float>((size_t)o * in);
    f.imp_Wt[l] = a.take<float>((size_t)in * o);
    f.imp_b[l] = a.take<float>(o < 264 ? 264 : o);
  }
  f.imp_b0_eff = a.take<float>(kHidden);
  for (int l = 0; l < f.n_ren; ++l) {
    const int in = f.ren_in[l], o = f.ren_out[l];
    f.ren_W[l] = a.take<float>((size_t)o * in);
    f.ren_Wt[l] = a.take<float>((size_t)in * o);
    f.ren_b[l] = a.take<float>(o < 264 ? 264 : o);
  }
  const int out0 = f.ren_out[0];
  f.ren_b0_eff = a.take<float>(out0 < 264 ? 264 : out0);
  f.ren_b0_base = a.take<float>(out0);
  f.ren_W0cond = a.take<float>((size_t)f.ren_cond_dim * out0);
  tc_pack_carve(a, f);
}

// The fp32 layers into the zeroed storage: weight norm and the skip's 1/sqrt(2) folded in, natural and transposed, and
// colour layer 0's conditioning columns split off for mp_field_set_cond.
static int field_fold(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, Field& f, cudaStream_t st) {
  for (int l = 0; l < f.n_imp; ++l) {
    const int in = f.imp_in[l], o = f.imp_out[l];
    const float scale = (l == f.skip_layer) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    MP_TRY(fold(imp->lin.weight_v[l], imp->lin.weight_g[l], o, in, scale, f.imp_W[l], st));
    MP_TRY(tcols(f.imp_W[l], o, in, 0, in, f.imp_Wt[l], o, st));
    MP_TRY(copy(f.imp_b[l], imp->lin.bias[l], o, st));
  }
  f.imp_W0cond = f.imp_Wt[0] + (size_t)f.emb_dim * kHidden;   // rows E.. of the transposed layer-0 weights
  for (int l = 0; l < f.n_ren; ++l) {
    const int in = f.ren_in[l], o = f.ren_out[l];
    MP_TRY(fold(ren->lin.weight_v[l], ren->lin.weight_g[l], o, in, 1.0f, f.ren_W[l], st));
    if (l == 0) {
      // Wt0 rows: [extra inputs | feature block]; the conditioning columns go to ren_W0cond
      const int cpos = f.ren_extra, cw = (f.ren_mode == 0) ? 8 : 32;
      MP_TRY(tcols(f.ren_W[0], o, in, 0, f.ren_extra, f.ren_Wt[0], o, st));
      MP_TRY(tcols(f.ren_W[0], o, in, cpos + cw, kHidden, f.ren_Wt[0] + (size_t)f.ren_extra * o, o, st));
    } else {
      MP_TRY(tcols(f.ren_W[l], o, in, 0, in, f.ren_Wt[l], o, st));
    }
    MP_TRY(copy(f.ren_b[l], ren->lin.bias[l], o, st));
  }
  const int in0 = f.ren_in[0], out0 = f.ren_out[0];
  if (f.ren_mode == 0) {
    pose_fold_kernel<<<div_up(out0, 128), 128, 0, st>>>(f.ren_W[0], in0, out0, f.ren_b[0], ren->lin_pose_weight,
                                                        ren->lin_pose_bias, 8, 69, 6, f.ren_W0cond, f.ren_b0_base);
    MP_LAUNCH_CHECK();
  } else {
    MP_TRY(tcols(f.ren_W[0], out0, in0, f.ren_extra, 32, f.ren_W0cond, out0, st));
    MP_TRY(copy(f.ren_b0_base, f.ren_b[0], out0, st));
  }
  return 0;
}

}  // namespace mp

extern "C" {

size_t mp_field_pack_bytes(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background) {
  mp::Field f{};
  if (!imp || !ren || mp::field_check(imp, ren, is_background, f) != 0) return 0;
  mp::Arena a;
  mp::field_carve(a, f);
  return a.off;
}

int mp_field_pack(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background, void* storage,
                  size_t storage_bytes, mp_net_t** out, void* stream) {
  using namespace mp;
  MP_REQUIRE(imp && ren && storage && out, "mp_field_pack: null argument (both networks are required)");
  std::unique_ptr<mp_net, void (*)(mp_net*)> h(new mp_net(), mp_field_free);
  Field& f = h->f;
  MP_TRY(field_check(imp, ren, is_background, f));
  f.tc = tc_new();
  Arena a(storage, storage_bytes);
  field_carve(a, f);
  MP_TRY(a.fits("mp_field_pack", "storage"));
  cudaStream_t st = (cudaStream_t)stream;
  // padded tails of biases / weight tiles must read as zero (0 * garbage could be NaN)
  MP_CHECK_CUDA(cudaMemsetAsync(storage, 0, a.off, st));
  MP_TRY(field_fold(imp, ren, f, st));
  MP_TRY(tc_pack(f, st));
  *out = h.release();
  return 0;
}

void mp_field_free(mp_net_t* f) {
  if (f) mp::tc_free(f->f.tc);
  delete f;
}

int mp_field_set_cond(mp_net_t* h, const float* cond, void* stream) {
  using namespace mp;
  MP_REQUIRE(h && cond, "mp_field_set_cond: null argument");
  Field& f = h->f;
  cudaStream_t st = (cudaStream_t)stream;
  bias_fold_kernel<<<div_up(kHidden, 128), 128, 0, st>>>(f.imp_b[0], f.imp_W0cond, cond, f.cond_dim, kHidden,
                                                         f.imp_b0_eff);
  MP_LAUNCH_CHECK();
  int out0 = f.ren_out[0];
  bias_fold_kernel<<<div_up(out0, 128), 128, 0, st>>>(f.ren_b0_base, f.ren_W0cond, cond, f.ren_cond_dim, out0,
                                                      f.ren_b0_eff);
  MP_LAUNCH_CHECK();
  if (f.ren_b0_fold) {
    add_vec_kernel<<<div_up(out0, 128), 128, 0, st>>>(f.ren_b0_eff, f.ren_cb, out0, f.ren_b0_fold);
    MP_LAUNCH_CHECK();
  }
  return 0;
}
}
