// Packing of ImplicitNet / RenderingNet parameters into kernel layouts.
//   reference: /root/reference/code/lib/model/networks.py
//     weight norm      W = g * v / ||v||_row                      (:82-83, :257-258)
//     cond concat      layer 0 input = [embed(x), cond]            (:163-164)  -> folded into the bias per call
//     skip             layer 4 input = [h3, embed(x)] / sqrt(2)    (:166-167)  -> 1/sqrt(2) folded into W4
//     lin_pose         colour input [x, n, lin_pose(pose), feat]   (:277-281)  -> folded into the bias per call
#include "common.cuh"

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

__global__ void copy_kernel(const float* __restrict__ s, float* __restrict__ d, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = s[i];
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

}  // namespace mp

extern "C" {

size_t mp_field_pack_bytes(void) {
  // fp32: 2 copies (natural + transposed) of <= 14 layers of <= 257x325 + small vectors; tc blobs
  size_t fp32 = (size_t)14 * 2 * 260 * 328 * sizeof(float) + (1u << 20);
  return fp32 + mp::tc_pack_bytes() + (1u << 16);
}

int mp_field_pack(const mp_implicit_desc_t* imp, const mp_render_desc_t* ren, int is_background, void* storage,
                  size_t storage_bytes, mp_net_t** out, void* stream) {
  using namespace mp;
  MP_REQUIRE(imp && ren && storage && out, "mp_field_pack: null argument (both networks are required)");
  MP_REQUIRE(storage_bytes >= mp_field_pack_bytes(), "mp_field_pack: storage too small (%zu < %zu)", storage_bytes,
             mp_field_pack_bytes());
  MP_REQUIRE(imp->lin.n_layers == 9, "mp_field_pack: ImplicitNet must have 9 linear layers (got %d)",
             imp->lin.n_layers);
  MP_REQUIRE(imp->skip_layer == 4, "mp_field_pack: skip_in must be [4]");
  Arena a(storage, storage_bytes);
  MP_TRY(a.fits("mp_field_pack", "storage"));     // the base's alignment; the layout is checked after its carve below
  cudaStream_t st = (cudaStream_t)stream;
  mp_net* h = new mp_net();
  Field& f = h->f;
  memset(&f, 0, sizeof(f));
  f.is_bg = is_background;
  f.d_in = imp->d_in;
  f.multires = imp->multires;
  f.emb_dim = imp->d_in * (1 + 2 * imp->multires);
  f.cond_dim = imp->cond_dim;
  f.skip_layer = imp->skip_layer;
  f.n_imp = imp->lin.n_layers;
  f.storage = (char*)storage;
  f.storage_bytes = storage_bytes;
  const int E = f.emb_dim;
  int rc = 0;
  // padded tails of biases / weight tiles must read as zero (0 * garbage could be NaN)
  MP_CHECK_CUDA(cudaMemsetAsync(storage, 0, mp_field_pack_bytes(), st));
  // ---- implicit net -------------------------------------------------------------------
  float* nat[MP_MAX_LAYERS];
  for (int l = 0; l < f.n_imp && rc == 0; ++l) {
    int in = imp->lin.in_dim[l], o = imp->lin.out_dim[l];
    f.imp_in[l] = in;
    f.imp_out[l] = o;
    bool ok = true;
    if (l == 0) ok = (in == E + f.cond_dim) && o == kHidden;
    else if (l == f.skip_layer - 1) ok = (in == kHidden) && (o == kHidden - E);
    else if (l == f.n_imp - 1) ok = (in == kHidden) && (o == kHidden + 1);
    else ok = (in == kHidden) && (o == kHidden);
    if (!ok) {
      set_error("mp_field_pack: implicit layer %d has unsupported shape %dx%d", l, o, in);
      rc = -1;
      break;
    }
    nat[l] = a.take<float>((size_t)o * in);
    f.imp_W[l] = nat[l];
    f.imp_Wt[l] = a.take<float>((size_t)in * o);
    f.imp_b[l] = a.take<float>(o < 264 ? 264 : o);   // padded: the tensor-core epilogue reads 256 columns
    if (!a.ok) break;
    float scale = (l == f.skip_layer) ? (float)(1.0 / sqrt(2.0)) : 1.0f;
    rc = fold(imp->lin.weight_v[l], imp->lin.weight_g[l], o, in, scale, nat[l], st);
    if (rc) break;
    rc = tcols(nat[l], o, in, 0, in, f.imp_Wt[l], o, st);
    if (rc) break;
    copy_kernel<<<div_up(o, 256), 256, 0, st>>>(imp->lin.bias[l], f.imp_b[l], o);
    g_launches++;
  }
  if (rc == 0 && a.ok) {
    f.imp_W0cond = f.imp_Wt[0] + (size_t)E * kHidden;   // rows E.. of the transposed layer-0 weights
    f.imp_b0_eff = a.take<float>(kHidden);
  }
  // ---- rendering net ------------------------------------------------------------------
  f.n_ren = ren->lin.n_layers;
  f.ren_mode = ren->mode;
  f.multires_view = ren->multires_view;
  float* rnat[MP_MAX_LAYERS];
  if (rc == 0 && a.ok) {
    int in0 = ren->lin.in_dim[0], out0 = ren->lin.out_dim[0];
    if (ren->mode == 0) {
      f.ren_extra = 6;
      f.ren_cond_dim = 69;
      if (in0 != 6 + 8 + kHidden || !ren->lin_pose_weight || !ren->lin_pose_bias) {
        set_error("mp_field_pack: pose_no_view colour net must take 270 inputs and carry lin_pose");
        rc = -1;
      }
    } else {
      f.ren_extra = 3 * (1 + 2 * ren->multires_view);
      f.ren_cond_dim = 32;
      if (in0 != f.ren_extra + 32 + kHidden) {
        set_error("mp_field_pack: nerf_frame_encoding colour net has unsupported input width %d", in0);
        rc = -1;
      }
    }
    for (int l = 0; l < f.n_ren && rc == 0; ++l) {
      int in = ren->lin.in_dim[l], o = ren->lin.out_dim[l];
      f.ren_in[l] = in;
      f.ren_out[l] = o;
      rnat[l] = a.take<float>((size_t)o * in);
      f.ren_W[l] = rnat[l];
      f.ren_Wt[l] = a.take<float>((size_t)in * o);
      f.ren_b[l] = a.take<float>(o < 264 ? 264 : o);
      if (!a.ok) break;
      rc = fold(ren->lin.weight_v[l], ren->lin.weight_g[l], o, in, 1.0f, rnat[l], st);
      if (rc) break;
      if (l == 0) {
        // Wt0 rows: [extra inputs | feature block]; the conditioning columns go to ren_W0cond
        int cpos = f.ren_extra, cw = (ren->mode == 0) ? 8 : 32;
        rc = tcols(rnat[0], o, in, 0, f.ren_extra, f.ren_Wt[0], o, st);
        if (rc) break;
        rc = tcols(rnat[0], o, in, cpos + cw, kHidden, f.ren_Wt[0] + (size_t)f.ren_extra * o, o, st);
        if (rc) break;
        f.ren_in[0] = f.ren_extra + kHidden;
      } else {
        rc = tcols(rnat[l], o, in, 0, in, f.ren_Wt[l], o, st);
        if (rc) break;
      }
      copy_kernel<<<div_up(o, 256), 256, 0, st>>>(ren->lin.bias[l], f.ren_b[l], o);
      g_launches++;
    }
    if (rc == 0 && a.ok) {
      f.ren_b0_eff = a.take<float>(out0 < 264 ? 264 : out0);
      f.ren_b0_base = a.take<float>(out0);
      f.ren_W0cond = a.take<float>((size_t)f.ren_cond_dim * out0);
      if (a.ok) {
        if (ren->mode == 0) {
          pose_fold_kernel<<<div_up(out0, 128), 128, 0, st>>>(rnat[0], in0, out0, f.ren_b[0], ren->lin_pose_weight,
                                                              ren->lin_pose_bias, 8, 69, 6, f.ren_W0cond,
                                                              f.ren_b0_base);
          g_launches++;
        } else {
          rc = tcols(rnat[0], out0, in0, f.ren_extra, 32, f.ren_W0cond, out0, st);
          copy_kernel<<<div_up(out0, 256), 256, 0, st>>>(f.ren_b[0], f.ren_b0_base, out0);
          g_launches++;
        }
      }
    }
  }
  if (rc == 0 && !a.ok) {
    set_error("mp_field_pack: arena overflow (need %zu bytes)", a.off);
    rc = -1;
  }
  if (rc == 0) rc = tc_pack(f, a, st);
  if (rc == 0 && cudaGetLastError() != cudaSuccess) {
    set_error("mp_field_pack: kernel launch failed");
    rc = -3;
  }
  if (rc) {
    tc_free(f);
    delete h;
    return rc;
  }
  *out = h;
  return 0;
}

void mp_field_free(mp_net_t* f) {
  if (f) mp::tc_free(f->f);
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
