// fp32 SIMT engine for the ImplicitNet / RenderingNet stacks (validation engine, engine = 0).
//   reference: /root/reference/code/lib/model/networks.py:126-208 (ImplicitNet.forward),
//              :263-312 (RenderingNet.forward), embedders.py:8-34,
//              lib/model/multiply.py:620-661 (forward_gradient: d sdf / d x_c, normals)
// Plain tiled SGEMM per layer with the activation fused into the store; activations live in
// global memory between layers.  It exists so that the tensor-core engine (mlp_tc.cu) can be
// checked against an independent fp32 implementation ON THE GPU and so the pipeline is
// testable end to end; it is not the fast path.
#include "common.cuh"

namespace mp {

enum { ACT_NONE = 0, ACT_SOFTPLUS = 1, ACT_RELU = 2, ACT_SIGMOID = 3 };

__global__ void sub_count_kernel(const int* c, int s, int* out);
__global__ void copy_cols_kernel(const float* __restrict__ src, int lds, int off, int ncols, int N,
                                 const int* __restrict__ n_dev, float* __restrict__ dst, int ldd, int doff);
__global__ void scatter_rgb4_kernel(const float* __restrict__ src, int N, const int* __restrict__ n_dev,
                                    const int* __restrict__ slot, float* __restrict__ dst);

// Y[n, :Nout] = act( (X[n,:K] (* Xmul[n,:K])) @ B[:K, :Nout] + bias )
//   B row stride ldb.  dact (optional, ld = ldy) receives d act / d pre-activation.
template <int BM, int BN, int BK>
__global__ void __launch_bounds__(256) dense_kernel(const float* __restrict__ X, int ldx,
                                                    const float* __restrict__ Xmul, int ldm,
                                                    const float* __restrict__ B, int ldb,
                                                    const float* __restrict__ bias, float* __restrict__ Y, int ldy,
                                                    float* __restrict__ dact, int N, const int* __restrict__ n_dev,
                                                    int K, int Nout, int act) {
  int n_rows = n_dev ? min(N, *n_dev) : N;
  int row0 = blockIdx.x * BM, col0 = blockIdx.y * BN;
  if (row0 >= n_rows) return;
  __shared__ float sX[BK][BM + 4];
  __shared__ float sB[BK][BN + 4];
  int tid = threadIdx.x;
  int tx = tid & 15, ty = tid >> 4;   // 16 x 16 threads, each 4 x 4 outputs (BM = BN = 64)
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += BK) {
    for (int i = tid; i < BM * BK; i += 256) {
      int r = i / BK, k = i - r * BK;
      int gr = row0 + r, gk = k0 + k;
      float v = 0.f;
      if (gr < n_rows && gk < K) {
        v = X[(size_t)gr * ldx + gk];
        if (Xmul) v *= Xmul[(size_t)gr * ldm + gk];
      }
      sX[k][r] = v;
    }
    for (int i = tid; i < BK * BN; i += 256) {
      int k = i / BN, c = i - k * BN;
      int gk = k0 + k, gc = col0 + c;
      sB[k][c] = (gk < K && gc < Nout) ? B[(size_t)gk * ldb + gc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sX[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sB[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int gr = row0 + ty * 4 + i;
    if (gr >= n_rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gc = col0 + tx * 4 + j;
      if (gc >= Nout) continue;
      float v = acc[i][j] + (bias ? bias[gc] : 0.f);
      float d = 1.f;
      if (act == ACT_SOFTPLUS) {
        d = softplus100_grad(v);
        v = softplus100(v);
      } else if (act == ACT_RELU) {
        d = v > 0.f ? 1.f : 0.f;
        v = fmaxf(v, 0.f);
      } else if (act == ACT_SIGMOID) {
        v = 1.f / (1.f + expf(-v));
      }
      Y[(size_t)gr * ldy + gc] = v;
      if (dact) dact[(size_t)gr * ldy + gc] = d;
    }
  }
}

static int dense(const float* X, int ldx, const float* Xmul, int ldm, const float* B, int ldb, const float* bias,
                 float* Y, int ldy, float* dact, int N, const int* n_dev, int K, int Nout, int act,
                 cudaStream_t st) {
  dim3 grid(div_up(N, 64), div_up(Nout, 64));
  dense_kernel<64, 64, 16><<<grid, 256, 0, st>>>(X, ldx, Xmul, ldm, B, ldb, bias, Y, ldy, dact, N, n_dev, K, Nout,
                                                 act);
  MP_LAUNCH_CHECK();
  return 0;
}

// embedders.py:8-34: e = [x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)]
__device__ __forceinline__ void embed_point(const float* x, int d, int L, float* e, int ld_unused) {
  for (int a = 0; a < d; ++a) e[a] = x[a];
  for (int f = 0; f < L; ++f) {
    float fr = (float)(1 << f);
    for (int a = 0; a < d; ++a) {
      float t = __fmul_rn(x[a], fr);
      e[d + (2 * f) * d + a] = sinf(t);
      e[d + (2 * f + 1) * d + a] = cosf(t);
    }
  }
}

// writes the embedding of each point to E1[n, off1 + :] (ld1) and optionally E2[n, off2 + :] (ld2)
__global__ void embed_kernel(const float* __restrict__ x, int d, int L, int N, const int* __restrict__ n_dev,
                             float* __restrict__ E1, int ld1, int off1, float* __restrict__ E2, int ld2, int off2) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (i >= n) return;
  float xv[4], e[96];
  for (int a = 0; a < d; ++a) xv[a] = x[(size_t)i * d + a];
  embed_point(xv, d, L, e, 0);
  int E = d * (1 + 2 * L);
  for (int k = 0; k < E; ++k) {
    E1[(size_t)i * ld1 + off1 + k] = e[k];
    if (E2) E2[(size_t)i * ld2 + off2 + k] = e[k];
  }
}

// d e / d x applied to the embedding gradient: gx = ge[0:d] + sum_f 2^f (cos(2^f x) ge_sin - sin(2^f x) ge_cos)
// ge = G0[n, :E] + Gs[n, offs + :E]
__global__ void embed_backward_kernel(const float* __restrict__ x, int d, int L, int N,
                                      const int* __restrict__ n_dev, const float* __restrict__ G0, int ld0,
                                      const float* __restrict__ Gs, int lds, int offs, float* __restrict__ gx) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (i >= n) return;
  for (int a = 0; a < d; ++a) {
    float xa = x[(size_t)i * d + a];
    float g = G0[(size_t)i * ld0 + a] + Gs[(size_t)i * lds + offs + a];
    for (int f = 0; f < L; ++f) {
      float fr = (float)(1 << f);
      float t = __fmul_rn(xa, fr);
      int ks = d + (2 * f) * d + a, kc = d + (2 * f + 1) * d + a;
      float gs = G0[(size_t)i * ld0 + ks] + Gs[(size_t)i * lds + offs + ks];
      float gc = G0[(size_t)i * ld0 + kc] + Gs[(size_t)i * lds + offs + kc];
      g += fr * (cosf(t) * gs - sinf(t) * gc);
    }
    gx[(size_t)i * d + a] = g;
  }
}

// Y[n, c] = v[c]  (broadcast a row vector; used to seed the backward pass with W8[0,:])
__global__ void broadcast_row_kernel(const float* __restrict__ v, int stride_v, int C, int N,
                                     const int* __restrict__ n_dev, float* __restrict__ Y, int ldy) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (idx >= n * C) return;
  int r = idx / C, c = idx - r * C;
  Y[(size_t)r * ldy + c] = v[(size_t)c * stride_v];
}

// scatter sdf (column 0 of the last layer) to its slot
__global__ void scatter_sdf_kernel(const float* __restrict__ h7, const float* __restrict__ w8col0, float b8_0,
                                   const float* __restrict__ b8, int N, const int* __restrict__ n_dev,
                                   const int* __restrict__ slot, float* __restrict__ sdf_out) {
  // one warp per point: sdf = h7 . W8[0,:] + b8[0]
  int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int n = n_dev ? min(N, *n_dev) : N;
  if (w >= n) return;
  float s = 0.f;
  for (int k = lane; k < kHidden; k += 32) s = fmaf(h7[(size_t)w * kHidden + k], w8col0[(size_t)k * (kHidden + 1)], s);
  s = warp_sum(s);
  if (lane == 0) sdf_out[slot ? slot[w] : w] = s + b8[0];
}

// normals: n = normalize(normalize(g @ Jinv), eps=1e-6)   (multiply.py:661, :606)
// colour input row = [x_c(3), n(3), feat(256)]
__global__ void normal_colour_input_kernel(const float* __restrict__ xc, const float* __restrict__ grad,
                                           const float* __restrict__ Jinv, const float* __restrict__ feat, int N,
                                           const int* __restrict__ n_dev, float* __restrict__ cin, int ldc,
                                           float* __restrict__ normal_tmp) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (i >= n) return;
  const float* J = Jinv + 12 * (size_t)i;
  float g0 = grad[3 * i], g1 = grad[3 * i + 1], g2 = grad[3 * i + 2];
  // einsum('bi,bij->bj', gradients, grads_inv)
  float v0 = g0 * J[0] + g1 * J[3] + g2 * J[6];
  float v1 = g0 * J[1] + g1 * J[4] + g2 * J[7];
  float v2 = g0 * J[2] + g1 * J[5] + g2 * J[8];
  float nr = fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-12f);
  v0 /= nr; v1 /= nr; v2 /= nr;
  float n2 = fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-6f);
  v0 /= n2; v1 /= n2; v2 /= n2;
  float* c = cin + (size_t)i * ldc;
  c[0] = xc[3 * i]; c[1] = xc[3 * i + 1]; c[2] = xc[3 * i + 2];
  c[3] = v0; c[4] = v1; c[5] = v2;
  normal_tmp[3 * i] = v0; normal_tmp[3 * i + 1] = v1; normal_tmp[3 * i + 2] = v2;
  (void)feat;
}

__global__ void scatter3_kernel(const float* __restrict__ src, int N, const int* __restrict__ n_dev,
                                const int* __restrict__ slot, float* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (i >= n) return;
  int s = slot ? slot[i] : i;
  dst[3 * (size_t)s] = src[3 * i];
  dst[3 * (size_t)s + 1] = src[3 * i + 1];
  dst[3 * (size_t)s + 2] = src[3 * i + 2];
}

__global__ void view_embed_kernel(const float* __restrict__ dirs, int L, int N, float* __restrict__ cin, int ldc) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float xv[3] = {dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]};
  float e[32];
  embed_point(xv, 3, L, e, 0);
  for (int k = 0; k < 3 * (1 + 2 * L); ++k) cin[(size_t)i * ldc + k] = e[k];
}

// ------------------------------------------------------------------------------------------
// chains
// ------------------------------------------------------------------------------------------
// points per pass of the chains: the backward keeps the 8 dact buffers, so it runs half as many
constexpr int kSimtChunk = 65536, kSimtChunkBwd = 32768;

struct SimtBufs {
  int* nrem;
  float *H0, *H1, *E, *dact[8], *cin, *feat, *grad, *ntmp, *ge0;
};

static void simt_carve(Arena& a, int N, bool need_grad, SimtBufs& b) {
  b.nrem = a.take<int>(1);
  b.H0 = a.take<float>((size_t)N * 256);
  b.H1 = a.take<float>((size_t)N * 256);
  b.E = a.take<float>((size_t)N * 96);
  for (int l = 0; l < 8; ++l) b.dact[l] = need_grad ? a.take<float>((size_t)N * 256) : nullptr;
  b.cin = a.take<float>((size_t)N * 296);
  b.feat = a.take<float>((size_t)N * 256);
  b.grad = a.take<float>((size_t)N * 4);
  b.ntmp = a.take<float>((size_t)N * 4);
  b.ge0 = a.take<float>((size_t)N * 96);
}

// the larger of the two chunk layouts a list of N points can carve
size_t simt_workspace_bytes(int N) {
  N = max(N, 0);
  Arena fwd, bwd;
  SimtBufs b;
  simt_carve(fwd, min(N, kSimtChunk), false, b);
  simt_carve(bwd, min(N, kSimtChunkBwd), true, b);
  return max(fwd.off, bwd.off);
}

// forward through layers 0..7 ; leaves h7 in *h7_out (one of H0/H1) ; h3 buffer holds [h3 | E]
static int simt_trunk(const Field& f, const float* x, int N, const int* n_dev, SimtBufs& b, bool need_grad,
                      float** h7_out, cudaStream_t st) {
  const int E = f.emb_dim;
  embed_kernel<<<div_up(N, 128), 128, 0, st>>>(x, f.d_in, f.multires, N, n_dev, b.E, 96, 0, nullptr, 0, 0);
  MP_LAUNCH_CHECK();
  float* cur = b.H0;
  float* nxt = b.H1;
  MP_TRY(dense(b.E, 96, nullptr, 0, f.imp_Wt[0], kHidden, f.imp_b0_eff, cur, 256, need_grad ? b.dact[0] : nullptr, N,
               n_dev, E, kHidden, ACT_SOFTPLUS, st));
  for (int l = 1; l < 8; ++l) {
    int outd = f.imp_out[l];
    MP_TRY(dense(cur, 256, nullptr, 0, f.imp_Wt[l], outd, f.imp_b[l], nxt, 256, need_grad ? b.dact[l] : nullptr, N,
                 n_dev, kHidden, outd, ACT_SOFTPLUS, st));
    if (l == f.skip_layer - 1) {
      // layer-4 input = [h3, embed] (the 1/sqrt(2) lives in W4)   networks.py:166-167
      embed_kernel<<<div_up(N, 128), 128, 0, st>>>(x, f.d_in, f.multires, N, n_dev, nxt, 256, kHidden - E, nullptr,
                                                   0, 0);
      MP_LAUNCH_CHECK();
    }
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  *h7_out = cur;
  return 0;
}

__global__ void sub_count_kernel(const int* c, int s, int* out) { *out = max(0, *c - s); }

// RenderingNet layers on the colour input cin [n, ldc] (networks.py:290-312): ReLU layers ping-ponging between c0 and
// c1, the sigmoid head into a [n,4]-strided buffer, then rgb repacked 3-strided to its slot (dense when slot is null)
static int simt_colour(const Field& f, const float* cin, int ldc, int n, const int* n_dev, float* c0, float* c1,
                       const int* slot, float* rgb_out, cudaStream_t st) {
  MP_TRY(dense(cin, ldc, nullptr, 0, f.ren_Wt[0], f.ren_out[0], f.ren_b0_eff, c0, 256, nullptr, n, n_dev, ldc,
               f.ren_out[0], ACT_RELU, st));
  for (int l = 1; l < f.n_ren - 1; ++l) {
    MP_TRY(dense(c0, 256, nullptr, 0, f.ren_Wt[l], f.ren_out[l], f.ren_b[l], c1, 256, nullptr, n, n_dev, f.ren_in[l],
                 f.ren_out[l], ACT_RELU, st));
    float* t = c0;
    c0 = c1;
    c1 = t;
  }
  const int L = f.n_ren - 1;
  MP_TRY(dense(c0, 256, nullptr, 0, f.ren_Wt[L], f.ren_out[L], f.ren_b[L], c1, 4, nullptr, n, n_dev, f.ren_in[L], 3,
               ACT_SIGMOID, st));
  scatter_rgb4_kernel<<<div_up(n, 256), 256, 0, st>>>(c1, n, n_dev, slot, rgb_out);
  MP_LAUNCH_CHECK();
  return 0;
}

// One MlpCall, the chain that mlp_prog picks, in chunks of the list.  sdf, rgb and normals are scattered to their slots.
int simt_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st) {
  const MlpProg prog = mlp_prog(c);
  const bool bwd = prog == MlpProg::kFull;
  const int CH = bwd ? kSimtChunkBwd : kSimtChunk;
  const int E = f.emb_dim;
  for (int s = 0; s < c.cap; s += CH) {
    int n = min(CH, c.cap - s);
    Arena a(ws, ws_bytes);
    SimtBufs b;
    simt_carve(a, n, bwd, b);
    MP_TRY(a.fits("simt_run"));
    int* nrem = b.nrem;
    if (c.count) {
      // remaining count for this chunk = count - s (clamped by the kernels through min(N, *n_dev))
      sub_count_kernel<<<1, 1, 0, st>>>(c.count, s, nrem);
      MP_LAUNCH_CHECK();
    } else {
      nrem = nullptr;
    }
    const float* x = c.x + (size_t)f.d_in * s;
    const int* slot = c.slot ? c.slot + s : nullptr;
    auto out = [&](float* p, int width) { return p && !c.slot ? p + (size_t)width * s : p; };   // slotted or dense
    float* h7;
    MP_TRY(simt_trunk(f, x, n, nrem, b, bwd, &h7, st));
    if (c.sdf) {
      scatter_sdf_kernel<<<div_up(n * 32, 256), 256, 0, st>>>(h7, f.imp_Wt[8], 0.f, f.imp_b[8], n, nrem, slot,
                                                              out(c.sdf, 1));
      MP_LAUNCH_CHECK();
    }
    if (prog == MlpProg::kSdf) continue;
    if (prog == MlpProg::kBg) {     // multiply.py:524-531
      const int X = f.ren_extra, ldc = X + 256;
      view_embed_kernel<<<div_up(n, 128), 128, 0, st>>>(c.dirs + 3 * (size_t)s, f.multires_view, n, b.cin, ldc);
      MP_LAUNCH_CHECK();
      // features straight into the colour input block
      MP_TRY(dense(h7, 256, nullptr, 0, f.imp_Wt[8] + 1, kHidden + 1, f.imp_b[8] + 1, b.cin + X, ldc, nullptr, n, nrem,
                   kHidden, kHidden, ACT_NONE, st));
      MP_TRY(simt_colour(f, b.cin, ldc, n, nrem, (h7 == b.H0) ? b.H1 : b.H0, h7, slot, out(c.rgb, 3), st));
      continue;
    }
    // features = h7 @ W8[1:,:]^T + b8[1:]
    float* featp = c.feat ? c.feat + (size_t)s * 256 : b.feat;
    MP_TRY(dense(h7, 256, nullptr, 0, f.imp_Wt[8] + 1, kHidden + 1, f.imp_b[8] + 1, featp, 256, nullptr, n, nrem,
                 kHidden, kHidden, ACT_NONE, st));
    if (prog == MlpProg::kForward) continue;
    // ---- backward: d sdf / d x_c ---------------------------------------------------------
    float* g = (h7 == b.H0) ? b.H1 : b.H0;   // free buffer
    float* g2 = h7;                          // h7 no longer needed after features
    broadcast_row_kernel<<<div_up(n * 256, 256), 256, 0, st>>>(f.imp_Wt[8], kHidden + 1, kHidden, n, nrem, g, 256);
    MP_LAUNCH_CHECK();
    // g holds d/dh7.  for l = 7..1: d/dh_{l-1} = (g * dact_l) @ W_l      (W_l natural [out][in])
    for (int l = 7; l >= 1; --l) {
      int outd = f.imp_out[l];      // contraction length
      MP_TRY(dense(g, 256, b.dact[l], 256, f.imp_W[l], f.imp_in[l], nullptr, g2, 256, nullptr, n, nrem, outd,
                   f.imp_in[l], ACT_NONE, st));
      if (l == f.skip_layer) {
        // columns [256-E, 256) of g2 are the skip gradient d/d embed: park them in ge0[:, 0:E] (ld 96)
        // (g2's first 256-E columns are d/dh3)
        copy_cols_kernel<<<div_up(n * E, 256), 256, 0, st>>>(g2, 256, kHidden - E, E, n, nrem, b.ge0, 96, 0);
        MP_LAUNCH_CHECK();
      }
      float* t = g;
      g = g2;
      g2 = t;
    }
    // layer 0: d/d embed = (g * dact_0) @ W0[:, :E]
    MP_TRY(dense(g, 256, b.dact[0], 256, f.imp_W[0], f.imp_in[0], nullptr, g2, 256, nullptr, n, nrem, kHidden, E,
                 ACT_NONE, st));
    float* gradp = c.grad ? c.grad + 3 * (size_t)s : b.grad;
    embed_backward_kernel<<<div_up(n, 128), 128, 0, st>>>(x, f.d_in, f.multires, n, nrem, g2, 256, b.ge0, 96, 0,
                                                          gradp);
    MP_LAUNCH_CHECK();
    if (!c.jinv) continue;
    // ---- normals + colour ----------------------------------------------------------------
    const int ldc = 6 + 256;
    normal_colour_input_kernel<<<div_up(n, 128), 128, 0, st>>>(x, gradp, c.jinv + 12 * (size_t)s, featp, n, nrem,
                                                               b.cin, ldc, b.ntmp);
    MP_LAUNCH_CHECK();
    copy_cols_kernel<<<div_up(n * 256, 256), 256, 0, st>>>(featp, 256, 0, 256, n, nrem, b.cin, ldc, 6);
    MP_LAUNCH_CHECK();
    MP_TRY(simt_colour(f, b.cin, ldc, n, nrem, b.H0, b.H1, slot, out(c.rgb, 3), st));
    scatter3_kernel<<<div_up(n, 256), 256, 0, st>>>(b.ntmp, n, nrem, slot, out(c.nrm, 3));
    MP_LAUNCH_CHECK();
  }
  return 0;
}

__global__ void copy_cols_kernel(const float* __restrict__ src, int lds, int off, int ncols, int N,
                                 const int* __restrict__ n_dev, float* __restrict__ dst, int ldd, int doff) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (idx >= n * ncols) return;
  int r = idx / ncols, c = idx - r * ncols;
  dst[(size_t)r * ldd + doff + c] = src[(size_t)r * lds + off + c];
}

__global__ void scatter_rgb4_kernel(const float* __restrict__ src, int N, const int* __restrict__ n_dev,
                                    const int* __restrict__ slot, float* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int n = n_dev ? min(N, *n_dev) : N;
  if (i >= n) return;
  int s = slot ? slot[i] : i;
  dst[3 * (size_t)s] = src[4 * i];
  dst[3 * (size_t)s + 1] = src[4 * i + 1];
  dst[3 * (size_t)s + 2] = src[4 * i + 2];
}

__global__ void colour_input_kernel(const float* __restrict__ pts, const float* __restrict__ nrm,
                                    const float* __restrict__ feat, int N, float* __restrict__ cin, int ldc) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * ldc) return;
  int r = idx / ldc, c = idx - r * ldc;
  float v;
  if (c < 3) v = pts[3 * r + c];
  else if (c < 6) v = nrm[3 * r + c - 3];
  else v = feat[(size_t)r * 256 + c - 6];
  cin[idx] = v;
}

// RenderingNet.forward 'pose_no_view' on explicit inputs (networks.py:263-312)
int simt_render(const Field& f, const float* pts, const float* nrm, const float* feat, int N, float* rgb, void* ws,
                size_t ws_bytes, cudaStream_t st) {
  MP_REQUIRE(f.ren_mode == 0, "mp_render_forward: only the pose_no_view colour net takes (points, normals, feat)");
  for (int s = 0; s < N; s += kSimtChunk) {
    int n = min(kSimtChunk, N - s);
    Arena a(ws, ws_bytes);
    SimtBufs b;
    simt_carve(a, n, false, b);
    MP_TRY(a.fits("simt_render"));
    const int ldc = 6 + 256;
    colour_input_kernel<<<div_up(n * ldc, 256), 256, 0, st>>>(pts + 3 * (size_t)s, nrm + 3 * (size_t)s,
                                                             feat + 256 * (size_t)s, n, b.cin, ldc);
    MP_LAUNCH_CHECK();
    MP_TRY(simt_colour(f, b.cin, ldc, n, nullptr, b.H0, b.H1, nullptr, rgb + 3 * (size_t)s, st));
  }
  return 0;
}

}  // namespace mp
