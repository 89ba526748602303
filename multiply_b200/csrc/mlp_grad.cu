// First-order backward of ImplicitNet and of RenderingNet 'pose_no_view' on the Hopper tensor cores (DESIGN.md §3.9).
//   reference: lib/model/networks.py:126-208 (ImplicitNet.forward), :263-312 (RenderingNet.forward), embedders.py:8-34;
//              torch autograd of F.linear, F.softplus(beta=100, threshold=20), relu and sigmoid
//
// Layer-major.  Per chunk of kChunk points the forward pre-activations Z_l are recomputed and stored (the activation is
// applied again when the next layer stages them), then the layers are walked backwards.  Layer l with activation s:
//     G_l       = dA_l * s'(Z_l)                 (formed while G is staged, never stored)
//     dA_{l-1}  = G_l W_l                        input gradient, [n x in]
//     dW_l     += G_l^T A_{l-1}                  weight gradient, K = points
//     db_l     += sum over points of G_l
// Every product runs on one wgmma GEMM kernel, C[M x N] = A[M x K] B[N x K]^T: its operand loaders read fp32 from
// global memory in either orientation, apply the activation or its derivative and split each value into fp16 hi + lo
// while staging the tile into shared memory (K-major, 128-byte swizzle), and each K-step issues A_hi B_hi + A_lo B_hi +
// A_hi B_lo with fp32 accumulation, as the forward does (§3.1, Precision).
//
// The tensor core accumulates with round-toward-zero.  A weight-gradient CTA owns kSplit points; its accumulator is
// restarted every kGroup points and added to a register sum with round-to-nearest fp32 adds.  The CTAs' partials are
// added in fp64 into per-layer accumulators in split order, chunk after chunk, so the result depends on N alone: not on
// the run, the grid or what the workspace held.
#include "common.cuh"
#include <atomic>

namespace mp {
namespace {

constexpr int kChunk = 32768;               // points per pass
constexpr int kSplit = 1024;                // points of one weight-gradient CTA (one partial)
constexpr int kGroup = 256;                 // points per wgmma accumulator before its round-to-nearest flush
constexpr int kBiasRows = 128;              // points of one bias partial
constexpr int kLd = 256;                    // row stride of the Z and dA buffers
constexpr int kEmbLd = 96;                  // row stride of the embedding (d_in * (1 + 2 multires) <= 96)
constexpr int kCinLd = 272;                 // row stride of the colour input and its gradient (270 columns)
constexpr int kMaxOut = 264;                // accumulator rows per layer (257 outputs at most)
constexpr int kMaxIn = 272;                 // accumulator columns per layer (270 inputs at most)
constexpr int kImpLayers = 9, kRenLayers = 5, kPoseDim = 8, kBodyPose = 69;

enum { ACT_NONE = 0, ACT_SOFTPLUS = 1, ACT_RELU = 2, ACT_SIGMOID = 3 };

__device__ __forceinline__ float sigmoidf(float z) { return 1.f / (1.f + expf(-z)); }
__device__ __forceinline__ float act_f(int a, float z) {
  if (a == ACT_SOFTPLUS) return softplus100(z);
  if (a == ACT_RELU) return z > 0.f ? z : 0.f;
  if (a == ACT_SIGMOID) return sigmoidf(z);
  return z;
}
// torch's backward formulas: softplus threshold_backward, relu (0 at 0), sigmoid y (1 - y) of the output y
__device__ __forceinline__ float act_d(int a, float z) {
  if (a == ACT_SOFTPLUS) return softplus100_grad(z);
  if (a == ACT_RELU) return z > 0.f ? 1.f : 0.f;
  if (a == ACT_SIGMOID) {
    const float y = sigmoidf(z);
    return (1.f - y) * y;
  }
  return 1.f;
}

// ---------------------------------------------------------------------------------------------
// operands: element (r, k) of a GEMM operand, zero outside it
// ---------------------------------------------------------------------------------------------
struct Seg {
  const float* p;      // null: zeros
  int ld, w, act;
};
// a layer's input rows: [act(seg0) | act(seg1)] of point r
struct ActOp {
  Seg s0, s1;
  int rows;
  __device__ __forceinline__ float operator()(int r, int k) const {
    if (r >= rows) return 0.f;
    if (k < s0.w) return act_f(s0.act, s0.p[(size_t)r * s0.ld + k]);
    k -= s0.w;
    if (k < s1.w) return act_f(s1.act, s1.p[(size_t)r * s1.ld + k]);
    return 0.f;
  }
};
// G of point r, output column k: the upstream gradient [d0 | d1] times the activation derivative at Z
struct GradOp {
  Seg d0, d1;
  const float* z;      // [rows][kLd] pre-activations (unused for ACT_NONE)
  int act, rows;
  __device__ __forceinline__ float operator()(int r, int k) const {
    if (r >= rows) return 0.f;
    float g;
    if (k < d0.w) {
      g = d0.p ? d0.p[(size_t)r * d0.ld + k] : 0.f;
    } else if (k - d0.w < d1.w) {
      g = d1.p ? d1.p[(size_t)r * d1.ld + k - d0.w] : 0.f;
    } else {
      return 0.f;
    }
    return act == ACT_NONE ? g : g * act_d(act, z[(size_t)r * kLd + k]);
  }
};
// p[r * sr + k * sk] inside [rows x cols]
struct MatOp {
  const float* p;
  int sr, sk, rows, cols;
  __device__ __forceinline__ float operator()(int r, int k) const {
    return (r < rows && k < cols) ? p[(size_t)r * sr + (size_t)k * sk] : 0.f;
  }
};
template <class Op>
struct Tr {
  Op op;
  __device__ __forceinline__ float operator()(int r, int k) const { return op(k, r); }
};

// ---------------------------------------------------------------------------------------------
// the GEMM kernel: one warpgroup, a 64 x 128 tile of C, K in steps of 64 through two shared-memory stages
// ---------------------------------------------------------------------------------------------
constexpr int kBM = 64, kBN = 128, kBK = 64;
constexpr int kImgA = kBM * 128, kImgB = kBN * 128;      // bytes of one fp16 image (64 K-columns)
constexpr int kStage = 2 * kImgA + 2 * kImgB;            // A hi, A lo, B hi, B lo
constexpr int kGemmSmem = 2 * kStage + 1024;              // + alignment of the swizzled images

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sts128(uint32_t a, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(a, b);
  float2 f = __half22float2(h);
  __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *(uint32_t*)&h;
  lo = *(uint32_t*)&l;
}
// K-major, 128-byte swizzle descriptor: start >> 4, LBO 1 (unused), SBO 1024 B between 8-row groups, SWIZZLE_128B
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

#define MP_R8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                 "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x 128] += A[64 x 16] . B[128 x 16]^T, both K-major in shared memory
__device__ __forceinline__ void mma_n128(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, 1, 1, 1, 0, 0;\n"
      : MP_R8(0), MP_R8(8), MP_R8(16), MP_R8(24), MP_R8(32), MP_R8(40), MP_R8(48), MP_R8(56)
      : "l"(a), "l"(b));
}
#undef MP_R8

// Stages rows [r0, r0 + ROWS) x K-columns [k0, k0 + 64) of op as fp16 hi / lo images.  Each thread converts one
// 8-column chunk of a row at a time; ROWFAST puts consecutive threads on consecutive rows (an operand whose memory is
// contiguous along rows), else on consecutive chunks of a row (contiguous along K).
template <int ROWS, bool ROWFAST, class Op>
__device__ __forceinline__ void stage(const Op& op, float sc, int r0, int k0, uint32_t hi, uint32_t lo) {
#pragma unroll 2
  for (int u = threadIdx.x; u < ROWS * 8; u += 128) {
    const int r = ROWFAST ? u % ROWS : u >> 3;
    const int ch = ROWFAST ? u / ROWS : u & 7;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = op(r0 + r, k0 + 8 * ch + e) * sc;
    uint4 h, l;
    split2(v[0], v[1], h.x, l.x);
    split2(v[2], v[3], h.y, l.y);
    split2(v[4], v[5], h.z, l.z);
    split2(v[6], v[7], h.w, l.w);
    const uint32_t off = (uint32_t)(r * 128 + ((ch ^ (r & 7)) << 4));
    sts128(hi + off, h);
    sts128(lo + off, l);
  }
}

// The power-of-two exponent that puts an operand's largest magnitude `amax` (as float bits; null: no scaling) in
// [2^13, 2^14): its fp16 hi and lo parts then stay normal wherever they matter, whatever the scale of the operand, and
// scaling by a power of two is exact.  Operands are scaled as they are staged and the product is unscaled in the
// epilogue, so a power-of-two factor on the upstream gradient gives exactly that factor on every result.
__device__ __forceinline__ int scale_exp(const unsigned* amax) {
  if (!amax) return 0;
  const float m = __uint_as_float(*amax);
  if (!(m > 0.f) || !isfinite(m)) return 0;
  int e;
  frexpf(m, &e);       // m = f 2^e, f in [0.5, 1)
  return max(-126, min(127, 14 - e));
}

// C tile (blockIdx.y, blockIdx.x) over K-range [z kper, (z + 1) kper) of blockIdx.z; the accumulator is flushed into
// the round-to-nearest sum every `group` K (a multiple of 64).  Accumulator register i of thread t (warp w, lane l):
// row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l % 4) + (i & 1).
template <bool AROW, bool BROW, class OA, class OB, class Epi>
__global__ void __launch_bounds__(128) grad_gemm_kernel(OA oa, OB ob, Epi ep, const unsigned* amax_a,
                                                        const unsigned* amax_b, int K, int kper, int group) {
  extern __shared__ char smem_raw[];
  const int ea = scale_exp(amax_a), eb = scale_exp(amax_b);
  const float sa = ldexpf(1.f, ea), sb = ldexpf(1.f, eb), ua = ldexpf(1.f, -ea), ub = ldexpf(1.f, -eb);
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const int kb = blockIdx.z * kper, ke = min(K, kb + kper);
  float acc[64], sum[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = sum[i] = 0.f;
  auto a_hi = [&](int s) { return base + s * kStage; };
  auto b_hi = [&](int s) { return base + s * kStage + 2 * kImgA; };
  if (kb < ke) {
    stage<kBM, AROW>(oa, sa, m0, kb, a_hi(0), a_hi(0) + kImgA);
    stage<kBN, BROW>(ob, sb, n0, kb, b_hi(0), b_hi(0) + kImgB);
  }
  int s = 0;
#pragma unroll 1
  for (int k0 = kb; k0 < ke; k0 += kBK) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t ah = make_desc(a_hi(s) + ks * 32), al = make_desc(a_hi(s) + kImgA + ks * 32);
      const uint64_t bh = make_desc(b_hi(s) + ks * 32), bl = make_desc(b_hi(s) + kImgB + ks * 32);
      mma_n128(acc, ah, bh);
      mma_n128(acc, al, bh);
      mma_n128(acc, ah, bl);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    const int kn = k0 + kBK;
    if (kn < ke) {      // the other stage's MMAs were waited for in the previous step, before the barrier above
      stage<kBM, AROW>(oa, sa, m0, kn, a_hi(s ^ 1), a_hi(s ^ 1) + kImgA);
      stage<kBN, BROW>(ob, sb, n0, kn, b_hi(s ^ 1), b_hi(s ^ 1) + kImgB);
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(acc[i])::"memory");
    if (kn >= ke || (kn - kb) % group == 0) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        sum[i] = __fadd_rn(sum[i], acc[i]);
        acc[i] = 0.f;
      }
    }
    s ^= 1;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int r = m0 + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1);
    const int c = n0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    ep(r, c, blockIdx.z, (sum[i] * ua) * ub);
  }
}

// out[r][c] = v (+ bias[c]) inside [rows x cols]
struct EpiStore {
  float* out;
  int ld;
  const float* bias;
  int rows, cols;
  __device__ __forceinline__ void operator()(int r, int c, int, float v) const {
    if (r < rows && c < cols) out[(size_t)r * ld + c] = bias ? v + bias[c] : v;
  }
};
// part[z][r][c] = v : one weight-gradient partial per K-split
struct EpiPartial {
  float* part;
  int rows, cols;
  __device__ __forceinline__ void operator()(int r, int c, int z, float v) const {
    if (r < rows && c < cols) part[((size_t)z * rows + r) * cols + c] = v;
  }
};

// amax_a / amax_b: device maxima of |operand| that scale it (scale_exp), or null
template <bool AROW, bool BROW, class OA, class OB, class Epi>
int gemm(const OA& a, const OB& b, const Epi& ep, const unsigned* amax_a, const unsigned* amax_b, int M, int N, int K,
         int kper, int group, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  auto kern = grad_gemm_kernel<AROW, BROW, OA, OB, Epi>;
  // the shared-memory opt-in, once per instantiation and device
  static std::atomic<unsigned long long> opted{0};
  int dev = 0;
  MP_CHECK_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted.load() & bit)) {
    MP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmem));
    opted.fetch_or(bit);
  }
  dim3 grid(div_up(N, kBN), div_up(M, kBM), div_up(K, kper));
  kern<<<grid, 128, kGemmSmem, st>>>(a, b, ep, amax_a, amax_b, K, kper, group);
  MP_LAUNCH_CHECK();
  return 0;
}
// Z = A W^T + bias (recompute), dA = G W (input gradient): K is a layer width, one accumulator
template <bool BROW, class OA, class OB>
int layer_gemm(const OA& a, const OB& b, const unsigned* amax_a, const unsigned* amax_b, float* out, int ld,
               const float* bias, int M, int N, int K, cudaStream_t st) {
  const int kp = div_up(K, kBK) * kBK;
  return gemm<false, BROW>(a, b, EpiStore{out, ld, bias, M, N}, amax_a, amax_b, M, N, K, kp, kp, st);
}

// *amax = max |op(r, c)| over [rows x cols] as float bits (the caller zeroes it); exact, so independent of the order
template <class Op>
__global__ void __launch_bounds__(256) absmax_kernel(Op op, int rows, int cols, unsigned* __restrict__ amax) {
  float m = 0.f;
  const long long n = (long long)rows * cols;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int r = (int)(i / cols), c = (int)(i - (long long)r * cols);
    m = fmaxf(m, fabsf(op(r, c)));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(amax, __float_as_uint(m));
}
template <class Op>
int absmax(const Op& op, int rows, int cols, unsigned* amax, cudaStream_t st) {
  MP_CHECK_CUDA(cudaMemsetAsync(amax, 0, sizeof(unsigned), st));
  const long long n = (long long)rows * cols;
  if (n <= 0) return 0;
  const int blocks = n >= 1024ll * 256 ? 1024 : (int)((n + 255) / 256);
  absmax_kernel<<<blocks, 256, 0, st>>>(op, rows, cols, amax);
  MP_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// reductions over points and the parameter-sized pieces
// ---------------------------------------------------------------------------------------------
// acc[r][c] += sum over s (ascending) of part[s][r][c], in fp64
__global__ void reduce_partials_kernel(const float* __restrict__ part, int ns, int rows, int cols,
                                       double* __restrict__ acc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  double s = acc[(size_t)r * kMaxIn + c];
  for (int z = 0; z < ns; ++z) s += (double)part[(size_t)z * rows * cols + i];
  acc[(size_t)r * kMaxIn + c] = s;
}
// partb[split][c] = sum over the split's kBiasRows points of G(p, c), in fp64: a block is 32 columns x 8 point lanes,
// each lane sums every 8th point, the lanes are added in lane order
__global__ void __launch_bounds__(256) colsum_kernel(GradOp g, int cols, int n, double* __restrict__ partb) {
  __shared__ double red[8][32];
  const int c = blockIdx.x * 32 + threadIdx.x, p0 = blockIdx.y * kBiasRows, p1 = min(n, p0 + kBiasRows);
  double s = 0.0;
  if (c < cols)
    for (int p = p0 + threadIdx.y; p < p1; p += 8) s += (double)g(p, c);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    for (int j = 1; j < 8; ++j) s += red[j][threadIdx.x];
    partb[(size_t)blockIdx.y * kMaxIn + c] = s;
  }
}
// acc[c] += the sum of partb[0 .. ns)[c] by a fixed tree: one block of 256 threads per column
__global__ void __launch_bounds__(256) reduce_bias_kernel(const double* __restrict__ partb, int ns,
                                                          double* __restrict__ acc) {
  __shared__ double red[256];
  const int c = blockIdx.x, t = threadIdx.x;
  double s = 0.0;
  for (int z = t; z < ns; z += 256) s += partb[(size_t)z * kMaxIn + c];
  red[t] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) acc[c] += red[0];
}
// dW[r][col_off + c] = acc[r][c] * scale
__global__ void finalize_w_kernel(const double* __restrict__ acc, int rows, int cols, double scale,
                                  float* __restrict__ dW, int ldw, int col_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  dW[(size_t)r * ldw + col_off + c] = (float)(acc[(size_t)r * kMaxIn + c] * scale);
}
__global__ void finalize_b_kernel(const double* __restrict__ acc, int n, float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) db[i] = (float)acc[i];
}
// ImplicitNet layer 0's cond columns: dW0[o][E + j] = db0[o] cond[j]; d_cond[j] = sum_o db0[o] W0[o][E + j]
__global__ void cond_grad_kernel(const double* __restrict__ db0, const float* __restrict__ cond, int cdim, int out0,
                                 const float* __restrict__ W0, int in0, int E, float* __restrict__ dW0,
                                 float* __restrict__ d_cond) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cdim) return;
  double s = 0.0;
  for (int o = 0; o < out0; ++o) {
    if (dW0) dW0[(size_t)o * in0 + E + j] = (float)(db0[o] * (double)cond[j]);
    s += db0[o] * (double)W0[(size_t)o * in0 + E + j];
  }
  if (d_cond) d_cond[j] = (float)s;
}
// lin_pose(body_pose) of RenderingNet (networks.py:277-281): pf[j] = b[j] + sum_k Wp[j][k] bp[k]
__global__ void pose_feat_kernel(const float* __restrict__ Wp, const float* __restrict__ bp_bias,
                                 const float* __restrict__ bp, float* __restrict__ pf) {
  const int j = threadIdx.x;
  if (j >= kPoseDim) return;
  float s = 0.f;
  for (int k = 0; k < kBodyPose; ++k) s = fmaf(Wp[j * kBodyPose + k], bp[k], s);
  pf[j] = s + bp_bias[j];
}
// d pf = W0[:, 6:14]^T db0 (the pose features are the same for every point), then the lin_pose chain
__global__ void pose_grad_kernel(const double* __restrict__ db0, const float* __restrict__ W0, int in0, int out0,
                                 const float* __restrict__ Wp, const float* __restrict__ bp, float* __restrict__ d_lpw,
                                 float* __restrict__ d_lpb, float* __restrict__ d_bp) {
  __shared__ double dpf[kPoseDim];
  const int t = threadIdx.x;
  if (t < kPoseDim) {
    double s = 0.0;
    for (int o = 0; o < out0; ++o) s += db0[o] * (double)W0[(size_t)o * in0 + 6 + t];
    dpf[t] = s;
    if (d_lpb) d_lpb[t] = (float)s;
  }
  __syncthreads();
  for (int i = t; i < kPoseDim * kBodyPose; i += blockDim.x)
    if (d_lpw) d_lpw[i] = (float)(dpf[i / kBodyPose] * (double)bp[i % kBodyPose]);
  for (int k = t; k < kBodyPose; k += blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < kPoseDim; ++j) s += dpf[j] * (double)Wp[j * kBodyPose + k];
    if (d_bp) d_bp[k] = (float)s;
  }
}

// embedders.py:8-34 as the forward engines evaluate it: [x, sin(2^f x), cos(2^f x) ...], 2^f x rounded once
__global__ void embed_kernel(const float* __restrict__ x, int d, int L, int n, float* __restrict__ emb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float* e = emb + (size_t)i * kEmbLd;
  for (int a = 0; a < d; ++a) {
    const float xa = x[(size_t)i * d + a];
    e[a] = xa;
    for (int f = 0; f < L; ++f) {
      const float t = __fmul_rn(xa, (float)(1 << f));
      e[d + 2 * f * d + a] = sinf(t);
      e[d + (2 * f + 1) * d + a] = cosf(t);
    }
  }
}
// d x = g[0:d] + sum_f 2^f (cos(2^f x) g_sin - sin(2^f x) g_cos), g = layer 0's part + the skip's part
__global__ void embed_backward_kernel(const float* __restrict__ x, int d, int L, int n, const float* __restrict__ g0,
                                      const float* __restrict__ g1, int off1, float* __restrict__ dx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* a0 = g0 + (size_t)i * kLd;
  const float* a1 = g1 + (size_t)i * kLd + off1;
  for (int a = 0; a < d; ++a) {
    const float xa = x[(size_t)i * d + a];
    float g = a0[a] + a1[a];
    for (int f = 0; f < L; ++f) {
      const float fr = (float)(1 << f);
      const float t = __fmul_rn(xa, fr);
      const int ks = d + 2 * f * d + a, kc = ks + d;
      g += fr * (cosf(t) * (a0[ks] + a1[ks]) - sinf(t) * (a0[kc] + a1[kc]));
    }
    dx[(size_t)i * d + a] = g;
  }
}
// colour input [points, normals, lin_pose(body_pose), feat] (networks.py:277-281)
__global__ void colour_input_kernel(const float* __restrict__ pts, const float* __restrict__ nrm,
                                    const float* __restrict__ pf, const float* __restrict__ feat, int n,
                                    float* __restrict__ cin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 270) return;
  const int r = i / 270, c = i - r * 270;
  float v;
  if (c < 3) v = pts[3 * (size_t)r + c];
  else if (c < 6) v = nrm[3 * (size_t)r + c - 3];
  else if (c < 14) v = pf[c - 6];
  else v = feat[(size_t)r * 256 + c - 14];
  cin[(size_t)r * kCinLd + c] = v;
}
// the colour input's gradient back to its sources (the pose features' part goes through db0 instead)
__global__ void colour_input_backward_kernel(const float* __restrict__ dcin, int n, float* __restrict__ dp,
                                             float* __restrict__ dn, float* __restrict__ df) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 270) return;
  const int r = i / 270, c = i - r * 270;
  const float v = dcin[(size_t)r * kCinLd + c];
  if (c < 3) { if (dp) dp[3 * (size_t)r + c] = v; }
  else if (c < 6) { if (dn) dn[3 * (size_t)r + c - 3] = v; }
  else if (c >= 14 && df) df[(size_t)r * 256 + c - 14] = v;
}

// ---------------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------------
struct GradWs {
  int n, ns;                  // points of a full chunk, weight-gradient splits of it
  float* Z[kImpLayers];       // [n][kLd] pre-activations
  float* in0;                 // implicit: embedding [n][kEmbLd]; colour: input [n][kCinLd]
  float* dA[3];               // [n][kLd] activation gradients; colour: dA[2] is d cin [n][kCinLd]
  float* part;                // [ns][kMaxOut * kMaxIn] weight-gradient partials of one layer
  double* partb;              // [n / kBiasRows][kMaxIn] bias partials
  double* accW;               // [layers][kMaxOut][kMaxIn]
  double* accB;               // [layers][kMaxIn]
  float* pf;                  // [8] colour: lin_pose(body_pose)
  unsigned* amax;             // max |operand| as float bits: [kAmaxW + l] weights, [kAmaxA + l] layer inputs, [kAmaxG + l] G
};
constexpr int kAmaxW = 0, kAmaxA = 16, kAmaxG = 32, kAmaxSlots = 48;

void grad_carve(Arena& a, int N, bool colour, GradWs& w) {
  w.n = min(max(N, 0), kChunk);
  w.ns = div_up(w.n, kSplit);
  const size_t n = w.n;
  const int layers = colour ? kRenLayers : kImpLayers;
  for (int l = 0; l < kImpLayers; ++l) w.Z[l] = l < layers - (colour ? 0 : 1) ? a.take<float>(n * kLd) : nullptr;
  w.in0 = a.take<float>(n * (colour ? kCinLd : kEmbLd));
  w.dA[0] = a.take<float>(n * kLd);
  w.dA[1] = a.take<float>(n * kLd);
  w.dA[2] = a.take<float>(n * (colour ? kCinLd : kLd));
  w.part = a.take<float>((size_t)w.ns * kMaxOut * kMaxIn);
  w.partb = a.take<double>((size_t)div_up(w.n, kBiasRows) * kMaxIn);
  const size_t acc_layers = n ? layers : 0;
  w.accW = a.take<double>(acc_layers * kMaxOut * kMaxIn);
  w.accB = a.take<double>(acc_layers * kMaxIn);
  w.pf = a.take<float>(colour && n ? kPoseDim : 0);
  w.amax = a.take<unsigned>(n ? kAmaxSlots : 0);
}

size_t grad_ws_bytes(int N, bool colour) {
  Arena a;
  GradWs w;
  grad_carve(a, N, colour, w);
  return a.off;
}

// one layer's parameter gradients over a chunk: dW += G^T A (M = out, N = in, K = points), db += column sums of G
template <class OA>
int layer_param_grads(const GradOp& g, const OA& a, const unsigned* amax_g, const unsigned* amax_a, int out, int in,
                      int n, int ns, bool want_w, bool want_b, const GradWs& w, double* accW, double* accB,
                      cudaStream_t st) {
  if (want_w) {
    MP_TRY((gemm<true, true>(Tr<GradOp>{g}, Tr<OA>{a}, EpiPartial{w.part, out, in}, amax_g, amax_a, out, in, n, kSplit,
                             kGroup, st)));
    reduce_partials_kernel<<<div_up(out * in, 256), 256, 0, st>>>(w.part, ns, out, in, accW);
    MP_LAUNCH_CHECK();
  }
  if (want_b) {
    const int nb = div_up(n, kBiasRows);
    colsum_kernel<<<dim3(div_up(out, 32), nb), dim3(32, 8), 0, st>>>(g, out, n, w.partb);
    MP_LAUNCH_CHECK();
    reduce_bias_kernel<<<out, 256, 0, st>>>(w.partb, nb, accB);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

int zero_out(float* p, size_t n, cudaStream_t st) {
  if (p && n) MP_CHECK_CUDA(cudaMemsetAsync(p, 0, n * sizeof(float), st));
  return 0;
}

// the input of implicit layer l: the embedding (l = 0), [h3 | embedding] (skip layer), else h_{l-1}
ActOp implicit_input(const Field& f, const GradWs& w, int l, int n) {
  const int E = f.emb_dim;
  if (l == 0) return ActOp{{w.in0, kEmbLd, E, ACT_NONE}, {nullptr, 0, 0, ACT_NONE}, n};
  if (l == f.skip_layer) return ActOp{{w.Z[l - 1], kLd, kHidden - E, ACT_SOFTPLUS}, {w.in0, kEmbLd, E, ACT_NONE}, n};
  return ActOp{{w.Z[l - 1], kLd, f.imp_in[l], ACT_SOFTPLUS}, {nullptr, 0, 0, ACT_NONE}, n};
}
// where dA of implicit layer l's input goes: ping-pong, except the skip layer's [d h3 | d embedding], which is kept
// until the embedding's backward at the end
int imp_out_buf(const Field& f, int l) { return l == f.skip_layer ? 2 : (l & 1); }

}  // namespace
}  // namespace mp

extern "C" {

size_t mp_implicit_backward_workspace_bytes(int N) { return mp::grad_ws_bytes(N, false); }
size_t mp_render_backward_workspace_bytes(int N) { return mp::grad_ws_bytes(N, true); }

int mp_implicit_backward(mp_net_t* h, const float* x, int N, const float* d_sdf, const float* d_feat, float* d_x,
                         mp_linear_grads_t* grads, float* d_cond, void* workspace, size_t workspace_bytes,
                         void* stream) {
  using namespace mp;
  MP_REQUIRE(h && N >= 0 && (x || N == 0), "mp_implicit_backward: null argument or negative N");
  const Field& f = h->f;
  const int E = f.emb_dim;
  MP_REQUIRE(E <= kEmbLd && f.cond_dim <= kMaxIn, "mp_implicit_backward: embedding of %d columns (at most %d)", E,
             kEmbLd);
  // the buffer rotation (imp_out_buf) and the skip split assume the shipped stack: 9 layers, the skip at layer 4
  MP_REQUIRE(f.n_imp == kImpLayers && f.skip_layer == 4 && f.imp_out[kImpLayers - 1] == kHidden + 1,
             "mp_implicit_backward: ImplicitNet must have 9 layers, the skip at layer 4 and 257 outputs");
  cudaStream_t st = (cudaStream_t)stream;
  mp_linear_grads_t none{};
  const mp_linear_grads_t& g = grads ? *grads : none;
  Arena a(workspace, workspace_bytes);
  GradWs w;
  grad_carve(a, N, false, w);
  if (N == 0) {      // an empty layout: nothing to refuse
    for (int l = 0; l < kImpLayers; ++l) {
      MP_TRY(zero_out(g.d_weight[l], (size_t)f.imp_out[l] * f.imp_in[l], st));
      MP_TRY(zero_out(g.d_bias[l], f.imp_out[l], st));
    }
    return zero_out(d_cond, f.cond_dim, st);
  }
  MP_TRY(a.fits("mp_implicit_backward"));
  const bool need_db0 = g.d_bias[0] || g.d_weight[0] || d_cond;
  MP_CHECK_CUDA(cudaMemsetAsync(w.accW, 0, sizeof(double) * kImpLayers * kMaxOut * kMaxIn, st));
  MP_CHECK_CUDA(cudaMemsetAsync(w.accB, 0, sizeof(double) * kImpLayers * kMaxIn, st));
  const int last = kImpLayers - 1;
  unsigned* const amW = w.amax + kAmaxW;
  unsigned* const amA = w.amax + kAmaxA;
  unsigned* const amG = w.amax + kAmaxG;
  for (int l = 0; l < kImpLayers; ++l)      // layer 0's products read its embedding columns only
    MP_TRY(absmax(MatOp{f.imp_W[l], f.imp_in[l], 1, f.imp_out[l], l == 0 ? E : f.imp_in[l]}, f.imp_out[l],
                  l == 0 ? E : f.imp_in[l], amW + l, st));
  for (int s = 0; s < N; s += kChunk) {
    const int n = min(kChunk, N - s), ns = div_up(n, kSplit);
    const float* xs = x + (size_t)f.d_in * s;
    embed_kernel<<<div_up(n, 128), 128, 0, st>>>(xs, f.d_in, f.multires, n, w.in0);
    MP_LAUNCH_CHECK();
    // recompute Z_0 .. Z_7 (layer 0: the cond is folded into its bias)
    for (int l = 0; l <= last; ++l) {
      const int K = l == 0 ? E : f.imp_in[l];
      MP_TRY(absmax(implicit_input(f, w, l, n), n, K, amA + l, st));
      if (l == last) break;      // layer 8's output is not needed
      const MatOp W{f.imp_W[l], f.imp_in[l], 1, f.imp_out[l], K};
      MP_TRY(layer_gemm<false>(implicit_input(f, w, l, n), W, amA + l, amW + l, w.Z[l], kLd,
                               l == 0 ? f.imp_b0_eff : f.imp_b[l], n, f.imp_out[l], K, st));
    }
    for (int l = last; l >= 0; --l) {
      const int out = f.imp_out[l], K = l == 0 ? E : f.imp_in[l];
      GradOp G;
      if (l == last)      // [d sdf | d feature], no activation
        G = GradOp{{d_sdf ? d_sdf + s : nullptr, 1, 1, 0}, {d_feat ? d_feat + (size_t)kHidden * s : nullptr, kHidden,
                   out - 1, 0}, nullptr, ACT_NONE, n};
      else
        G = GradOp{{w.dA[imp_out_buf(f, l + 1)], kLd, out, 0}, {nullptr, 0, 0, 0}, w.Z[l], ACT_SOFTPLUS, n};
      const ActOp Ain = implicit_input(f, w, l, n);
      MP_TRY(absmax(G, n, out, amG + l, st));
      MP_TRY(layer_param_grads(G, Ain, amG + l, amA + l, out, K, n, ns, g.d_weight[l] != nullptr,
                               g.d_bias[l] || (l == 0 && need_db0), w, w.accW + (size_t)l * kMaxOut * kMaxIn,
                               w.accB + (size_t)l * kMaxIn, st));
      if (l > 0) {
        const MatOp Wt{f.imp_Wt[l], out, 1, f.imp_in[l], out};     // [in][out]: B(n = input, k = output)
        MP_TRY(layer_gemm<false>(G, Wt, amG + l, amW + l, w.dA[imp_out_buf(f, l)], kLd, nullptr, n, f.imp_in[l], out,
                                 st));
      } else if (d_x) {
        const MatOp Wt{f.imp_Wt[0], kHidden, 1, E, kHidden};
        MP_TRY(layer_gemm<false>(G, Wt, amG, amW, w.dA[imp_out_buf(f, 0)], kLd, nullptr, n, E, kHidden, st));
        embed_backward_kernel<<<div_up(n, 128), 128, 0, st>>>(xs, f.d_in, f.multires, n, w.dA[imp_out_buf(f, 0)],
                                                              w.dA[imp_out_buf(f, f.skip_layer)], kHidden - E,
                                                              d_x + (size_t)f.d_in * s);
        MP_LAUNCH_CHECK();
      }
    }
  }
  for (int l = 0; l < kImpLayers; ++l) {
    const int out = f.imp_out[l], K = l == 0 ? E : f.imp_in[l];
    const double* aw = w.accW + (size_t)l * kMaxOut * kMaxIn;
    const double* ab = w.accB + (size_t)l * kMaxIn;
    if (g.d_weight[l]) {
      // the pack folds the skip's 1/sqrt(2) into W4; the reference's W4 sees [h3, embedding] / sqrt(2)
      const double scale = l == f.skip_layer ? 1.0 / sqrt(2.0) : 1.0;
      finalize_w_kernel<<<div_up(out * K, 256), 256, 0, st>>>(aw, out, K, scale, g.d_weight[l], f.imp_in[l], 0);
      MP_LAUNCH_CHECK();
    }
    if (g.d_bias[l]) {
      finalize_b_kernel<<<div_up(out, 256), 256, 0, st>>>(ab, out, g.d_bias[l]);
      MP_LAUNCH_CHECK();
    }
  }
  if (g.d_weight[0] || d_cond) {
    cond_grad_kernel<<<1, 128, 0, st>>>(w.accB, f.cond, f.cond_dim, f.imp_out[0], f.imp_W[0], f.imp_in[0], E,
                                        g.d_weight[0], d_cond);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

int mp_render_backward(mp_net_t* h, const float* points, const float* normals, const float* feat, int N,
                       const float* d_rgb, float* d_points, float* d_normals, float* d_feat, mp_linear_grads_t* grads,
                       float* d_lin_pose_weight, float* d_lin_pose_bias, float* d_body_pose, void* workspace,
                       size_t workspace_bytes, void* stream) {
  using namespace mp;
  MP_REQUIRE(h && N >= 0 && ((points && normals && feat && d_rgb) || N == 0),
             "mp_render_backward: null argument or negative N");
  const Field& f = h->f;
  MP_REQUIRE(!f.is_bg && f.ren_mode == 0, "mp_render_backward: not a foreground (pose_no_view) field");
  bool shape_ok = f.n_ren == kRenLayers && f.ren_in[0] == 270 && f.ren_out[kRenLayers - 1] == 3;
  for (int l = 0; l < kRenLayers - 1; ++l) shape_ok = shape_ok && f.ren_out[l] == kHidden;
  MP_REQUIRE(shape_ok, "mp_render_backward: the colour net must be 270 -> 4 x 256 -> 3");
  cudaStream_t st = (cudaStream_t)stream;
  mp_linear_grads_t none{};
  const mp_linear_grads_t& g = grads ? *grads : none;
  Arena a(workspace, workspace_bytes);
  GradWs w;
  grad_carve(a, N, true, w);
  if (N == 0) {
    for (int l = 0; l < kRenLayers; ++l) {
      MP_TRY(zero_out(g.d_weight[l], (size_t)f.ren_out[l] * f.ren_in[l], st));
      MP_TRY(zero_out(g.d_bias[l], f.ren_out[l], st));
    }
    MP_TRY(zero_out(d_lin_pose_weight, kPoseDim * kBodyPose, st));
    MP_TRY(zero_out(d_lin_pose_bias, kPoseDim, st));
    return zero_out(d_body_pose, kBodyPose, st);
  }
  MP_TRY(a.fits("mp_render_backward"));
  const bool need_db0 = g.d_bias[0] || d_lin_pose_weight || d_lin_pose_bias || d_body_pose;
  const bool need_dcin = d_points || d_normals || d_feat;
  MP_CHECK_CUDA(cudaMemsetAsync(w.accW, 0, sizeof(double) * kRenLayers * kMaxOut * kMaxIn, st));
  MP_CHECK_CUDA(cudaMemsetAsync(w.accB, 0, sizeof(double) * kRenLayers * kMaxIn, st));
  pose_feat_kernel<<<1, 32, 0, st>>>(f.ren_pose_W, f.ren_pose_b, f.cond, w.pf);
  MP_LAUNCH_CHECK();
  const int last = kRenLayers - 1;
  unsigned* const amW = w.amax + kAmaxW;
  unsigned* const amA = w.amax + kAmaxA;
  unsigned* const amG = w.amax + kAmaxG;
  for (int l = 0; l < kRenLayers; ++l)
    MP_TRY(absmax(MatOp{f.ren_W[l], f.ren_in[l], 1, f.ren_out[l], f.ren_in[l]}, f.ren_out[l], f.ren_in[l], amW + l, st));
  auto input = [&](int l, int n) {
    return l == 0 ? ActOp{{w.in0, kCinLd, 270, ACT_NONE}, {nullptr, 0, 0, ACT_NONE}, n}
                  : ActOp{{w.Z[l - 1], kLd, f.ren_in[l], ACT_RELU}, {nullptr, 0, 0, ACT_NONE}, n};
  };
  for (int s = 0; s < N; s += kChunk) {
    const int n = min(kChunk, N - s), ns = div_up(n, kSplit);
    colour_input_kernel<<<div_up(n * 270, 256), 256, 0, st>>>(points + 3 * (size_t)s, normals + 3 * (size_t)s, w.pf,
                                                             feat + (size_t)kHidden * s, n, w.in0);
    MP_LAUNCH_CHECK();
    for (int l = 0; l < kRenLayers; ++l) {
      const MatOp W{f.ren_W[l], f.ren_in[l], 1, f.ren_out[l], f.ren_in[l]};
      MP_TRY(absmax(input(l, n), n, f.ren_in[l], amA + l, st));
      MP_TRY(layer_gemm<false>(input(l, n), W, amA + l, amW + l, w.Z[l], kLd, f.ren_b[l], n, f.ren_out[l], f.ren_in[l],
                               st));
    }
    for (int l = last; l >= 0; --l) {
      const int out = f.ren_out[l], in = f.ren_in[l];
      const GradOp G = l == last ? GradOp{{d_rgb + 3 * (size_t)s, 3, 3, 0}, {nullptr, 0, 0, 0}, w.Z[l], ACT_SIGMOID, n}
                                 : GradOp{{w.dA[(l + 1) & 1], kLd, out, 0}, {nullptr, 0, 0, 0}, w.Z[l], ACT_RELU, n};
      MP_TRY(absmax(G, n, out, amG + l, st));
      MP_TRY(layer_param_grads(G, input(l, n), amG + l, amA + l, out, in, n, ns, g.d_weight[l] != nullptr,
                               g.d_bias[l] || (l == 0 && need_db0), w, w.accW + (size_t)l * kMaxOut * kMaxIn,
                               w.accB + (size_t)l * kMaxIn, st));
      if (l > 0) {
        const MatOp Wt{f.ren_Wt[l], out, 1, in, out};
        MP_TRY(layer_gemm<false>(G, Wt, amG + l, amW + l, w.dA[l & 1], kLd, nullptr, n, in, out, st));
      } else if (need_dcin) {
        const MatOp Wt{f.ren_W[0], 1, in, in, out};              // B(n = input, k = output) = W0[k][n]
        MP_TRY(layer_gemm<true>(G, Wt, amG, amW, w.dA[2], kCinLd, nullptr, n, in, out, st));
        colour_input_backward_kernel<<<div_up(n * 270, 256), 256, 0, st>>>(
            w.dA[2], n, d_points ? d_points + 3 * (size_t)s : nullptr, d_normals ? d_normals + 3 * (size_t)s : nullptr,
            d_feat ? d_feat + (size_t)kHidden * s : nullptr);
        MP_LAUNCH_CHECK();
      }
    }
  }
  for (int l = 0; l < kRenLayers; ++l) {
    const int out = f.ren_out[l], in = f.ren_in[l];
    if (g.d_weight[l]) {
      finalize_w_kernel<<<div_up(out * in, 256), 256, 0, st>>>(w.accW + (size_t)l * kMaxOut * kMaxIn, out, in, 1.0,
                                                               g.d_weight[l], in, 0);
      MP_LAUNCH_CHECK();
    }
    if (g.d_bias[l]) {
      finalize_b_kernel<<<div_up(out, 256), 256, 0, st>>>(w.accB + (size_t)l * kMaxIn, out, g.d_bias[l]);
      MP_LAUNCH_CHECK();
    }
  }
  if (d_lin_pose_weight || d_lin_pose_bias || d_body_pose) {
    pose_grad_kernel<<<1, 128, 0, st>>>(w.accB, f.ren_W[0], f.ren_in[0], f.ren_out[0], f.ren_pose_W, f.cond,
                                        d_lin_pose_weight, d_lin_pose_bias, d_body_pose);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
