// Tensor-core engine: the fused ImplicitNet (+ backward for normals) + RenderingNet chain on the
// Hopper tensor cores of sm_90a (wgmma, TMA bulk copies, mbarrier).
//   reference: lib/model/networks.py:126-208 (ImplicitNet.forward),
//              :263-312 (RenderingNet.forward), lib/model/multiply.py:620-661 (forward_gradient)
//
// Design (DESIGN.md §3.1):
//   * one persistent CTA per SM; a tile is 128 sample points.  Two consumer warpgroups own 64 rows each and
//     run the whole chain of their rows: every layer is D[64 x 256] (fp32, in registers) = A[64 x K] . W^T,
//     K in chunks of 64, as wgmma.m64n256k16 issued by the warpgroup.
//     A (the activations) lives in shared memory as fp16 hi + fp16 lo (K-major, 128B swizzle).  A warpgroup
//     only ever reads and writes its own 64 rows of A, so handing the operand to the next layer is a
//     128-thread barrier, and the two warpgroups drift freely against each other (one's epilogue overlaps
//     the other's MMAs).
//   * the weights are streamed as pre-swizzled fp16 hi/lo tiles ("slots", 256 x 64, 32 KB) by the
//     TMA engine (cp.async.bulk + mbarrier complete_tx) through a 3-slot ring that both warpgroups read.
//   * split precision: D = A_hi.W_hi + A_lo.W_hi + A_hi.W_lo (three f16 MMAs per K-step,
//     fp32 accumulate) — 22 significand bits per operand, which is what keeps RGB/SDF within the
//     1e-4 gate that a single bf16/fp16 pass misses by two orders of magnitude.
//   * warp roles: warpgroup 0 = weight loader (one lane), warpgroups 1, 2 = MMA issue + epilogue
//     (accumulator registers -> activation -> fp16 hi/lo -> shared memory through stmatrix).
//   * the whole per-sample chain runs inside the tile: embed, L0..L7 (+ sigma' stash), SDF dot,
//     the reverse sweep B7..B0 (d sdf / d x_c), normals, colour layers (the feature layer L8 folded
//     into colour layer 0, its extra inputs as a fifth K-block), RGB.
//
// Accumulator layout of wgmma.m64n256k16 (f32): thread t of a warpgroup (warp w = t / 32, lane l) holds
// register i at row 16 w + l / 4 + 8 ((i >> 1) & 1) and column 8 (i >> 2) + 2 (l % 4) + (i & 1): two rows, 64
// columns each.  Per-row results (dots, normals) are reduced over the four lanes of a quad.
#include "common.cuh"
#include <vector>
#include <mutex>
#include <type_traits>
#include <stdlib.h>

namespace mp {

// ---------------------------------------------------------------------------------------------
// program description
// ---------------------------------------------------------------------------------------------
// Step kinds: the epilogue of a layer step is compiled once per kind, so that every kind gets its own instruction
// schedule and register allocation instead of one loop that tests the step descriptor in its body.
enum {
  K_SP_PLAIN = 0,      // softplus
  K_SP_SAVE = 1,       // softplus; store d softplus / dz to the sigma' scratch (forward of the fused chain)
  K_SP_SEED = 2,       // last SDF layer of the fused chain: park h7 in scratch (it returns as the colour net's input
                       // after the reverse sweep), then A = W8[0,:] * sigma'_7 (start of the reverse sweep)
  K_FEAT = 3,          // L8 features, written to feat (operator API)
  K_BWD = 4,           // reverse sweep: g_{l-1} = (g_l * sigma'_l) . W_l
  K_FINAL_GRAD = 5,    // reverse sweep end: d sdf / d x -> grad, normal ; then reload the features into A
  K_RELU = 6           // colour layers
};
// Modifiers of a step within its kind
enum {
  F_INJECT_EMB = 1,    // columns >= inj_col receive the input embedding (skip connection, networks.py:166)
  F_SDF_DOT = 2,       // sdf = h7 . W8[0,:] + b8[0]
  F_SKIP_GRAD = 4,     // reverse sweep: columns >= inj_col are d/d embed of the skip; park them, zero A there
  F_EXTRA_IN = 8,      // colour layer 0: a fifth K-block carries the extra inputs ([x_c, n] or the view embedding): they are
                       // staged into A's K-block 0 once its MMAs have drained, and accumulate into the same tile
  F_RGB_OUT = 16       // last colour layer: rgb = sigmoid(h . Wrgb^T + b)
};
constexpr int kMaxSteps = 24;
constexpr int kSlotBytes = 32768;          // 256 rows x 64 fp16
constexpr int kRing = 3;

struct TcStep {
  int nk;               // 64-wide K chunks of A consumed by this layer (5 with F_EXTRA_IN: the last one re-uses K-block 0)
  int kind;             // K_*
  int flags;            // F_*
  int sig;              // sigma' scratch layer (save: forward, load: reverse) or -1
  const float* bias;    // [256] or nullptr
  int slot_off;         // first weight slot of this step in the blob
  int sc;               // index of this layer's 2^-s in inv_scale[]
  int terms;            // split-precision terms of this step's products: 3 = A_hi.W_hi + A_lo.W_hi + A_hi.W_lo (default),
                        // 1 = A_hi.W_hi only (the lo weight slots are then neither loaded nor issued)
};

// A step's weight slots: K-chunk kc owns two slots of the blob, hi then lo, from slot_off on (tc_programs reserves them,
// whatever the precision mode, and tc_pack writes them).  The step consumes chunk by chunk the hi slot and,
// unless it is single-term, the lo slot: the loader fetches the j-th of them in the order in which the consumers wait.
__host__ __device__ inline bool tc_one_term(const TcStep& st) { return st.terms == 1; }
__host__ __device__ inline int tc_packed_slots(int nk) { return 2 * nk; }     // the blob slots of nk K-chunks
__host__ __device__ inline int tc_slots(const TcStep& st) { return tc_one_term(st) ? st.nk : tc_packed_slots(st.nk); }
__host__ __device__ inline int tc_chunk_slot(const TcStep& st, int kc, bool lo) { return st.slot_off + 2 * kc + lo; }
__host__ __device__ inline int tc_slot(const TcStep& st, int j) {
  return tc_one_term(st) ? tc_chunk_slot(st, j, false) : tc_chunk_slot(st, j >> 1, j & 1);
}

struct TcProgram {
  int nsteps;
  TcStep step[kMaxSteps];
  const uint4* blob;     // weight slots in consumption order
  const float* inv_scale;   // [nsteps] 2^-s of each step's weights
  // network constants
  int d_in, multires, E, inj_col, n_extra;
  const float* w8row;    // W8[0,:]  [256]
  const float* b8;       // b8[0]
  const float* Wrgb;     // [3][256]
  const float* brgb;     // [3]
};

struct TcIO : MlpCall {
  float rz;              // relative truncation loss of ONE tensor-core accumulation (see kRzPerMma)
  char* scratch;         // per-CTA scratch
  size_t scratch_per_cta;
  unsigned long long* stalls;   // stall-accounting build only: per CTA [kStallWarps][MP_STALL_WORDS] clock64 totals
};

constexpr int kConsumers = 2;                                 // consumer warpgroups (64 rows each)
constexpr int kThreads = 128 * (1 + kConsumers);

// Stall accounting (mp_profile_enable(2), the PROF instantiation of the kernel): phases of a step, as laid out in
// include/multiply_b200.h
enum { PH_STEP = 0, PH_FULL = 1, PH_WGMMA = 2, PH_BAR = 3, PH_EPI = 4, PH_EMPTY = 5 };
constexpr int kStallWarps = 1 + 4 * kConsumers;               // the loader lane, then the consumer warps
static_assert(MP_STALL_WARPS == kStallWarps && MP_STALL_KINDS == K_RELU + 1 && MP_STALL_PHASES == PH_EMPTY + 1 &&
                  MP_STALL_PROLOGUE == MP_STALL_KINDS * MP_STALL_PHASES && MP_STALL_ELAPSED == MP_STALL_PROLOGUE + 1 &&
                  MP_STALL_WORDS == MP_STALL_ELAPSED + 1,
              "stall record layout of include/multiply_b200.h");
// One warp's stall record (PROF): its whole run, its tile prologues, and per step the whole step, the clocks blocked in
// each phase's waits and the epilogue, added by the lead thread (the loader lane, lane 0 of a consumer warp) to record w
// of its CTA (0 the loader lane, 1.. the consumer warps).  The default build's recorder reads no clock and adds nothing.
template <bool PROF>
struct StallRec {
  unsigned long long* rec;
  bool lead;
  long long t_run, t_tile = 0, t_step = 0, t_epi = 0, c[PH_EMPTY + 1] = {};     // c: this step's clocks in each phase
  __device__ StallRec(const TcIO& io, int w, bool lead)
      : rec(io.stalls + ((size_t)blockIdx.x * kStallWarps + w) * MP_STALL_WORDS), lead(lead), t_run(now()) {}
  static __device__ long long now() {
    if constexpr (PROF) return clock64();
    return 0;
  }
  template <int PH, class F>
  __device__ __forceinline__ void wait(F&& f) {
    const long long t0 = now();
    f();
    c[PH] += now() - t0;
  }
  __device__ void tile_start() { t_tile = now(); }
  __device__ void prologue_done() { add(MP_STALL_PROLOGUE, now() - t_tile); }
  __device__ void step_start() {
    t_step = now();
    for (long long& v : c) v = 0;
  }
  __device__ void epilogue_start() { t_epi = now(); }
  // the step's whole time and phases PH0 .. PH1 of its kind: the loader's PH_EMPTY, the consumers' PH_FULL .. PH_EPI
  template <int PH0, int PH1>
  __device__ void step_done(int kind) {
    const long long t = now();
    if constexpr (PH1 >= PH_EPI) c[PH_EPI] = t - t_epi;
    add(kind * MP_STALL_PHASES + PH_STEP, t - t_step);
    for (int ph = PH0; ph <= PH1; ++ph) add(kind * MP_STALL_PHASES + ph, c[ph]);
  }
  __device__ void run_done() { add(MP_STALL_ELAPSED, now() - t_run); }
  __device__ void add(int word, long long clocks) {
    if (PROF && lead) atomicAdd(rec + word, (unsigned long long)clocks);
  }
};

// per-CTA scratch layout (bytes); sigma' and the stashed features are indexed by (warpgroup, register group, thread)
constexpr size_t kSigBytes = (size_t)8 * kConsumers * 32 * 128 * 16;   // sigma' [8][2][32][128] float4
constexpr size_t kFeatBytes = (size_t)kConsumers * 32 * 128 * 16;      // features [2][hi 16 | lo 16][128] uint4
constexpr size_t kGeBytes = (size_t)96 * 128 * 4;            // skip gradient [E<=96][128 rows]
constexpr size_t kEmbBytes = (size_t)96 * 128 * 4;           // input embedding of the tile [E<=96][128 rows]
constexpr size_t kScratchPerCta = kSigBytes + kFeatBytes + kGeBytes + kEmbBytes;

// The epilogue's scratch reads (sigma' in the reverse sweep, the stashed features) go through volatile asm, which the
// compiler keeps in program order with the discard of the previous group (which waits for that group's data) and the
// stmatrix stores: issued in place, every load would start only after the previous one returned.  So they are issued
// kAhead of the epilogue's 16 column groups (16 columns each) ahead of their use.
constexpr int kAhead = 4;
// The epilogue issues the arithmetic of kEpiW column groups before their stores, and loads the per-step constants a
// group reads (bias, W8 row, rgb weights) kCAhead groups ahead of their use, in registers the epilogue frees as it
// stores the accumulator's column groups.
constexpr int kEpiW = 2;
constexpr int kCAhead = 3;

// shared memory carve-up
constexpr int kABytes = 2 * 4 * 128 * 128;                   // hi + lo, 4 K-blocks of [128 x 128B]
constexpr int kSmemBytes = kABytes + kRing * kSlotBytes + 256 + 1024;
static_assert(kSmemBytes <= 232448, "shared memory budget of one CTA (227 KB)");

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// bulk prefetch of `bytes` (a multiple of 16) of global memory into L2
__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// barrier of one consumer warpgroup (ids 1, 2)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// The MMAs write the accumulator registers asynchronously: after a wait, this tells the compiler that every register
// may have changed, so that no read of the accumulator is scheduled before the wait.
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define MP_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define MP_D16(i) MP_D4(i), MP_D4(i + 4), MP_D4(i + 8), MP_D4(i + 12)
// D[64 x 256] += A[64 x 16] . B[256 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, 1, 1, 1, 0, 0;\n"
      : MP_D16(0), MP_D16(16), MP_D16(32), MP_D16(48), MP_D16(64), MP_D16(80), MP_D16(96), MP_D16(112)
      : "l"(a_desc), "l"(b_desc));
}
#undef MP_D16
#undef MP_D4
// D[64 x 256] = A[64 x 16] . B[256 x 16]^T: the first MMA of a layer step (scale-d 0).  Its outputs are write-only, so
// the previous step's accumulator is dead once its epilogue has read it, and the registers of the column groups an
// epilogue has already stored are free for the rest of that epilogue.  The MMA writes them asynchronously: the "+f"
// operands of the step's later MMAs and of acc_fence keep them in place until the wait.
#define MP_D4(i) "=f"(d[i]), "=f"(d[i + 1]), "=f"(d[i + 2]), "=f"(d[i + 3])
#define MP_D16(i) MP_D4(i), MP_D4(i + 4), MP_D4(i + 8), MP_D4(i + 12)
__device__ __forceinline__ void wgmma_f16_first(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, 0, 1, 1, 0, 0;\n"
      : MP_D16(0), MP_D16(16), MP_D16(32), MP_D16(48), MP_D16(64), MP_D16(80), MP_D16(96), MP_D16(112)
      : "l"(a_desc), "l"(b_desc));
}
#undef MP_D16
#undef MP_D4

// K-major, 128-byte swizzle shared-memory matrix descriptor of wgmma:
//   [0,14) start>>4, [16,30) LBO>>4 (unused for swizzled K-major, 1), [32,46) SBO>>4 = 1024B between
//   8-row groups, [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// ---------------------------------------------------------------------------------------------
// the weight ring
// ---------------------------------------------------------------------------------------------
// kRing shared-memory slots, each with a `full` barrier (the loader's expect_tx, completed by the bulk copy) and an
// `empty` barrier.  The loader and each consumer warpgroup walk the same ring positions, one per slot of the tc_slot
// schedule: position it is slot it % kRing in round it / kRing.
constexpr int kEmptyArrivals = 4 * kConsumers;     // one release per consumer warp
struct Ring {
  char* slots;           // [kRing][kSlotBytes]
  uint64_t* full;        // [kRing]
  uint64_t* empty;       // [kRing]
  uint32_t it = 0;
  __device__ __forceinline__ static int slot(uint32_t pos) { return pos % kRing; }
  __device__ __forceinline__ uint32_t phase() const { return (it / kRing) & 1; }
  __device__ __forceinline__ char* data() const { return slots + (size_t)slot(it) * kSlotBytes; }
  __device__ __forceinline__ void init() const {
    for (int i = 0; i < kRing; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kEmptyArrivals);
    }
  }
  // loader: wait until the previous round of position it has been released, then fill it from src
  __device__ __forceinline__ void wait_empty() const { mbar_wait(&empty[slot(it)], phase() ^ 1); }
  __device__ __forceinline__ void fill(const char* src) {
    mbar_expect_tx(&full[slot(it)], kSlotBytes);
    bulk_g2s(data(), src, kSlotBytes, &full[slot(it)]);
    ++it;
  }
  // consumers
  __device__ __forceinline__ void wait_full() const { mbar_wait(&full[slot(it)], phase()); }
  __device__ __forceinline__ void release(uint32_t pos) const {
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[slot(pos)]);
  }
};

// A consumer warpgroup's side of the ring, one per layer step.  Every weight slot's MMAs form one commit group.  A slot
// is released as soon as the group after it has been committed and all but that newest group have completed, so a
// warpgroup holds at most one slot in flight while it waits for the next: the ring (3 slots) never waits on a slot
// that its own reader still holds.  The waits are timed by the warp's stall recorder.
template <bool PROF>
struct RingReader {
  Ring& ring;
  StallRec<PROF>& rec;
  bool held = false;       // a slot whose MMAs may still be running
  uint32_t held_pos = 0;
  // the shared address of the next slot, once it is filled
  __device__ __forceinline__ uint32_t wait_full() {
    rec.template wait<PH_FULL>([&] { ring.wait_full(); });
    return smem_u32(ring.data());
  }
  // the MMAs over the slot of wait_full() have been issued
  __device__ __forceinline__ void issued() {
    wgmma_commit();
    if (held) {
      rec.template wait<PH_WGMMA>([] { wgmma_wait<1>(); });
      ring.release(held_pos);
    }
    held = true;
    held_pos = ring.it++;
  }
  // wait for every MMA issued into acc, and release the slot still held
  __device__ __forceinline__ void drain(float* acc) {
    rec.template wait<PH_WGMMA>([&] { wgmma_wait<0>(); acc_fence(acc); });
    if (held) ring.release(held_pos);
    held = false;
  }
};

// ---------------------------------------------------------------------------------------------
// epilogue helpers
// ---------------------------------------------------------------------------------------------
// byte offset of (row, 8-column chunk `ch` of K-block `kb`) in the swizzled A image
__device__ __forceinline__ uint32_t a_off(int row, int kb, int ch) {
  return (uint32_t)(kb * 16384 + row * 128 + ((ch ^ (row & 7)) << 4));
}

__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(a, b);
  float2 f = __half22float2(h);
  __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *(uint32_t*)&h;
  lo = *(uint32_t*)&l;
}
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  split2(v[0], v[1], hi.x, lo.x);
  split2(v[2], v[3], hi.y, lo.y);
  split2(v[4], v[5], hi.z, lo.z);
  split2(v[6], v[7], hi.w, lo.w);
}

// 16-byte store into the operand image through a 32-bit shared-window address.
// (volatile, no memory clobber: ordered against the volatile proxy fence that publishes the image; no C++ access reads
// these bytes back.)
__device__ __forceinline__ void sts128(uint32_t A32, uint32_t off, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(A32 + off), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}
// one fp16 element of the operand image (same ordering as sts128)
__device__ __forceinline__ void sts16(uint32_t A32, uint32_t off, __half v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(A32 + off), "h"(__half_as_ushort(v)));
}
// eight consecutive columns of one row
__device__ __forceinline__ void store_a8(uint32_t A32, int row, int col, const float* v) {
  uint4 hi, lo;
  split8(v, hi, lo);
  uint32_t o = a_off(row, col >> 6, (col >> 3) & 7);
  sts128(A32, o, hi);
  sts128(A32, 65536 + o, lo);
}
__device__ __forceinline__ void stsm4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t e) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c),
               "r"(e));
}
// Accumulator registers 8 jp .. 8 jp + 7 (columns 16 jp .. 16 jp + 15 of the thread's two rows), already split into
// fp16 hi / lo pairs, -> A.  stmatrix writes four 8 x 8 blocks: (column group 2 jp, rows 0-7 | rows 8-15 of the warp's
// 16), then column group 2 jp + 1; lane l gives the address of row l % 8 of block l / 8.  `lane_base` is A + that
// row * 128, `lane_x` the swizzle term ((l / 16) ^ (row & 7)) of the block's 16-byte chunk.
__device__ __forceinline__ void store_pairs(uint32_t lane_base, uint32_t lane_x, int jp, const uint4& hi, const uint4& lo) {
  const uint32_t addr = lane_base + (uint32_t)(jp >> 2) * 16384u + ((((uint32_t)(2 * jp) & 7u) ^ lane_x) << 4);
  stsm4(addr, hi.x, hi.y, hi.z, hi.w);
  stsm4(addr + 65536u, lo.x, lo.y, lo.z, lo.w);
}
__device__ __forceinline__ void store_acc16(uint32_t lane_base, uint32_t lane_x, int jp, const float* v) {
  uint4 hi, lo;
  split8(v, hi, lo);
  store_pairs(lane_base, lane_x, jp, hi, lo);
}

template <int V>
using IntC = std::integral_constant<int, V>;
// f(IntC<flags & MASK>): one instantiation of f for every subset of the flags in MASK
template <int MASK, int FL = 0, class F>
__device__ __forceinline__ void with_flags(int flags, F&& f) {
  if constexpr (MASK == 0) {
    f(IntC<FL>{});
  } else {
    constexpr int bit = MASK & -MASK;
    if (flags & bit) with_flags<MASK & ~bit, FL | bit>(flags, f);
    else with_flags<MASK & ~bit, FL>(flags, f);
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// The per-CTA scratch (sigma', stashed features) streams: it is written once and read once per tile.  L2-only
// accesses keep it out of the small L1 that is left beside 224 KB of shared memory, so that the read-only vectors
// every column group needs (bias, W8 row, rgb weights) stay L1-resident.
__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
// (volatile, no memory clobber: the scratch these stores write is read back only by ld_stream, whose volatile asm stays
// in program order with them, and by no C++ access.)
__device__ __forceinline__ void st_stream(float4* p, const float4& v) {
  asm volatile("st.global.cg.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
}
__device__ __forceinline__ void st_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

// The scratch lines of a tile are dead once read (sigma' and the stashed features are written once and read once):
// `discard.global.L2` drops the line without write-back, so the dead lines neither travel to DRAM when they are
// evicted nor compete for L2 capacity with the live part of the stash.  `dep` is a value computed FROM the loaded
// data: the consumer instruction waits for the load of every lane of the warp, so the discard cannot overtake it.
__device__ __forceinline__ void discard_line(const void* p, float dep) {
  asm volatile("discard.global.L2 [%0], 128;" ::"l"(p), "f"(dep) : "memory");
}
__device__ __forceinline__ void discard_line(const void* p, uint32_t dep) {
  asm volatile("discard.global.L2 [%0], 128;" ::"l"(p), "r"(dep) : "memory");
}

// softplus(beta=100, threshold=20) and its derivative (networks.py:85)
// Branch-free so that the elements pipeline through the MUFU unit (a per-element branch serialises
// them).  Raw MUFU approximations (ex2 / lg2 / rcp .approx.ftz) without the
// denormal fix-ups of __expf/__logf: 1+u >= 1, the overflow side is replaced by the linear branch, results only need
// ~1e-7 absolute accuracy (softplus = log1p(exp(100 z))/100).
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float softplus_fast(float z) {
  float t = z * 144.26950408889634f;                 // 100 z log2(e)
  float u = ex2_approx(t);                           // inf above ~128: discarded by the select below
  float y = lg2_approx(1.f + u) * 0.0069314718055994531f;   // ln2 / 100
  return t > 28.853900817779268f ? z : y;
}
__device__ __forceinline__ void softplus_fast_grad(float z, float& y, float& d) {
  float t = z * 144.26950408889634f;
  float u = ex2_approx(t);                           // inf above ~128: u * rcp(inf) = NaN, discarded below
  float w = 1.f + u;
  float r = rcp_approx(w);
  float ys = lg2_approx(w) * 0.0069314718055994531f;
  bool big = t > 28.853900817779268f;
  y = big ? z : ys;
  d = big ? 1.f : u * r;
}

// Last step of the reverse sweep (K_FINAL_GRAD): d sdf / d x of the thread's two rows from B0's accumulator, written to
// io.grad, and the normals, written to io.nrm and returned in nrm (the foreground colour net's extra inputs).
// B0's output columns are permuted at pack time BY AXIS: columns [16 a, 16 a + 16) (a < d_in) hold every embedding index
// that depends on x_a -- [x_a, sin(2^0 x_a), cos(2^0 x_a), sin(2^1 x_a), ...] (embedders.py:8-34) -- so the chain rule
//   d sdf / d x_a = sum_k (g_k + skip_k) * d embed_k / d x_a
// of one axis lives in column groups 2 a, 2 a + 1, reduced over the quad.  The skip gradient (parked at the F_SKIP_GRAD
// step) and the partner sin / cos of each index (parked by the tile prologue) come from scratch.
__device__ __forceinline__ void final_grad(const TcProgram& P, const TcIO& io, const float* acc, float isc, int q,
                                           const float* ge, const float* emb, const int (&rowt)[2],
                                           const bool (&valid)[2], const int (&pt)[2], const int (&slot)[2],
                                           float (&nrm)[2][3]) {
  const int d = P.d_in;
  float gax[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const int nterm = 1 + 2 * P.multires;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < 2 * d) {
      const int a = j >> 1;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int jj = (8 * j + 2 * q + (e & 1)) & 15;
        if (jj < nterm) {
          const int h = e >> 1;
          // jj = 0: x_a itself; jj = 1 + 2 f: sin(2^f x_a); jj = 2 + 2 f: cos(2^f x_a)
          const int fq = (jj - 1) >> 1;
          const bool is_cos = ((jj - 1) & 1) != 0;
          const int k = (jj == 0) ? a : d + 2 * fq * d + (is_cos ? d : 0) + a;
          const float pg = ge[(size_t)k * 128 + rowt[h]];
          const float tot = fmaf(acc[4 * j + e], isc, pg);     // through layer 0 + through the skip connection
          float w = 1.f;
          if (jj > 0) {
            // partner: cos for a sin entry (+d), sin for a cos entry (-d)
            const float pe = emb[(size_t)(is_cos ? k - d : k + d) * 128 + rowt[h]];
            // d sin(2^f x) = 2^f cos(2^f x) ; d cos(2^f x) = -2^f sin(2^f x)
            w = (float)(1 << fq) * (is_cos ? -pe : pe);
          }
          gax[h][a] = fmaf(w, tot, gax[h][a]);
        }
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int a = 0; a < 4; ++a) gax[h][a] = quad_sum(gax[h][a]);
    // normal = normalize(g . J^-1) (multiply.py:661), normalised again with eps 1e-6 (:606)
    const float gx0 = gax[h][0], gx1 = d > 1 ? gax[h][1] : 0.f, gx2 = d > 2 ? gax[h][2] : 0.f;
    if (q == 0 && io.grad && valid[h]) {
      io.grad[3 * (size_t)pt[h]] = gx0;
      io.grad[3 * (size_t)pt[h] + 1] = gx1;
      io.grad[3 * (size_t)pt[h] + 2] = gx2;
    }
    float n0 = 0.f, n1 = 0.f, n2 = 0.f;
    if (io.jinv && valid[h]) {
      const float4* J4 = (const float4*)(io.jinv + 12 * (size_t)pt[h]);
      const float4 ja = __ldg(J4), jb = __ldg(J4 + 1), jc = __ldg(J4 + 2);
      float v0 = gx0 * ja.x + gx1 * ja.w + gx2 * jb.z;
      float v1 = gx0 * ja.y + gx1 * jb.x + gx2 * jb.w;
      float v2 = gx0 * ja.z + gx1 * jb.y + gx2 * jc.x;
      float nr = fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-12f);     // multiply.py:661
      const float inr = 1.f / nr;
      v0 *= inr; v1 *= inr; v2 *= inr;
      float n2r = fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-6f);     // multiply.py:606
      const float in2 = 1.f / n2r;
      n0 = v0 * in2; n1 = v1 * in2; n2 = v2 * in2;
      if (q == 0 && io.nrm) {
        io.nrm[3 * (size_t)slot[h]] = n0;
        io.nrm[3 * (size_t)slot[h] + 1] = n1;
        io.nrm[3 * (size_t)slot[h] + 2] = n2;
      }
    }
    nrm[h][0] = n0;
    nrm[h][1] = n1;
    nrm[h][2] = n2;
  }
}

// ---------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------
// The loader lane: every step's weight slots of every tile, in tc_slot order, each into the next ring position once
// it is free.
template <bool PROF>
__device__ __forceinline__ void load_weights(const TcProgram& P, const TcIO& io, Ring ring, int ntiles) {
  StallRec<PROF> rec(io, 0, true);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    for (int s = 0; s < P.nsteps; ++s) {
      const TcStep& st = P.step[s];
      rec.step_start();
      for (int j = 0; j < tc_slots(st); ++j) {
        rec.template wait<PH_EMPTY>([&] { ring.wait_empty(); });
        ring.fill((const char*)P.blob + (size_t)tc_slot(st, j) * kSlotBytes);
      }
      rec.template step_done<PH_EMPTY, PH_EMPTY>(st.kind);
    }
  }
  rec.run_done();
}

// PROF: the stall-accounting build (mp_profile_enable(2)); the default build reads no clock.
template <bool PROF>
__global__ void __launch_bounds__(kThreads, 1) tc_chain_kernel(const __grid_constant__ TcProgram P,
                                                               const __grid_constant__ TcIO io) {
  extern __shared__ uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // 1024-byte aligned carve-up (SWIZZLE_128B atoms)
  char* base = (char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  char* A = base;                                   // [hi | lo] x 4 K-blocks
  const uint32_t A32 = smem_u32(A);
  char* slots = base + kABytes;                     // kRing weight slots, then their full and empty barriers
  uint64_t* bars = (uint64_t*)(slots + kRing * kSlotBytes);
  Ring ring{slots, bars, bars + kRing};

  const int count = io.count ? min(io.cap, *io.count) : io.cap;
  const int ntiles = (count + 127) >> 7;

  if (threadIdx.x == 0) {
    ring.init();
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== weight loader =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && lane == 0) load_weights<PROF>(P, io, ring, ntiles);
    return;
  }
  // ===================== consumer warpgroups: MMAs + epilogue =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  StallRec<PROF> rec(io, warp - 3, lane == 0);
  const int g = (warp >> 2) - 1;                 // consumer warpgroup: tile rows 64 g .. 64 g + 63
  const int t = threadIdx.x & 127;               // thread in the warpgroup
  const int wq = warp & 3, q = lane & 3;
  const int bar_id = 1 + g;
  int rowt[2];                                   // this thread's two tile rows
  rowt[0] = 64 * g + 16 * wq + (lane >> 2);
  rowt[1] = rowt[0] + 8;
  // stmatrix addressing (store_pairs)
  const int mi = lane >> 3, rr = lane & 7;
  const uint32_t lane_base = A32 + (uint32_t)(64 * g + 16 * wq + 8 * (mi & 1) + rr) * 128u;
  const uint32_t lane_x = (uint32_t)((mi >> 1) ^ rr);
  const uint32_t a_hi = A32 + (uint32_t)g * 8192u, a_lo = a_hi + 65536u;   // this warpgroup's 64 rows of A

  char* scr = io.scratch + (size_t)blockIdx.x * io.scratch_per_cta;
  float4* sig = (float4*)scr;                                  // [8][2][32][128]
  uint4* fsc = (uint4*)(scr + kSigBytes) + (size_t)g * 32 * 128;   // [hi 16 | lo 16][128] of this warpgroup
  float* ge = (float*)(scr + kSigBytes + kFeatBytes);          // [96][128]
  float* emb = (float*)(scr + kSigBytes + kFeatBytes + kGeBytes);   // [96][128]
  const int d = P.d_in, E = P.E;

  float acc[128];                                // written by each step's first MMA (wgmma_f16_first)

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    rec.tile_start();
    int pt[2], slot[2];
    bool valid[2];
    float x[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      pt[h] = tile * 128 + rowt[h];
      valid[h] = pt[h] < count;
      for (int a = 0; a < 4; ++a) x[h][a] = 0.f;
      if (valid[h])
        for (int a = 0; a < d; ++a) x[h][a] = io.x[(size_t)pt[h] * d + a];
      slot[h] = valid[h] ? (io.slot ? io.slot[pt[h]] : pt[h]) : 0;
    }
    // ---- tile prologue: embedding -> A (K-blocks 0 .. nk0-1), zero padded ----
    {
      // positional embedding (embedders.py:8-34): the (frequency, axis) pairs of a row are split over the four lanes
      // that hold it, one sincosf each, parked in scratch so that the skip connection of layer 4 and the chain rule at
      // the end of the reverse sweep re-read instead of recomputing them
      const int npair = d * P.multires;
      for (int pi = q; pi < npair; pi += 4) {
        const int f = pi / d, a = pi - f * d;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float sn, cs;
          sincosf(__fmul_rn(x[h][a], (float)(1 << f)), &sn, &cs);
          emb[(size_t)(d + 2 * f * d + a) * 128 + rowt[h]] = sn;
          emb[(size_t)(d + (2 * f + 1) * d + a) * 128 + rowt[h]] = cs;
        }
      }
      if (q == 0)
        for (int a = 0; a < d; ++a)
#pragma unroll
          for (int h = 0; h < 2; ++h) emb[(size_t)a * 128 + rowt[h]] = x[h][a];
      if (io.dirs) {
        // background: embedding of the view direction (n_extra = 3 + 6 * frequencies values), same split
        float dv[2][3];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          for (int a = 0; a < 3; ++a) dv[h][a] = valid[h] ? io.dirs[(size_t)pt[h] * 3 + a] : 0.f;
        const int nvp = (P.n_extra - 3) / 2;
        for (int pi = q; pi < nvp; pi += 4) {
          const int f = pi / 3, a = pi - f * 3;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float sn, cs;
            sincosf(__fmul_rn(dv[h][a], (float)(1 << f)), &sn, &cs);
            ge[(size_t)(3 + 6 * f + a) * 128 + rowt[h]] = sn;
            ge[(size_t)(3 + 6 * f + 3 + a) * 128 + rowt[h]] = cs;
          }
        }
        if (q == 0)
          for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int h = 0; h < 2; ++h) ge[(size_t)a * 128 + rowt[h]] = dv[h][a];
      }
      __threadfence_block();
      wg_sync(bar_id);
      const int njp = P.step[0].nk * 4;
      for (int jp = 0; jp < njp; ++jp) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = 16 * jp + 8 * (i >> 2) + 2 * q + (i & 1);
          v[i] = (c < E) ? emb[(size_t)c * 128 + rowt[(i >> 1) & 1]] : 0.f;
        }
        store_acc16(lane_base, lane_x, jp, v);
      }
    }
    // colour-net extra inputs: foreground [x_c, n] (networks.py:281) live in registers (n arrives at the end of the
    // reverse sweep); the background view-dir embedding (:275) was parked in `ge` by the prologue
    float nrm[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    rec.prologue_done();
    for (int s = 0; s < P.nsteps; ++s) {
      const TcStep st = P.step[s];
      rec.step_start();
      // 2^-s of the weight scaling, times the compensation of the accumulator's round-toward-zero (kRzPerMma)
      const float isc = P.inv_scale[st.sc] * fmaf(io.rz, (float)(4 * st.nk * (tc_one_term(st) ? 1 : 3)), 1.f);
      // The 132 CTAs' stash (1.2 MB each) does not fit in L2: the sigma' this reverse step's epilogue reads, and the
      // features the final-gradient step reloads, were mostly evicted to DRAM since the forward sweep wrote them.  Pull
      // this warpgroup's 64 KB block back into L2 while the step's MMAs run, so the epilogue's loads hit L2.  (Issued
      // one step earlier it gains less: the block competes longer with the rest of the stash.)
      if (t == 0) {
        char* ws = io.scratch + (size_t)blockIdx.x * io.scratch_per_cta;
        if (st.kind == K_BWD && st.sig >= 0)
          prefetch_l2(ws + (((size_t)st.sig * kConsumers + g) * 32 * 128) * 16, 32 * 128 * 16);
        if (st.kind == K_FINAL_GRAD) prefetch_l2(ws + kSigBytes + (size_t)g * 32 * 128 * 16, 32 * 128 * 16);
      }

      // ---------------- MMAs: acc = A . W^T over st.nk K-blocks ----------------
      // this warpgroup's rows of A are complete: publish them to the tensor cores
      fence_async_smem();
      rec.template wait<PH_BAR>([&] { wg_sync(bar_id); });
      wgmma_fence();
      RingReader<PROF> rd{ring, rec};
      // The MMAs over K-chunk kc.  FIRST (kc = 0): its first MMA starts the accumulator, so that no accumulator value
      // lives from one step into the next.  ONE_TERM: A_hi.W_hi only.  Both are compile-time, so that no MMA sits on a
      // branch between two others (ptxas would serialise the MMAs to move the accumulator registers there).
      auto chunk = [&](int kc, auto first, auto one) {
        constexpr bool FIRST = decltype(first)::value, ONE_TERM = decltype(one)::value;
        if (!FIRST && kc == 4) {
          // extra-input K-block (colour layer 0): once the MMAs over K-block 0 have drained it, this row's extra inputs
          // (16 columns per lane of the quad, zero padded to 64) take its place and accumulate into the same tile
          rd.drain(acc);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int c8 = 0; c8 < 16; c8 += 8) {
              const int e0 = 16 * q + c8;
              float xv[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) xv[j] = 0.f;
              if (io.dirs) {
#pragma unroll
                for (int j = 0; j < 8; ++j)
                  if (e0 + j < P.n_extra) xv[j] = ge[(size_t)(e0 + j) * 128 + rowt[h]];
              } else if (e0 == 0) {
                xv[0] = x[h][0]; xv[1] = x[h][1]; xv[2] = x[h][2];
                xv[3] = nrm[h][0]; xv[4] = nrm[h][1]; xv[5] = nrm[h][2];
              }
              store_a8(A32, rowt[h], e0, xv);
            }
          }
          fence_async_smem();
          rec.template wait<PH_BAR>([&] { wg_sync(bar_id); });
          wgmma_fence();
        }
        const uint32_t ka = (uint32_t)(kc & 3) * 16384u;
        // hi slot (tc_chunk_slot(st, kc, false)): A_hi.W_hi + A_lo.W_hi
        uint32_t wb = rd.wait_full();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t bd = make_desc(wb + ks * 32);
          if (FIRST && ks == 0) wgmma_f16_first(acc, make_desc(a_hi + ka + ks * 32), bd);
          else wgmma_f16(acc, make_desc(a_hi + ka + ks * 32), bd);
          if constexpr (!ONE_TERM) wgmma_f16(acc, make_desc(a_lo + ka + ks * 32), bd);
        }
        rd.issued();
        if constexpr (!ONE_TERM) {
          // lo slot (tc_chunk_slot(st, kc, true)): A_hi.W_lo
          wb = rd.wait_full();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) wgmma_f16(acc, make_desc(a_hi + ka + ks * 32), make_desc(wb + ks * 32));
          rd.issued();
        }
      };
      auto mmas = [&](auto one) {
        chunk(0, std::true_type{}, one);
        for (int kc = 1; kc < st.nk; ++kc) chunk(kc, std::false_type{}, one);
      };
      if (tc_one_term(st)) mmas(std::true_type{});
      else mmas(std::false_type{});
      rd.drain(acc);

      // ---------------- epilogue ----------------
      rec.epilogue_start();
      auto reload_features = [&]() {
        // loaded kAhead groups ahead of their use: a load issued after the previous group's discard and stmatrix
        // would wait for that group's load to return (see kAhead)
        uint4 pre[kAhead][2];
#pragma unroll
        for (int k = 0; k < kAhead; ++k) {
          pre[k][0] = ld_stream(&fsc[(size_t)k * 128 + t]);
          pre[k][1] = ld_stream(&fsc[(size_t)(16 + k) * 128 + t]);
        }
#pragma unroll
        for (int jp = 0; jp < 16; ++jp) {
          const uint4 fh = pre[jp % kAhead][0];
          const uint4 fl = pre[jp % kAhead][1];
          if (jp + kAhead < 16) {
            pre[jp % kAhead][0] = ld_stream(&fsc[(size_t)(jp + kAhead) * 128 + t]);
            pre[jp % kAhead][1] = ld_stream(&fsc[(size_t)(16 + jp + kAhead) * 128 + t]);
          }
          store_pairs(lane_base, lane_x, jp, fh, fl);
          if ((lane & 7) == 0) {
            discard_line(&fsc[(size_t)jp * 128 + t], fh.x);
            discard_line(&fsc[(size_t)(16 + jp) * 128 + t], fl.x);
          }
        }
      };
      if (st.kind == K_FINAL_GRAD) {
        final_grad(P, io, acc, isc, q, ge, emb, rowt, valid, pt, slot, nrm);
        // the MMAs of the reverse sweep are done with A: the features return as the colour net's input
        if (s + 1 < P.nsteps) reload_features();
        rec.template step_done<PH_FULL, PH_EPI>(st.kind);
        continue;
      }

      // The epilogue of one step kind.  FL: the step's flags that change the column loop (F_SDF_DOT, F_RGB_OUT), fixed
      // at compile time so that the unrolled loop holds no branch on them.  The 16 column groups are taken W at a
      // time: the arithmetic of all W groups first, then their stores (sigma', the feature stash, stmatrix), so that
      // the MUFU work of several groups overlaps.  The per-step constants a group reads (bias, W8 row, rgb weights)
      // are loaded kCAhead groups ahead of their use.
      auto run_epi = [&](auto kind, auto flags) {
        constexpr int KIND = decltype(kind)::value;
        constexpr int FL = decltype(flags)::value;
        constexpr bool kBias = KIND != K_BWD;
        constexpr bool kW8 = KIND == K_SP_SEED || (FL & F_SDF_DOT) != 0;
        constexpr bool kRgb = KIND == K_RELU && (FL & F_RGB_OUT) != 0;
        // the reverse step stores nothing but the next A: batching its groups gains nothing there and measured slower
        constexpr int W = KIND == K_BWD ? 1 : kEpiW;
        float dot[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};     // sdf / rgb partial dots of the two rows
        struct Consts {
          float2 b[2], w8[2], rgb[2][3];     // of the group's two 8-column halves
        };
        auto load_consts = [&](int jp, Consts& k) {
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int c = 16 * jp + 8 * jj + 2 * q;
            if constexpr (kBias) k.b[jj] = __ldg((const float2*)(st.bias + c));
            if constexpr (kW8) k.w8[jj] = __ldg((const float2*)(P.w8row + c));
            if constexpr (kRgb) {
#pragma unroll
              for (int kk = 0; kk < 3; ++kk) k.rgb[jj][kk] = __ldg((const float2*)(P.Wrgb + 256 * kk + c));
            }
          }
        };
        Consts cpre[kCAhead];
#pragma unroll
        for (int k = 0; k < kCAhead; ++k) load_consts(k, cpre[k]);
        // K_BWD: this step's sigma' groups j = 0 .. 31 (8 columns each), loaded 2 kAhead groups ahead of their use
        const float4* sig_g = &sig[((size_t)(st.sig < 0 ? 0 : st.sig) * kConsumers + g) * 32 * 128 + t];
        float4 sig_pre[2 * kAhead];
        if constexpr (KIND == K_BWD) {
#pragma unroll
          for (int k = 0; k < 2 * kAhead; ++k)
            sig_pre[k] = st.sig >= 0 ? ld_stream(sig_g + (size_t)k * 128) : make_float4(1.f, 1.f, 1.f, 1.f);
        }
#pragma unroll
        for (int jp0 = 0; jp0 < 16; jp0 += W) {
          float dsv[W][2][4];            // K_SP_SAVE: sigma' of the groups' two 8-column halves
          float yv[W][8];                // K_SP_SEED: h7 (the stashed features); A receives the seed
#pragma unroll
          for (int wi = 0; wi < W; ++wi) {
            const int jp = jp0 + wi;
            float* v = acc + 8 * jp;
            const Consts cs = cpre[jp % kCAhead];
            if (jp + kCAhead < 16) load_consts(jp + kCAhead, cpre[jp % kCAhead]);
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              const int j = 2 * jp + jj;
              const int c = 8 * j + 2 * q;     // columns c, c + 1 of u[0], u[1] (row 0) and u[2], u[3] (row 1)
              float* u = v + 4 * jj;
              float b[2] = {0.f, 0.f};
              if constexpr (kBias) {
                b[0] = cs.b[jj].x;
                b[1] = cs.b[jj].y;
              }
              if constexpr (KIND == K_SP_SEED) {
                // last SDF layer of the fused chain: sigma'_7 is consumed right here -- the reverse sweep starts from
                // A = W8[0,:] * sigma'_7 (d sdf / d z7), h7 only feeds the sdf dot and the feature stash
                const float w[2] = {cs.w8[jj].x, cs.w8[jj].y};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  float y, dd;
                  softplus_fast_grad(fmaf(u[e], isc, b[e & 1]), y, dd);
                  dot[e >> 1][0] = fmaf(y, w[e & 1], dot[e >> 1][0]);
                  yv[wi][4 * jj + e] = y;
                  u[e] = dd * w[e & 1];
                }
              } else if constexpr (KIND == K_SP_SAVE || KIND == K_SP_PLAIN) {
                if constexpr (KIND == K_SP_SAVE) {
#pragma unroll
                  for (int e = 0; e < 4; ++e) softplus_fast_grad(fmaf(u[e], isc, b[e & 1]), u[e], dsv[wi][jj][e]);
                } else {
#pragma unroll
                  for (int e = 0; e < 4; ++e) u[e] = softplus_fast(fmaf(u[e], isc, b[e & 1]));
                }
                if constexpr ((FL & F_SDF_DOT) != 0) {
                  const float2 w2 = cs.w8[jj];
                  dot[0][0] = fmaf(u[0], w2.x, fmaf(u[1], w2.y, dot[0][0]));
                  dot[1][0] = fmaf(u[2], w2.x, fmaf(u[3], w2.y, dot[1][0]));
                }
              } else if constexpr (KIND == K_FEAT) {
#pragma unroll
                for (int e = 0; e < 4; ++e) u[e] = fmaf(u[e], isc, b[e & 1]);
                if (io.feat) {
#pragma unroll
                  for (int h = 0; h < 2; ++h)
                    if (valid[h]) *(float2*)(io.feat + (size_t)pt[h] * 256 + c) = make_float2(u[2 * h], u[2 * h + 1]);
                }
              } else if constexpr (KIND == K_BWD) {
                const float4 s4 = sig_pre[j % (2 * kAhead)];
                if (j + 2 * kAhead < 32 && st.sig >= 0)
                  sig_pre[j % (2 * kAhead)] = ld_stream(sig_g + (size_t)(j + 2 * kAhead) * 128);
                const float4* sp = sig_g + (size_t)j * 128;
                const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
                if ((st.flags & F_SKIP_GRAD) && c + 1 >= P.inj_col) {
                  // columns >= inj_col are d/d embed through the skip connection: park them, zero them in A
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float gval = u[e] * isc;
                    const int col = c + (e & 1);
                    if (col >= P.inj_col) {
                      ge[(size_t)(col - P.inj_col) * 128 + rowt[e >> 1]] = gval;
                      u[e] = 0.f;
                    } else {
                      u[e] = gval * sv[e];
                    }
                  }
                } else {
#pragma unroll
                  for (int e = 0; e < 4; ++e) u[e] *= isc * sv[e];
                }
                // this group's sigma' line is dead: drop it from L2
                if (st.sig >= 0 && (lane & 7) == 0) discard_line(sp, s4.x);
              } else {   // K_RELU
#pragma unroll
                for (int e = 0; e < 4; ++e) u[e] = fmaxf(fmaf(u[e], isc, b[e & 1]), 0.f);
                if constexpr (kRgb) {
#pragma unroll
                  for (int k = 0; k < 3; ++k) {
                    const float2 w2 = cs.rgb[jj][k];
                    dot[0][k] = fmaf(u[0], w2.x, fmaf(u[1], w2.y, dot[0][k]));
                    dot[1][k] = fmaf(u[2], w2.x, fmaf(u[3], w2.y, dot[1][k]));
                  }
                }
              }
            }
          }
#pragma unroll
          for (int wi = 0; wi < W; ++wi) {
            const int jp = jp0 + wi;
            if constexpr (KIND == K_SP_SAVE) {
#pragma unroll
              for (int jj = 0; jj < 2; ++jj)
                st_stream(&sig[(((size_t)st.sig * kConsumers + g) * 32 + 2 * jp + jj) * 128 + t],
                          make_float4(dsv[wi][jj][0], dsv[wi][jj][1], dsv[wi][jj][2], dsv[wi][jj][3]));
            }
            if constexpr (KIND == K_SP_SEED) {
              uint4 fh, fl;
              split8(yv[wi], fh, fl);
              st_stream(&fsc[(size_t)jp * 128 + t], fh);
              st_stream(&fsc[(size_t)(16 + jp) * 128 + t], fl);
            }
            // activations of these 16 columns -> A (fp16 hi/lo, swizzled) unless this is the last layer
            if constexpr (!kRgb) store_acc16(lane_base, lane_x, jp, acc + 8 * jp);
          }
        }
        // ---- step-specific tails: per-row dots reduced over the quad ----
        if (kW8 && (st.flags & F_SDF_DOT)) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float sdot = quad_sum(dot[h][0]);
            if (q == 0 && valid[h] && io.sdf) io.sdf[slot[h]] = __ldg(P.b8) + sdot;
          }
        }
        if constexpr (kRgb) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const float z = __ldg(P.brgb + k) + quad_sum(dot[h][k]);
              if (q == 0 && valid[h] && io.rgb) io.rgb[3 * (size_t)slot[h] + k] = 1.f / (1.f + __expf(-z));
            }
          }
        }
      };
      // Skip connection (F_INJECT_EMB, softplus kinds): columns >= inj_col of this warpgroup's rows of A receive the
      // input embedding, split into fp16 hi / lo element by element exactly as split2 splits an activation.  Done after
      // the column loop, over the injected columns only, so that the loop holds no test of the column against inj_col.
      // The barrier orders these stores after every lane's stmatrix stores of the same rows.  (The SDF dot of a step
      // reads the activations before injection; mp_field_pack fixes the skip at layer 4, so F_INJECT_EMB (layer 3) and
      // F_SDF_DOT (layer 7) never meet in one step.)
      auto inject_emb = [&]() {
        wg_sync(bar_id);
        const int row = 64 * g + (t >> 1);
        for (int col = P.inj_col + (t & 1); col < kHidden; col += 2) {
          const float v = emb[(size_t)(col - P.inj_col) * 128 + row];
          const __half h = __float2half_rn(v);
          const __half l = __float2half_rn(v - __half2float(h));
          const uint32_t o = a_off(row, col >> 6, (col >> 3) & 7) + 2u * (uint32_t)(col & 7);
          sts16(A32, o, h);
          sts16(A32, 65536u + o, l);
        }
      };
      // each kind's epilogue instantiated for every combination of the flags its column loop reads
      switch (st.kind) {
        case K_SP_PLAIN:
          with_flags<F_SDF_DOT>(st.flags, [&](auto fl) { run_epi(IntC<K_SP_PLAIN>{}, fl); });
          if (st.flags & F_INJECT_EMB) inject_emb();
          break;
        case K_SP_SAVE:
          with_flags<F_SDF_DOT>(st.flags, [&](auto fl) { run_epi(IntC<K_SP_SAVE>{}, fl); });
          if (st.flags & F_INJECT_EMB) inject_emb();
          break;
        case K_SP_SEED: run_epi(IntC<K_SP_SEED>{}, IntC<0>{}); break;
        case K_FEAT: run_epi(IntC<K_FEAT>{}, IntC<0>{}); break;
        case K_BWD: run_epi(IntC<K_BWD>{}, IntC<0>{}); break;
        default: with_flags<F_RGB_OUT>(st.flags, [&](auto fl) { run_epi(IntC<K_RELU>{}, fl); }); break;
      }
      // the skip gradient parked in `ge` is read by other lanes of the quad at the final-gradient step
      if (st.flags & F_SKIP_GRAD) __threadfence_block();
      rec.template step_done<PH_FULL, PH_EPI>(st.kind);
    }
  }
  rec.run_done();
}

// ---------------------------------------------------------------------------------------------
// packing
// ---------------------------------------------------------------------------------------------
// Where one packed layer's weights come from: the weight slots of its step hold
// B[n][k] = W[n_off + n][k] (transposed: W[k][n_off + n]) for n < n_valid, k < k_valid, zero elsewhere, scaled by the
// 2^s of max |W[0, total)|.
struct TcSrc {
  const float* W;
  int ld, transposed, n_off, n_valid, k_valid, total, perm16;
  TcStep step;     // as tc_programs packed it; tc_pack reads its slot layout (nk, slot_off) only
};

constexpr int kLdM = 320;     // row stride of the chains' folded colour layer 0 (see tc_pack)

struct TcBlob {
  TcProgram sdf_prog;     // L0..L7 + sdf dot
  TcProgram full_prog;    // forward + reverse + colour (Field::tc_full)
  TcProgram fwd_prog;     // L0..L8 (sdf + features), operator API
  // what tc_pack writes into the field's storage: the chains' folded colour layer 0, the programs' constants, and for
  // packed layer i (src[i]) its 2^-s at inv_scale[i] and its weight slots in blob
  float* Mfold;           // [256][kLdM]
  float* w8row;           // W8[0,:]
  float* Wrgb;            // [3][256] rgb head, zero padded
  float* b8feat;          // b8[1:], 16-byte aligned copy (the epilogue loads float4)
  float* inv_scale;
  uint8_t* blob;
  std::vector<TcSrc> src;
};

// inv_scale[0] = 2^-s of the weights W[0, n)
__global__ void absmax_kernel(const float* __restrict__ W, int n, float* __restrict__ inv_scale) {
  __shared__ float s[256];
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(W[i]));
  s[threadIdx.x] = m;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] = fmaxf(s[threadIdx.x], s[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    // scale = 2^s with max|W| * 2^s in (2^13, 2^14]  (fp16 hi/lo both stay in the normal range)
    float mx = s[0];
    int ex = 0;
    if (mx > 0.f) frexpf(mx, &ex);       // mx = f * 2^ex, f in [0.5,1)
    float sc = ldexpf(1.f, 14 - ex);
    inv_scale[0] = 1.f / sc;
  }
}

// One weight slot: B[n][k] for n < 256, k < 64 at K offset kc*64; value from W (natural [out][in], ld):
//   transposed == 0 : B[n][k] = W[(n_off + n) * ld + k_off + kc*64 + k]   (n < n_valid, kk < k_valid)
//   transposed == 1 : B[n][k] = W[(k_off + kc*64 + k) * ld + n_off + n]
__global__ void pack_slot_kernel(const float* __restrict__ W, int ld, int transposed, int n_off, int k_off,
                                 int n_valid, int k_valid, int kc, const float* __restrict__ inv_scale,
                                 uint8_t* __restrict__ dst_hi, uint8_t* __restrict__ dst_lo, int perm16) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 256 * 64) return;
  int n = idx >> 6, k = idx & 63;
  int kk = kc * 64 + k;
  // perm16 = d_in > 0 (final step of the reverse sweep): output column a * 16 + j (a < d_in) carries the embedding index
  // of axis a in the order [x_a, sin(2^0 x_a), cos(2^0 x_a), sin(2^1 x_a), ...] (embedders.py:8-34), i.e.
  // j = 0 -> a ; j = 1 + 2 f + t -> d + 2 f d + t d + a ; every other column is padding.  Column part a of the epilogue
  // owns columns [16 a, 16 a + 16) of K-block 0, so it holds every term of d sdf / d x_a.
  int ns = n;
  if (perm16) {
    const int dd = perm16, a = n >> 4, j = n & 15;
    ns = n_valid;
    if (n < 64 && a < dd) {
      const int k = (j == 0) ? a : dd + ((j - 1) >> 1) * 2 * dd + ((j - 1) & 1) * dd + a;
      if (k < n_valid) ns = k;
    }
  }
  float w = 0.f;
  if (ns < n_valid && kk < k_valid)
    w = transposed ? W[(size_t)(k_off + kk) * ld + n_off + ns] : W[(size_t)(n_off + ns) * ld + k_off + kk];
  w = __fdiv_rn(w, inv_scale[0]);     // = w * 2^s exactly rounded, as inv_scale is a power of two
  __half h = __float2half_rn(w);
  __half l = __float2half_rn(w - __half2float(h));
  uint32_t off = (uint32_t)(n * 128 + ((((k >> 3) ^ (n & 7))) << 4) + (k & 7) * 2);
  *(__half*)(dst_hi + off) = h;
  *(__half*)(dst_lo + off) = l;
}

// M[n][k] = sum_j Wc[n][coff + j] * W8f[j][k]   (n < n_rows, k < 256; W8f = W8[1:], row stride ld8; M row stride ldm)
// cb[n]   = sum_j Wc[n][coff + j] * b8f[j]
__global__ void fold_mm_kernel(const float* __restrict__ Wc, int ldc, int coff, const float* __restrict__ W8f, int ld8,
                               const float* __restrict__ b8f, int n_rows, float* __restrict__ M, int ldm,
                               float* __restrict__ cb) {
  int k = blockIdx.x * 16 + threadIdx.x, n = blockIdx.y * 16 + threadIdx.y;
  if (n >= n_rows || k >= 256) return;
  const float* w = Wc + (size_t)n * ldc + coff;
  double acc = 0.0;
  for (int j = 0; j < 256; ++j) acc += (double)w[j] * (double)W8f[(size_t)j * ld8 + k];
  M[(size_t)n * ldm + k] = (float)acc;
  if (k == 0) {
    double a2 = 0.0;
    for (int j = 0; j < 256; ++j) a2 += (double)w[j] * (double)b8f[j];
    cb[n] = (float)a2;
  }
}

// columns 256 .. 319 of the combined colour layer 0: M[n][256 + e] = Wc0[n][e] for the extra inputs e < n_extra
// (Wt = Wc0 transposed, [in][n_out]), zero elsewhere
__global__ void fill_extra_cols_kernel(const float* __restrict__ Wt, int n_out, int n_extra, float* __restrict__ M, int ldm) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 256 * 64) return;
  int n = i >> 6, e = i & 63;
  M[(size_t)n * ldm + 256 + e] = (n < n_out && e < n_extra) ? Wt[(size_t)e * n_out + n] : 0.f;
}

TcBlob* tc_new() { return new TcBlob(); }
void tc_free(TcBlob* tb) { delete tb; }

// The three programs, one layer() per packed step (kind, flags, sigma' layer, bias, then the weight source).  L0..L7 are
// packed once and shared: the sdf-only, forward and background programs run them as plain softplus steps, the fused
// foreground program saves sigma' and seeds the reverse sweep.  Slots are assigned in packing order and the number
// assigned is returned; on a sizing layout (null pointers) that is all this is for.
static int tc_programs(const Field& f, TcBlob& tb) {
  int nslots = 0;
  auto layer = [&](TcStep& stp, int kind, int flags, int sig, const float* bias, const float* W, int ld, int transposed,
                   int n_off, int n_valid, int k_valid, int nk, int total, int perm16 = 0) {
    stp = TcStep{nk, kind, flags, sig, bias, nslots, (int)tb.src.size(), 3};
    tb.src.push_back(TcSrc{W, ld, transposed, n_off, n_valid, k_valid, total, perm16, stp});
    nslots += tc_packed_slots(nk);
  };
  const int E = f.emb_dim;
  TcProgram P{};
  P.d_in = f.d_in;
  P.multires = f.multires;
  P.E = E;
  P.inj_col = kHidden - E;
  P.w8row = tb.w8row;
  P.b8 = f.imp_b[8];
  P.Wrgb = tb.Wrgb;
  P.n_extra = f.ren_extra;
  int s = 0;
  // ---- forward L0..L7: the sdf-only program ----
  for (int l = 0; l < 8; ++l) {
    const int in = f.imp_in[l], out = f.imp_out[l];
    const int flags = ((l == f.skip_layer - 1) ? F_INJECT_EMB : 0) | ((l == 7) ? F_SDF_DOT : 0);
    layer(P.step[s++], K_SP_PLAIN, flags, l, (l == 0) ? f.imp_b0_eff : f.imp_b[l], f.imp_W[l], in, 0, 0, out,
          (l == 0) ? E : in, (l == 0) ? (E + 63) / 64 : 4, out * in);
  }
  P.nsteps = s;
  tb.sdf_prog = P;
  // ---- L8 features (operator API: sdf + features) ----
  tb.fwd_prog = P;
  layer(tb.fwd_prog.step[s], K_FEAT, 0, -1, tb.b8feat, f.imp_W[8], 256, 0, 1, 256, 256, 4, 257 * 256);
  tb.fwd_prog.nsteps = s + 1;
  if (f.tc_full && f.ren_mode == 1) {
    // background: folded colour layer 0 (view embedding + h7 -> 128, ReLU) and the rgb head (multiply.py:531)
    layer(P.step[s++], K_RELU, F_EXTRA_IN | F_RGB_OUT, -1, f.ren_b0_fold, tb.Mfold, kLdM, 0, 0, f.ren_out[0], kLdM, 5,
          256 * kLdM);
    P.brgb = f.ren_b[1];
    P.nsteps = s;
    tb.full_prog = P;
  }
  if (f.tc_full && f.ren_mode == 0) {
    // L0..L7 save sigma' for the reverse sweep, which starts right after L7; h7 is parked (it returns as the folded
    // colour layer's input)
    for (int l = 0; l < 8; ++l) P.step[l].kind = (l == 7) ? K_SP_SEED : K_SP_SAVE;
    // ---- reverse sweep B7..B1: g_{l-1} = (g_l * sigma'_l) . W_l ----
    for (int l = 7; l >= 1; --l) {
      const int in = f.imp_in[l], out = f.imp_out[l];
      // B[n][k] = W_l[k][n] : n over in (valid in), k over out (valid out)
      layer(P.step[s++], K_BWD, (l == f.skip_layer) ? F_SKIP_GRAD : 0, l - 1, nullptr, f.imp_W[l], in, 1, 0, in, out, 4,
            out * in);
    }
    // ---- B0: d/d embed = (g_0 * sigma'_0) . W0[:, :E] ----
    layer(P.step[s++], K_FINAL_GRAD, 0, -1, nullptr, f.imp_W[0], f.imp_in[0], 1, 0, E, 256, 4, 256 * f.imp_in[0],
          /*perm16=*/f.d_in);
    // ---- colour net: folded layer 0, then layers 1..3 ----
    layer(P.step[s++], K_RELU, F_EXTRA_IN, -1, f.ren_b0_fold, tb.Mfold, kLdM, 0, 0, 256, kLdM, 5, 256 * kLdM);
    for (int l = 1; l < 4; ++l)
      layer(P.step[s++], K_RELU, (l == 3) ? F_RGB_OUT : 0, -1, f.ren_b[l], f.ren_W[l], 256, 0, 0, 256, 256, 4,
            256 * 256);
    P.brgb = f.ren_b[4];
    P.nsteps = s;
    tb.full_prog = P;
  }
  return nslots;
}

// The tensor-core share of a field's storage, taken at the end of its carve: the chains' folded colour layer 0 and its
// biases, the programs' constants, then one 2^-s per packed layer and the weight slots, as many as the programs assign.
// Lays out f.tc, or on a sizing Arena (f.tc null) a blob that is thrown away.
void tc_pack_carve(Arena& a, Field& f) {
  TcBlob sizing{};
  TcBlob& tb = f.tc ? *f.tc : sizing;
  tb.Mfold = a.take<float>(256 * kLdM);
  f.ren_cb = a.take<float>(264);
  f.ren_b0_fold = a.take<float>(264);
  tb.w8row = a.take<float>(256);
  tb.Wrgb = a.take<float>(3 * 256);
  tb.b8feat = a.take<float>(256);
  const int nslots = tc_programs(f, tb);
  tb.inv_scale = a.take<float>(tb.src.size());
  tb.blob = a.take<uint8_t>((size_t)nslots * kSlotBytes);
  for (TcProgram* P : {&tb.sdf_prog, &tb.fwd_prog, &tb.full_prog}) {
    P->inv_scale = tb.inv_scale;
    P->blob = (const uint4*)tb.blob;
  }
}

// Fills what tc_pack_carve laid out in the zeroed storage, from the fp32 layers mp_field_pack has folded: the programs'
// constants, the chains' folded colour layer 0, then every packed layer's 2^-s and weight slots.
int tc_pack(const Field& f, cudaStream_t st) {
  const TcBlob& tb = *f.tc;
  MP_CHECK_CUDA(cudaMemcpyAsync(tb.w8row, f.imp_W[8], 256 * sizeof(float), cudaMemcpyDeviceToDevice, st));  // W8[0,:]
  MP_CHECK_CUDA(cudaMemcpyAsync(tb.b8feat, f.imp_b[8] + 1, 256 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (f.tc_full) {
    // The feature layer L8 and the colour layer 0 have no non-linearity in between (networks.py:199-207 -> :281,:305):
    //   C0_pre = Wc0[:, feat] (W8[1:] h7 + b8[1:]) + Wc0[:, extra] extra + b0  =  M h7 + (Wc0f b8f + b0) + ...
    // so the fused chains run ONE layer with M = Wc0[:, feat] . W8[1:, :] instead of two: [ M | extra-input columns | 0 ]
    // (256 x 320, K-blocks 0..3 | 4).  The feature block is colour layer 0's last 256 inputs.
    const int in0 = f.ren_in[0], o0 = f.ren_out[0];
    fold_mm_kernel<<<dim3(256 / 16, div_up(o0, 16)), dim3(16, 16), 0, st>>>(f.ren_W[0], in0, in0 - kHidden,
                                                                          f.imp_W[8] + 256, 256, f.imp_b[8] + 1, o0,
                                                                          tb.Mfold, kLdM, f.ren_cb);
    MP_LAUNCH_CHECK();
    fill_extra_cols_kernel<<<64, 256, 0, st>>>(f.ren_Wt[0], o0, f.ren_extra, tb.Mfold, kLdM);
    MP_LAUNCH_CHECK();
    // the rgb head [3][256]: the last colour layer, whose inputs are the background's 128 (o0) wide
    const size_t w = (f.ren_mode == 0 ? kHidden : o0) * sizeof(float);
    MP_CHECK_CUDA(cudaMemcpy2DAsync(tb.Wrgb, 256 * sizeof(float), f.ren_W[f.n_ren - 1], w, w, 3,
                                    cudaMemcpyDeviceToDevice, st));
  }
  for (size_t i = 0; i < tb.src.size(); ++i) {
    const TcSrc& c = tb.src[i];
    absmax_kernel<<<1, 256, 0, st>>>(c.W, c.total, tb.inv_scale + i);
    MP_LAUNCH_CHECK();
    for (int kc = 0; kc < c.step.nk; ++kc) {
      pack_slot_kernel<<<64, 256, 0, st>>>(c.W, c.ld, c.transposed, c.n_off, 0, c.n_valid, c.k_valid, kc,
                                           tb.inv_scale + i,
                                           tb.blob + (size_t)tc_chunk_slot(c.step, kc, false) * kSlotBytes,
                                           tb.blob + (size_t)tc_chunk_slot(c.step, kc, true) * kSlotBytes, c.perm16);
      MP_LAUNCH_CHECK();
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
// One scratch slice per persistent CTA; a launch runs at most one CTA per SM and per 128-point tile.
static int tc_max_grid(int cap) { return max(0, min(sm_count(), div_up(cap, 128))); }
// the stall-accounting build's counters (mp_profile_enable(2)) follow the scratch, one record per warp of each CTA
constexpr size_t kStallWordsPerCta = (size_t)kStallWarps * MP_STALL_WORDS;
static std::atomic<bool> g_prof_stalls{false};
static void tc_carve(Arena& a, int grid, bool stalls, TcIO& io) {
  io.scratch = a.take<char>((size_t)grid * kScratchPerCta);
  io.stalls = stalls ? a.take<unsigned long long>((size_t)grid * kStallWordsPerCta) : nullptr;
}

size_t tc_workspace_bytes(int N) {
  Arena a;
  TcIO io{};
  tc_carve(a, tc_max_grid(N), g_prof_stalls.load(), io);
  return a.off;
}

// total[w] += sum over the grid's CTAs of rec[cta][w]
__global__ void stall_sum_kernel(const unsigned long long* __restrict__ rec, int grid, unsigned long long* total) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (int)kStallWordsPerCta) return;
  unsigned long long v = 0;
  for (int c = 0; c < grid; ++c) v += rec[(size_t)c * kStallWordsPerCta + w];
  atomicAdd(total + w, v);
}

// optional per-launch timing of the tensor-core kernel (bench.py roofline): CUDA events on the
// launching stream + an async copy of the device-side point count into pinned memory
struct ProfEntry {
  cudaEvent_t e0, e1;
  int kind;        // MlpProg: 0 sdf-only, 1 forward (sdf+features), 2 full shade, 3 background
  int cap;
  int* host_count; // pinned
};
// The profile is a process-wide diagnostic (bench.py): its state is guarded by g_prof_mu so that concurrent
// launches from several host threads stay well defined.
static std::mutex g_prof_mu;
static std::atomic<bool> g_prof_on{false};
static std::vector<ProfEntry>* g_prof = nullptr;
static int* g_prof_pinned = nullptr;
static int g_prof_used = 0;
constexpr int kProfMax = 1 << 16;
static unsigned long long* g_stall_total = nullptr;     // device [4 program kinds][kStallWordsPerCta]
constexpr size_t kStallTotalBytes = 4 * kStallWordsPerCta * sizeof(unsigned long long);

int prof_enable(int on) {
  MP_REQUIRE(on >= 0 && on <= 2, "mp_profile_enable: 0 (off), 1 (launch times) or 2 (launch times and stall clocks)");
  std::lock_guard<std::mutex> g(g_prof_mu);
  if (on && !g_prof) {
    g_prof = new std::vector<ProfEntry>();
    MP_CHECK_CUDA(cudaMallocHost(&g_prof_pinned, kProfMax * sizeof(int)));
  }
  if (on == 2 && !g_stall_total) {
    MP_CHECK_CUDA(cudaMalloc(&g_stall_total, kStallTotalBytes));
    MP_CHECK_CUDA(cudaMemset(g_stall_total, 0, kStallTotalBytes));
  }
  g_prof_stalls = on == 2;
  g_prof_on = on != 0;
  return 0;
}
int prof_read_stalls(unsigned long long* clocks, int reset) {
  std::lock_guard<std::mutex> g(g_prof_mu);
  if (!g_stall_total) {
    memset(clocks, 0, kStallTotalBytes);
    return 0;
  }
  MP_CHECK_CUDA(cudaDeviceSynchronize());
  MP_CHECK_CUDA(cudaMemcpy(clocks, g_stall_total, kStallTotalBytes, cudaMemcpyDeviceToHost));
  if (reset) MP_CHECK_CUDA(cudaMemset(g_stall_total, 0, kStallTotalBytes));
  return 0;
}
int prof_read(double* ms, long long* launches, double* points, int reset) {
  for (int k = 0; k < 4; ++k) {
    ms[k] = 0;
    launches[k] = 0;
    points[k] = 0;
  }
  std::lock_guard<std::mutex> g(g_prof_mu);
  if (!g_prof) return 0;
  for (auto& e : *g_prof) {
    MP_CHECK_CUDA(cudaEventSynchronize(e.e1));
    float t = 0.f;
    MP_CHECK_CUDA(cudaEventElapsedTime(&t, e.e0, e.e1));
    ms[e.kind] += t;
    launches[e.kind] += 1;
    int n = e.host_count ? *e.host_count : e.cap;
    points[e.kind] += (double)(n < e.cap ? n : e.cap);
  }
  if (reset) {
    for (auto& e : *g_prof) {
      cudaEventDestroy(e.e0);
      cudaEventDestroy(e.e1);
    }
    g_prof->clear();
    g_prof_used = 0;
  }
  return 0;
}

// Precision mode of the tensor-core engine (mp_set_precision): which of the three split-precision product terms each layer
// step issues.  The weight blob always holds the hi and lo slots; a single-term step just skips the lo slots.
//   0  parity (default): every step A_hi.W_hi + A_lo.W_hi + A_hi.W_lo  -- RGB / SDF within 1e-4 of the fp32 reference
//   1  colour layers single-term (A_hi.W_hi): SDF / normals unchanged, RGB error ~2e-5 (still inside the gate)
//   2  throughput: every step single-term, i.e. plain fp16 operands with fp32 accumulation -- misses the 1e-4 gate
//      (SDF ~3e-4, normals ~1e-3; measured values in DESIGN.md) and is reported separately by bench.py
std::atomic<int> g_precision{0};

// The tensor core adds each MMA's products into the fp32 accumulator with round-toward-zero: every one of the
// n = 4 nk terms accumulations of a layer step (K = 16 per wgmma) drops on average half an ulp of the running sum,
// always toward zero.  Unlike round-to-nearest noise this loss is coherent -- every pre-activation shrinks by the same
// relative amount, layer after layer -- and uncompensated it dominates the error of the rendered normals where
// |grad sdf| is small.  First-order model: a running sum that grows linearly to its final value z loses
// sum_i ulp(z i/n)/2 ~= (n/2) * E[ulp(z)/|z|]/2 * |z|, with E[ulp/|z|] = 2^-23 / (2 ln 2) for a log-uniform mantissa:
// 2.15e-8 |z| per accumulation, 1.03e-6 |z| for the 48 accumulations of a 256-wide three-term layer.  The epilogue
// multiplies the accumulator by (1 + n * kRzPerMma), which is free (it is folded into the 2^-s rescale).  The constant
// is 0.8 times the model's 2.15e-8; MP_TC_RZ_SCALE multiplies it (0 switches it off) and scripts/gpu_normal_diag.py
// measures the per-sample SDF / gradient / normal error against the fp64 evaluation of the same weights.
constexpr float kRzPerMma = 1.72e-8f;

static int tc_launch(const TcProgram& P0, TcIO io, void* ws, size_t ws_bytes, cudaStream_t st, MlpProg kind) {
  TcProgram P = P0;
  {
    const int mode = g_precision.load();
    for (int s = 0; s < P.nsteps; ++s)
      P.step[s].terms = (mode == 2 || (mode == 1 && P.step[s].kind == K_RELU)) ? 1 : 3;
  }
  int grid = tc_max_grid(io.cap);
  static const int grid_override = [] {
    const char* eg = getenv("MP_TC_GRID");     // experiment knob: number of persistent CTAs
    return eg ? atoi(eg) : 0;
  }();
  if (grid_override > 0 && grid_override < grid) grid = grid_override;
  if (grid < 1) return 0;
  Arena a(ws, ws_bytes);
  tc_carve(a, grid, g_prof_stalls.load(), io);
  MP_TRY(a.fits("tensor-core engine"));
  io.scratch_per_cta = kScratchPerCta;
  if (io.stalls) {
    MP_REQUIRE(g_stall_total, "tensor-core engine: stall accounting is not enabled");
    MP_CHECK_CUDA(cudaMemsetAsync(io.stalls, 0, (size_t)grid * kStallWordsPerCta * sizeof(unsigned long long), st));
  }
  static const float rz_scale = [] {
    const char* er = getenv("MP_TC_RZ_SCALE");      // experiment knob: multiplies kRzPerMma (0 switches it off)
    return er ? (float)atof(er) : 1.f;
  }();
  io.rz = kRzPerMma * rz_scale;
  {
    // the > 48 KB dynamic shared memory opt-in is per device
    static std::mutex attr_mu;
    static unsigned long long attr_done = 0;      // bit d: cudaFuncSetAttribute done on device d
    int dev = 0;
    MP_CHECK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> g(attr_mu);
    if (dev < 0 || dev >= 64 || !((attr_done >> dev) & 1ull)) {
      MP_CHECK_CUDA(cudaFuncSetAttribute(tc_chain_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
      MP_CHECK_CUDA(cudaFuncSetAttribute(tc_chain_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
      if (dev >= 0 && dev < 64) attr_done |= 1ull << dev;
    }
  }
  ProfEntry pe;
  std::unique_lock<std::mutex> prof_lock(g_prof_mu, std::defer_lock);
  if (g_prof_on.load()) prof_lock.lock();
  const bool prof = prof_lock.owns_lock() && g_prof_on.load() && g_prof && g_prof_used < kProfMax;
  if (prof) {
    MP_CHECK_CUDA(cudaEventCreate(&pe.e0));
    MP_CHECK_CUDA(cudaEventCreate(&pe.e1));
    pe.kind = (int)kind;
    pe.cap = io.cap;
    pe.host_count = nullptr;
    if (io.count) {
      pe.host_count = g_prof_pinned + g_prof_used++;
      MP_CHECK_CUDA(cudaMemcpyAsync(pe.host_count, io.count, sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    MP_CHECK_CUDA(cudaEventRecord(pe.e0, st));
  }
  if (io.stalls) {
    tc_chain_kernel<true><<<grid, kThreads, kSmemBytes, st>>>(P, io);
  } else {
    tc_chain_kernel<false><<<grid, kThreads, kSmemBytes, st>>>(P, io);
  }
  MP_LAUNCH_CHECK();
  if (prof) {
    MP_CHECK_CUDA(cudaEventRecord(pe.e1, st));
    g_prof->push_back(pe);
  }
  if (io.stalls) {
    stall_sum_kernel<<<div_up((int)kStallWordsPerCta, 128), 128, 0, st>>>(io.stalls, grid,
                                                                          g_stall_total + (int)kind * kStallWordsPerCta);
    MP_LAUNCH_CHECK();
  }
  return 0;
}

int tc_run(const Field& f, const MlpCall& c, void* ws, size_t ws_bytes, cudaStream_t st) {
  MP_REQUIRE(f.tc, "tensor-core engine: field not packed");
  const TcBlob& tb = *f.tc;
  const MlpProg prog = mlp_prog(c);
  TcIO io{};
  static_cast<MlpCall&>(io) = c;
  if (prog == MlpProg::kSdf) return tc_launch(tb.sdf_prog, io, ws, ws_bytes, st, prog);
  if (prog == MlpProg::kForward) return tc_launch(tb.fwd_prog, io, ws, ws_bytes, st, prog);
  if (prog == MlpProg::kBg) {
    MP_REQUIRE(f.tc_full && f.ren_mode == 1, "tensor-core engine: not a background field");
    return tc_launch(tb.full_prog, io, ws, ws_bytes, st, prog);
  }
  MP_REQUIRE(f.tc_full, "tensor-core engine: this field has no fused shading program");
  if (c.feat) {
    // the fused program folds L8's feature rows into the colour layer and never materialises the features: the
    // forward program writes them (operator API only; the render passes no feature output)
    TcIO fio{};
    fio.x = c.x;
    fio.slot = c.slot;
    fio.count = c.count;
    fio.cap = c.cap;
    fio.feat = c.feat;
    MP_TRY(tc_launch(tb.fwd_prog, fio, ws, ws_bytes, st, MlpProg::kForward));
    io.feat = nullptr;
  }
  return tc_launch(tb.full_prog, io, ws, ws_bytes, st, prog);
}

}  // namespace mp
