// Hand-written Hopper GEMM / implicit-GEMM convolution:  C[M,N] = alpha * op(A) · op(B)  (+bias, +ReLU), bf16 or tf32 in, fp32 accumulate.
//
//   * persistent: one CTA per SM walks the tile list; 384 threads = warpgroup 0 producer (one warp issues TMA, the register
//     budget of the group is handed to the consumers with setmaxnreg), warpgroups 1 and 2 consumers: consumer c owns rows
//     [64c, 64c + 64) of every 128-row sub-tile and keeps its accumulators in registers;
//   * operands staged global→shared by TMA (tiled 2-D / 3-D boxes or im2col-mode 4-D boxes, 128 B swizzle) into a 3–8 stage
//     mbarrier ring; wgmma.mma_async m64nNk16 (bf16) / m64nNk8 (tf32) straight from the ring; a consumer hands a slot back
//     once its wgmma group has retired;
//   * MT = 2: a CTA computes a 256-row tile as two wgmmas per k-step against ONE B tile (half the B reads per flop);
//   * epilogue (consumer warps, after the k loop): accumulator fragments → bias / ReLU → per-warp smem staging of a
//     16-row x 32-column chunk → coalesced 16 B row-segment stores, or red.global.add.v4.f32 for split-K;
//   * two same-shape problems (the two groups of a grouped convolution) can share one launch.
//
// Both operands may be K-major ([rows, K], K contiguous) or MN-major ([K, rows], rows contiguous): forward, dgrad and wgrad of
// FC and conv layers all run on this one kernel without transposed copies in global memory (reference: cuBLAS SGEMM / cuDNN
// through Theano, layers2.py:927-929, :380-388, GpuCorrMM :597-653).  bf16 wgmma reads MN-major tiles directly (transpose
// bits); tf32 wgmma accepts K-major tiles only, so the consumers transpose an MN-major tf32 tile shared→shared first.
#pragma once
#include "common.cuh"
#include "api.h"
#include <cuda.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>

namespace tmpi {

namespace wgmma {

constexpr int BM = 128;
constexpr int NUM_THREADS = 384;       // warpgroup 0 TMA producer, warpgroups 1..2 wgmma consumers + epilogue
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

// Operand element type: __nv_bfloat16 (wgmma bf16) or float (wgmma tf32: fp32 storage, the tensor core reads the top 19 bits).
// A k-block is always ONE 128-byte swizzle row per operand row, so the byte geometry of the smem ring, the descriptors' K-major
// stepping (32 B per wgmma) and the TMA box widths in bytes are identical for both types; what changes is the number of
// ELEMENTS per k-block / wgmma / MN-major atom.
// Kernel operand tag: the element type itself, or SgdEpilogue<element type> for the momentum-SGD epilogue (see gemm_wgmma)
template <typename T> struct SgdEpilogue {};
template <typename OP> struct Operand { using Type = OP; static constexpr bool kSgd = false; };
template <typename T> struct Operand<SgdEpilogue<T>> { using Type = T; static constexpr bool kSgd = true; };

template <typename T> struct Elem {
  static constexpr int ESZ = (int)sizeof(T);
  static constexpr int BK = 128 / ESZ;            // elements per k-block: 64 (bf16) / 32 (tf32)
  static constexpr int MMA_K = 32 / ESZ;          // K of one wgmma: 16 / 8
  static constexpr int ATOM = 128 / ESZ;          // MN-major: elements of one 128-byte atom row (TMA box width): 64 / 32
  static constexpr bool TF32 = ESZ == 4;
};

// MT = number of 128-row sub-tiles a CTA computes per k-block against ONE copy of the B tile.
template <typename T, int BN, int MT> struct Cfg {
  static constexpr int A_BYTES = MT * BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // epilogue staging: each consumer warp moves one 16-row x 32-column chunk at a time through its own region
  // (row pitch = chunk bytes + 16 B: conflict-free 16 B accesses)
  static constexpr int STAGING_ROW = 32 * 4 + 16;
  static constexpr int STAGING_BYTES = NUM_CONSUMER_WARPS * 16 * STAGING_ROW;
  // tf32 MN-major operands: per consumer warpgroup, a K-major copy of its 64 A rows and of the whole B tile (MT = 1 only)
  static constexpr bool XPOSE = Elem<T>::TF32 && MT == 1;
  static constexpr int XA_BYTES = 64 * 128;
  static constexpr int XPOSE_BYTES = XPOSE ? 2 * (XA_BYTES + B_BYTES) : 0;
  static constexpr int SMEM_LIMIT = 232448;                                // 227 KB per CTA
  static constexpr int RING_BUDGET = SMEM_LIMIT - STAGING_BYTES - XPOSE_BYTES - 1024 /*align slack*/ - 256 /*barriers*/;
  static constexpr int STAGES = (RING_BUDGET / STAGE_BYTES) > 8 ? 8 : (RING_BUDGET / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + XPOSE_BYTES + STAGING_BYTES + 1024 + 256;
  static_assert(STAGES >= 3, "operand ring too shallow");
};

struct Params {
  void* C;
  const float* bias;
  float alpha;
  int M, N, K;
  long long ldc;
  int a_mn, b_mn;       // 1 = operand is MN-major in global memory
  int out_bf16;         // 1 = bf16 output, 0 = fp32
  int bias_mode;        // 0 none, 1 per-column (N), 2 per-row (M)
  int relu;
  int kb_per_split;     // k-blocks per split-K slice
  int mt, nt, splits;   // tile grid (the kernel is persistent: tiles are walked round-robin by the CTAs)
  int num_kb;           // total k-blocks (GEMM: ceil(K/BK); conv: taps*chunks or pixel blocks)
  // implicit-GEMM convolution (operands gathered by TMA im2col loads, no col matrix in memory):
  //   conv_mode 1  fprop / dgrad : A = activation im2col tile [128 pixels x BK ch] per (tap, chunk); B = weights [O][tap][C] 3-D tiled
  //   conv_mode 2  wgrad         : A = dy (MN-major tiled);  B = activation im2col boxes [BK pixels x ATOM ch]; n-tiles = (tap, channel chunk)
  int conv_mode;
  int cHo, cWo, cS, cP, cKH, cKW, cCg, c_chunks;
  int atomic_out;       // 1 = fp32 atomicAdd (split-K)
  // second problem of the same shape run by the same launch (the two groups of an AlexNet-style grouped convolution): tiles
  // [0, per_group) belong to group 0 (maps a/b, C, bias), tiles [per_group, 2*per_group) to group 1 (maps a1/b1, C1, bias1)
  void* C1;
  const float* bias1;
  int groups;           // 1 or 2
  int group_m;          // tile raster: m-tiles per band (0 = plain m-fastest order); see tile_mn()
  int dbg;              // bottleneck probe (scripts/gemm_probe.py): 1 = skip A loads, 2 = skip B loads, 4 = skip the MMAs
  // reduce-scatter fused into the epilogue (fp32 wgrad outputs living in the symmetric gradient arena): element e of the G
  // region is owned by rank ((e >> 10) - rs_blo) / rs_per; every row segment of dW is added into the OWNER's G over NVLink
  // (rs_g[q] = rank q's G region as mapped here) by the bulk copy engine instead of being stored locally.  rs_world == 0: off.
  int rs_world = 0, rs_rank = 0;
  unsigned rs_blo = 0, rs_per = 1;
  long long rs_e0 = 0;  // element index of C[0, 0] inside the G region
  float* rs_g[kMaxRanks] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // momentum-SGD epilogue (gemm_wgmma<SgdEpilogue<T>, ...> only): C is not written; the accumulator at (m, n) is the gradient of weight element
  // m * ldw + n, updated in place together with its momentum and bf16 shadow, exactly as sgd_flat would update it
  struct Sgd {
    float* W = nullptr;
    float* U = nullptr;
    __nv_bfloat16* H = nullptr;   // nullptr: no shadow
    const float* lr_ptr = nullptr;
    float lr_mult = 1.f, wd = 0.f, mu = 0.f, inv_k = 1.f;
    int nesterov = 0;
    long long ldw = 0;
  } sgd;
};

// owner-rank address of element e of the gradient region (no dynamic indexing of the kernel-parameter array)
__device__ __forceinline__ float* rs_addr(const Params& p, long long e, bool& local) {
  unsigned owner = ((unsigned)(e >> 10) - p.rs_blo) / p.rs_per;
  if (owner >= (unsigned)p.rs_world) owner = (unsigned)p.rs_world - 1u;
  float* base = p.rs_g[0];
#pragma unroll
  for (int q = 1; q < kMaxRanks; ++q) if (owner == (unsigned)q) base = p.rs_g[q];
  local = owner == (unsigned)p.rs_rank;
  return base + e;
}
__device__ __forceinline__ void red_add_sys_f32(float* addr, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded wait: a protocol bug traps (launch failure) instead of hanging the GPU.  The spin loop lives INSIDE the asm
// statement so the compiler sees straight-line code: a C++ loop around try_wait has a per-thread exit condition, which
// makes everything after it "potentially divergent" and pushes the producer loop indices out of the uniform registers.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1, P2;\n\t"
      ".reg .u32 cnt;\n\t"
      "mov.u32 cnt, 0;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "add.u32 cnt, cnt, 1;\n\t"
      "setp.lt.u32 P2, cnt, 0x10000000;\n\t"
      "@P2 bra LAB_WAIT;\n\t"
      "trap;\n\t"
      "DONE:\n\t"
      "}"
      ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over the 128 threads of consumer warpgroup cw (ids 1 and 2; id 0 is __syncthreads).  The id is an immediate so
// the kernel reserves only those two barriers.
template <int ID> __device__ __forceinline__ void bar_sync_128() { asm volatile("bar.sync %0, 128;" ::"n"(ID) : "memory"); }
__device__ __forceinline__ void wg_bar(int cw) { if (cw == 0) bar_sync_128<1>(); else bar_sync_128<2>(); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// im2col-mode TMA on an NHWC tensor (dims C,W,H,N): coordinates are the input position of the window's top-left corner
// (w = q*stride - pad, h = p*stride - pad) of the FIRST pixel of the tile; the filter tap goes in the 16-bit offsets.
// The unit then walks pixelsPerColumn output positions (W, then H, then N) and zero-fills padding / out-of-range pixels.
// (Semantics checked with csrc/probe_im2col.cu.)
__device__ __forceinline__ void tma_load_im2col(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c, int w, int h, int n,
                                                int off_w, int off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"((uint16_t)off_w), "h"((uint16_t)off_h) : "memory");
}
// Bulk (TMA engine) epilogue ops: one contiguous row segment of fp32 in shared memory added into global (or peer-mapped)
// memory as ONE packet per call instead of 16-byte vector atomics.
__device__ __forceinline__ void bulk_reduce_add_f32(void* gdst, uint32_t ssrc, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// one lane of a fully converged warp (elect.sync): the issuing thread of the TMA warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N> __device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma.mma_async with both operands in shared memory; D (64 x N fp32) in registers.  TA / TB = 1: that operand is MN-major
// (bf16 only — the transpose bits do not exist for tf32).
template <int N, int TA, int TB> struct WgBF16 {};
template <int N> struct WgTF32 {};

template <int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d, WgBF16<32, TA, TB>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d, WgBF16<64, TA, TB>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d, WgBF16<128, TA, TB>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d, WgTF32<32>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d, WgTF32<64>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d, WgTF32<128>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(scale_d));
}

// n96 / n192: the tile widths the convolution planner picks for 96- and 192-channel outputs (see choose_conv_tile)
template <int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d, WgBF16<96, TA, TB>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, %52;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[96], uint64_t da, uint64_t db, uint32_t scale_d, WgBF16<192, TA, TB>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, %99, %100;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
               : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d, WgTF32<96>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma(float (&d)[96], uint64_t da, uint64_t db, uint32_t scale_d, WgTF32<192>) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
               : "l"(da), "l"(db), "r"(scale_d));
}

// Hopper shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor bit layout): start address, leading / stride byte
// offsets in 16-byte units, layout type 1 = SWIZZLE_128B.
//   K-major:  8-row groups 1024 B apart (SBO); LBO unused (a wgmma's K extent stays inside one 128 B swizzle row).
//   MN-major: 8-k-row groups 1024 B apart (SBO), ATOM-element MN atoms BK * 128 B apart (LBO).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);            // start address      bits [0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;       // leading byte off   bits [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;       // stride byte off    bits [32,46)
  d |= (uint64_t)1 << 62;                                 // SWIZZLE_128B       bits [62,64)
  return d;
}

// One k-block of wgmmas for a consumer warpgroup, issued as one group and retired before returning: STEPS k-steps x the first
// LIVE of the MT sub-tiles, all against the same B descriptor.  a_step / b_step: descriptor advance per step (K-major: 32 B;
// MN-major: MMA_K k-rows of 128 B).
template <typename T, int BN, int MT, int TA, int TB, int STEPS, int LIVE>
__device__ __forceinline__ void mma_kblock(float (&acc)[MT][BN / 2], uint64_t da, uint64_t db, uint32_t a_step, uint32_t b_step) {
  constexpr uint64_t SUB = (uint64_t)(BM * 128) >> 4;
#pragma unroll
  for (int u = 0; u < MT; ++u) acc_fence(acc[u]);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < STEPS; ++k) {
#pragma unroll
    for (int u = 0; u < LIVE; ++u) {
      if constexpr (Elem<T>::TF32) wgmma(acc[u], da + u * SUB + a_step * k, db + b_step * k, 1u, WgTF32<BN>{});
      else wgmma(acc[u], da + u * SUB + a_step * k, db + b_step * k, 1u, WgBF16<BN, TA, TB>{});
    }
  }
  wgmma_commit();
  wgmma_wait0();
#pragma unroll
  for (int u = 0; u < MT; ++u) acc_fence(acc[u]);
}

// The k-block with warpgroup-uniform trims: `steps` <= BK / MMA_K k-steps (the steps past a partial channel chunk would only
// multiply the boxes' zero fill) and the first `n_live` sub-tiles (the rest hold no row of this warpgroup below M).  Each
// count selects a whole fence / wgmma / commit / wait sequence: a branch between the wgmmas of one group makes ptxas
// serialize every wgmma of the kernel (C7520).
template <typename T, int BN, int MT, int TA, int TB, int LIVE>
__device__ __forceinline__ void mma_kblock_steps(float (&acc)[MT][BN / 2], uint64_t da, uint64_t db, uint32_t a_step, uint32_t b_step,
                                                 int steps) {
  static_assert(Elem<T>::BK / Elem<T>::MMA_K == 4, "k-steps per k-block");
  if (steps == 4) mma_kblock<T, BN, MT, TA, TB, 4, LIVE>(acc, da, db, a_step, b_step);
  else if (steps == 3) mma_kblock<T, BN, MT, TA, TB, 3, LIVE>(acc, da, db, a_step, b_step);
  else if (steps == 2) mma_kblock<T, BN, MT, TA, TB, 2, LIVE>(acc, da, db, a_step, b_step);
  else mma_kblock<T, BN, MT, TA, TB, 1, LIVE>(acc, da, db, a_step, b_step);
}
template <typename T, int BN, int MT, int TA, int TB>
__device__ __forceinline__ void mma_kblock_trim(float (&acc)[MT][BN / 2], uint64_t da, uint64_t db, uint32_t a_step, uint32_t b_step,
                                                int steps, int n_live) {
  if (MT == 2 && n_live == 1) mma_kblock_steps<T, BN, MT, TA, TB, 1>(acc, da, db, a_step, b_step, steps);
  else mma_kblock_steps<T, BN, MT, TA, TB, MT>(acc, da, db, a_step, b_step, steps);
}

// tf32 MN-major tile (32-element atoms of 32 k-rows x 128 B, 4 KB apart, 128 B swizzle) → K-major 128 B-swizzled rows,
// rounded to tf32 on the way.  One 16-byte chunk (4 consecutive MN elements at one k) per thread and step.
__device__ __forceinline__ void xpose_tf32(uint8_t* dst, const uint8_t* src, int rows, int tid) {
  for (int c = tid; c < rows * 8; c += 128) {
    const int k = c & 31, mn = (c >> 5) * 4;
    const int mi = mn & 31;
    const float4 v = *reinterpret_cast<const float4*>(src + (mn >> 5) * 4096 + k * 128 + ((((mi >> 2) ^ (k & 7))) << 4));
    const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = mn + i;
      uint32_t t;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(e[i]));
      *reinterpret_cast<uint32_t*>(dst + r * 128 + ((((k >> 2) ^ (r & 7))) << 4) + (k & 3) * 4) = t;
    }
  }
}

// Tile raster.  Default: m fastest (all CTAs of a wave share the few B tiles — right for conv / FC where one operand is
// small).  For GEMMs with many tiles in both directions the wave is folded into bands of group_m m-tiles so the tiles that
// run concurrently form a near-square block and re-use both operands out of L2 instead of streaming one from HBM.
__device__ __forceinline__ void tile_mn(const Params& p, int rem, int& mti, int& nti) {
  if (p.group_m <= 0) { nti = rem / p.mt; mti = rem - nti * p.mt; return; }
  const int band_sz = p.group_m * p.nt;
  const int band = rem / band_sz, within = rem - band * band_sz;
  const int rows = min(p.group_m, p.mt - band * p.group_m);
  nti = within / rows; mti = band * p.group_m + (within - nti * rows);
}

// ------------------------------------------------------------------ the kernel
// Persistent: grid = min(#tiles, #SMs); CTA c processes tiles c, c+grid, … .  The TMA warp fills the smem ring (full/empty
// mbarriers) ahead of the two consumer warpgroups, so the loads of tile i+1 overlap the epilogue of tile i; all per-CTA
// setup (barrier init, descriptor fetch) is paid once per SM instead of once per tile.
// OP = the operand element type (epilogue: store C), or SgdEpilogue<element type>: the momentum-SGD epilogue (Params::sgd; plain
// GEMM, MT = 1, one split, one group) instead of storing C — the FC weight update of a single-GPU step without the fp32 G round
// trip through memory.
template <typename OP, int BN, int MT>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma(const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_b0,
           const __grid_constant__ CUtensorMap tmap_a1, const __grid_constant__ CUtensorMap tmap_b1, const Params p) {
  using T = typename Operand<OP>::Type;
  constexpr bool SGD = Operand<OP>::kSgd;
  static_assert(!SGD || MT == 1, "the SGD epilogue handles 128-row tiles");
  using C = Cfg<T, BN, MT>;
  using E = Elem<T>;
  constexpr int BK = E::BK, MMA_K = E::MMA_K, ATOM = E::ATOM;
  constexpr int SUB_BYTES = BM * 128;              // one 128-row operand sub-tile of one k-block
  constexpr int TM = MT * BM;                      // rows of a CTA tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_raw_u32 = smem_u32(smem_raw);
  const uint32_t smem_base = (smem_raw_u32 + 1023u) & ~1023u;             // SWIZZLE_128B needs 1024B alignment
  const uint32_t xpose_base = smem_base + C::STAGES * C::STAGE_BYTES;
  const uint32_t staging_base = xpose_base + C::XPOSE_BYTES;
  const uint32_t bar_base = staging_base + C::STAGING_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
  auto generic = [&](uint32_t a) { return smem_raw + (a - smem_raw_u32); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int num_kb_total = p.num_kb;
  const int tiles_mn = p.mt * p.nt;
  const int per_group = tiles_mn * p.splits;
  const int total_tiles = per_group * p.groups;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a0);
    tma_prefetch_desc(&tmap_b0);
    if (p.groups > 1) { tma_prefetch_desc(&tmap_a1); tma_prefetch_desc(&tmap_b1); }
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), NUM_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp != 0) return;
    // ===================== TMA producer =====================
    // The WHOLE warp walks the loops (so every index stays warp-uniform and lives in uniform registers); one elected lane
    // issues.  All per-k-block index math is incremental: no divisions inside the k loop.
    const bool leader = elect_one();
    const bool skip_a = (p.dbg & 1) != 0, skip_b = (p.dbg & 2) != 0;
    const bool issue_a = leader && !skip_a, issue_b = leader && !skip_b;
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int grp = tile >= per_group ? 1 : 0;
      const int t2 = tile - grp * per_group;
      const CUtensorMap* const tma_a = grp ? &tmap_a1 : &tmap_a0;
      const CUtensorMap* const tma_b = grp ? &tmap_b1 : &tmap_b0;
      const int split = t2 / tiles_mn, rem = t2 - split * tiles_mn;
      int mti, nti;
      tile_mn(p, rem, mti, nti);
      const int m0 = mti * TM, n0 = nti * BN;
      const int kb0 = split * p.kb_per_split, kb1 = min(num_kb_total, kb0 + p.kb_per_split);
      // sub-tiles that start beyond M are not loaded at all (the consumers issue no wgmma for them; the epilogue drops the rows)
      const int n_sub = (MT == 2 && m0 + BM < p.M) ? 2 : 1;
      if (p.conv_mode == 1) {
        // ---- conv fprop / dgrad: A = im2col box [128 pixels x BK ch] of filter tap (r_, s_), channel chunk cc; B = weights
        const int hw = p.cHo * p.cWo;
        int img0[MT], bw0[MT], bh0[MT];
#pragma unroll
        for (int u = 0; u < MT; ++u) {
          const int mu = m0 + u * BM;
          img0[u] = mu / hw; const int r0_ = mu - img0[u] * hw; const int p0 = r0_ / p.cWo, q0 = r0_ - p0 * p.cWo;
          bw0[u] = q0 * p.cS - p.cP; bh0[u] = p0 * p.cS - p.cP;
        }
        int tap = kb0 / p.c_chunks, cc = kb0 - tap * p.c_chunks;
        int r_ = tap / p.cKW, s_ = tap - r_ * p.cKW;
        const uint32_t tx = (skip_a ? 0u : (uint32_t)(n_sub * SUB_BYTES)) + (skip_b ? 0u : (uint32_t)C::B_BYTES);
        const bool b_t = p.b_mn != 0;
        const int ntaps = p.cKH * p.cKW;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t fb = full_bar(stage);
          if (leader) mbar_expect_tx(fb, tx);
          if (issue_a) {
#pragma unroll
            for (int u = 0; u < MT; ++u)
              if (u < n_sub) tma_load_im2col(sa + u * SUB_BYTES, tma_a, fb, cc * BK, bw0[u], bh0[u], img0[u], s_, r_);
          }
          if (issue_b) {
            if (!b_t) {
              tma_load_3d(sa + C::A_BYTES, tma_b, fb, cc * BK, tap, n0);            // weights [n][tap][k]: K-major box
            } else {
              // dgrad reads the FORWARD filter [k = out-ch][tap][n = in-ch] in place: MN-major boxes {ATOM n, 1 tap, BK k} of
              // the mirrored tap (no flipped / transposed copy of the weights)
#pragma unroll
              for (int j = 0; j < (BN >= ATOM ? BN / ATOM : 1); ++j)
                tma_load_3d(sa + C::A_BYTES + j * (BK * 128), tma_b, fb, n0 + ATOM * j, ntaps - 1 - tap, cc * BK);
            }
          }
          if (++cc == p.c_chunks) { cc = 0; ++tap; if (++s_ == p.cKW) { s_ = 0; ++r_; } }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
        }
      } else if (p.conv_mode == 2) {
        // ---- conv wgrad: A = dy (MN-major) [ATOM m x BK pixels] boxes;  B = BN/ATOM im2col boxes [BK pixels x ATOM ch], one
        //      per (filter tap, channel chunk); the k loop walks pixels BK at a time (W, then H, then N)
        constexpr int NBOX = (BN >= ATOM) ? BN / ATOM : 1;
        const int total_boxes = p.cKH * p.cKW * p.c_chunks;
        const int w_box0 = nti * NBOX;
        int bc[NBOX], bs[NBOX], br[NBOX];
        int nbox = 0;
#pragma unroll
        for (int j = 0; j < NBOX; ++j) {
          const int box = w_box0 + j;
          const int tapj = box / p.c_chunks, c64 = box - tapj * p.c_chunks;
          br[j] = tapj / p.cKW; bs[j] = tapj - br[j] * p.cKW; bc[j] = c64 * ATOM;
          if (box < total_boxes) ++nbox;
        }
        if (skip_b) nbox = 0;
        const uint32_t tx = (skip_a ? 0u : (uint32_t)C::A_BYTES) + (uint32_t)(nbox * (BK * 128));
        const int hw = p.cHo * p.cWo;
        int pix = kb0 * BK;
        int img = pix / hw; const int r2 = pix - img * hw; int pp = r2 / p.cWo, qq = r2 - pp * p.cWo;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + C::A_BYTES;
          const uint32_t fb = full_bar(stage);
          if (leader) mbar_expect_tx(fb, tx);
          if (issue_a) {
#pragma unroll
            for (int j = 0; j < BM / ATOM; ++j) tma_load_2d(sa + j * (BK * 128), tma_a, fb, m0 + ATOM * j, pix);
          }
          if (issue_b) {
            const int cw = qq * p.cS - p.cP, ch = pp * p.cS - p.cP;
#pragma unroll
            for (int j = 0; j < NBOX; ++j)
              if (j < nbox) tma_load_im2col(sb + j * (BK * 128), tma_b, fb, bc[j], cw, ch, img, bs[j], br[j]);
          }
          pix += BK; qq += BK;
          while (qq >= p.cWo) { qq -= p.cWo; if (++pp == p.cHo) { pp = 0; ++img; } }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
        }
      } else {
        // ---- plain GEMM: K-major operands are one box {BK k, rows}; MN-major operands are ATOM-wide column boxes {ATOM mn, BK k}
        const uint32_t tx = (skip_a ? 0u : (uint32_t)(n_sub * SUB_BYTES)) + (skip_b ? 0u : (uint32_t)C::B_BYTES);
        const bool a_mn = p.a_mn != 0, b_mn = p.b_mn != 0;
        int k0 = kb0 * BK;
        for (int kb = kb0; kb < kb1; ++kb, k0 += BK) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + C::A_BYTES;
          const uint32_t fb = full_bar(stage);
          if (leader) mbar_expect_tx(fb, tx);
          if (issue_a) {
#pragma unroll
            for (int u = 0; u < MT; ++u) {
              if (u < n_sub) {
                if (!a_mn) {
                  tma_load_2d(sa + u * SUB_BYTES, tma_a, fb, k0, m0 + u * BM);
                } else {
#pragma unroll
                  for (int j = 0; j < BM / ATOM; ++j) tma_load_2d(sa + u * SUB_BYTES + j * (BK * 128), tma_a, fb, m0 + u * BM + ATOM * j, k0);
                }
              }
            }
          }
          if (issue_b) {
            if (!b_mn) {
              tma_load_2d(sb, tma_b, fb, k0, n0);
            } else {
#pragma unroll
              for (int j = 0; j < (BN >= ATOM ? BN / ATOM : 1); ++j) tma_load_2d(sb + j * (BK * 128), tma_b, fb, n0 + ATOM * j, k0);
            }
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
    return;
  }

  // ===================== consumers: wgmma main loop, then the epilogue of the tile =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int cw = wg - 1;                           // consumer warpgroup: rows [64 cw, 64 cw + 64) of every sub-tile
  const int ctid = threadIdx.x & 127;
  const int wi = warp & 3;                         // warp inside the warpgroup: rows [16 wi, 16 wi + 16) of those
  const bool skip_mma = (p.dbg & 4) != 0;
  const bool a_mn = p.a_mn != 0, b_mn = p.b_mn != 0;
  const bool xa = C::XPOSE && a_mn, xb = C::XPOSE && b_mn;    // tf32 MN-major: wgmma reads the transposed copy
  const uint32_t xa_base = xpose_base + (uint32_t)cw * (C::XA_BYTES + C::B_BYTES), xb_base = xa_base + C::XA_BYTES;
  constexpr uint32_t kMnStep = (uint32_t)(MMA_K * 128) >> 4;
  const uint32_t a_step = (a_mn && !xa) ? kMnStep : 2u, b_step = (b_mn && !xb) ? kMnStep : 2u;
  const uint32_t a_lbo = (a_mn && !xa) ? (uint32_t)(BK * 128) : 16u, b_lbo = (b_mn && !xb) ? (uint32_t)(BK * 128) : 16u;
  const int mode = E::TF32 ? 0 : ((a_mn ? 1 : 0) | (b_mn ? 2 : 0));

  const int esz = p.out_bf16 ? 2 : 4;
  const uint32_t pitch = (uint32_t)(32 * esz + 16);
  uint8_t* const wstage = generic(staging_base) + (size_t)(cw * 4 + wi) * 16 * C::STAGING_ROW;
  const int vec_per_row = (32 * esz) / 16;         // 16-byte vectors per chunk row: 8 (fp32) or 4 (bf16)
  const int rows_per_it = 32 / vec_per_row;
  const int lr = lane / vec_per_row, lv = lane % vec_per_row;
  const bool ld_ok = (((long long)p.ldc * esz) % 16) == 0;
  const int fr = lane >> 2, fc = 2 * (lane & 3);   // accumulator fragment: rows fr, fr + 8 / columns fc, fc + 1 of each 8
  // fprop / dgrad k-blocks walk (tap, channel chunk) with the chunk fastest; the last chunk of a tap holds only
  // Cg - (c_chunks - 1) * BK channels, and the k-steps past them would multiply the boxes' zero fill
  constexpr int STEPS = BK / MMA_K;
  const int k_chunks = p.conv_mode == 1 ? p.c_chunks : 1;
  const int tail_steps = p.conv_mode == 1 ? (p.cCg - (p.c_chunks - 1) * BK + MMA_K - 1) / MMA_K : STEPS;
  // global columns [nb, n_end_c) of the tile's 32-column chunk c (nb + j: column j of the chunk)
  auto chunk_cols = [&](int nti, int n0, int c, int& nb, int& n_end_c) {
    const int cc = 32 * c;                                     // column offset inside the tile
    nb = n0 + cc; n_end_c = p.N;
    if (p.conv_mode == 2) {
      // wgrad: every ATOM-column box of the tile is one (filter tap, ATOM-channel chunk) and lands at column
      // tap*Cg + chunk*ATOM of dW (a 32-column chunk never straddles two boxes)
      const int box = nti * (BN >= ATOM ? BN / ATOM : 1) + cc / ATOM;
      if (box < p.cKH * p.cKW * p.c_chunks) {
        const int tap = box / p.c_chunks, cch = box - tap * p.c_chunks;
        nb = tap * p.cCg + cch * ATOM + (cc % ATOM);
        n_end_c = tap * p.cCg + min(p.cCg, cch * ATOM + ATOM);
      } else {
        nb = 0; n_end_c = 0;
      }
    }
  };
  float acc[MT][BN / 2];
  int stage = 0; uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int grp = tile >= per_group ? 1 : 0;
    const int t2 = tile - grp * per_group;
    const int split = t2 / tiles_mn, rem = t2 - split * tiles_mn;
    int mti, nti;
    tile_mn(p, rem, mti, nti);
    const int m0 = mti * TM, n0 = nti * BN;
    const int kb0 = split * p.kb_per_split, kb1 = min(num_kb_total, kb0 + p.kb_per_split);
    // per-column bias of this lane's columns of the tile, all loaded at once: at tile start, so that the k loop hides the load
    // latency (loaded chunk by chunk in the epilogue, every 32-column chunk waited for its loads between two warp syncs).
    // 256-row tf32 tiles keep the per-chunk loads: their accumulators leave no registers for it.
    float bcol[BN / 8][2];
    auto load_bias = [&]() {
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) bcol[i][0] = bcol[i][1] = 0.f;
      if (p.bias_mode != 1) return;
      const float* const bias_ptr = grp ? p.bias1 : p.bias;
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        int nb, n_end_c;
        chunk_cols(nti, n0, c, nb, n_end_c);
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          const int n = nb + 8 * f + fc;
          if (n < n_end_c) bcol[4 * c + f][0] = __ldg(bias_ptr + n);
          if (n + 1 < n_end_c) bcol[4 * c + f][1] = __ldg(bias_ptr + n + 1);
        }
      }
    };
    constexpr bool kEarlyBias = !(E::TF32 && MT == 2);
    if constexpr (kEarlyBias) load_bias();
    // sub-tiles in which this warpgroup owns at least one row below M (a prefix of the MT sub-tiles); a warpgroup with none
    // issues no wgmma for the tile but still hands every slot back
    int n_live = 0;
#pragma unroll
    for (int u = 0; u < MT; ++u) n_live += (m0 + u * BM + 64 * cw < p.M) ? 1 : 0;
    int cc = kb0 % k_chunks;
#pragma unroll
    for (int u = 0; u < MT; ++u)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[u][i] = 0.f;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const int steps = cc == k_chunks - 1 ? tail_steps : STEPS;
      if (++cc == k_chunks) cc = 0;
      const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
      uint32_t a_addr = sa + (uint32_t)cw * (64 * 128), b_addr = sa + C::A_BYTES;
      if (n_live > 0) {
        if constexpr (C::XPOSE) {
          if (xa || xb) {
            wg_bar(cw);                              // every warp of the group is past the previous k-block's wgmmas
            if (xa) { xpose_tf32(generic(xa_base), generic(a_addr), 64, ctid); a_addr = xa_base; }
            if (xb) { xpose_tf32(generic(xb_base), generic(b_addr), BN, ctid); b_addr = xb_base; }
            fence_proxy_async();                     // generic-proxy writes → visible to wgmma
            wg_bar(cw);
          }
        }
        if (!skip_mma) {
          const uint64_t da = make_smem_desc(a_addr, a_lbo, 1024u), db = make_smem_desc(b_addr, b_lbo, 1024u);
          if (mode == 0) mma_kblock_trim<T, BN, MT, 0, 0>(acc, da, db, a_step, b_step, steps, n_live);
          else if (mode == 1) mma_kblock_trim<T, BN, MT, 1, 0>(acc, da, db, a_step, b_step, steps, n_live);
          else if (mode == 2) mma_kblock_trim<T, BN, MT, 0, 1>(acc, da, db, a_step, b_step, steps, n_live);
          else mma_kblock_trim<T, BN, MT, 1, 1>(acc, da, db, a_step, b_step, steps, n_live);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(stage));           // this warp is done with the slot
      if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
    }

    if constexpr (SGD) {
      // ---- SGD epilogue, one 32-column chunk of the warp's 16-row band at a time: the W and U vectors of the NEXT chunk are
      // loaded before this chunk is updated (up to 16 x 16 B in flight per lane), the staged fp32 chunk gives G as row vectors,
      // and W, U and the bf16 shadow are written back.  The host guarantees ldw % 4 == 0 and 16-byte aligned W / U.
      const Params::Sgd& s = p.sgd;
      const Hyper h{*s.lr_ptr, s.mu, s.inv_k, s.nesterov};
      const int mbase = m0 + 64 * cw + 16 * wi;
      if (mbase >= p.M) continue;                              // warp-uniform: whole band out of range
      constexpr int kPitch = 32 * 4 + 16;
      const int vr = lane >> 3, vc = lane & 7;                 // row inside a 4-row pass, 16-byte vector inside a chunk row
      float4 wb[2][4], ub[2][4];
      auto load_wu = [&](int c, float4 (&w)[4], float4 (&u)[4]) {
        const int nb = n0 + 32 * c;
        if (nb + 32 > p.N) return;                             // partial chunk: loaded element by element below
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const long long gm = (long long)mbase + 4 * it + vr;
          if (gm < p.M) {
            const long long e = gm * s.ldw + nb + 4 * vc;
            w[it] = *reinterpret_cast<const float4*>(s.W + e);
            u[it] = *reinterpret_cast<const float4*>(s.U + e);
          }
        }
      };
      load_wu(0, wb[0], ub[0]);
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        const int nb = n0 + 32 * c;
        const bool full = nb + 32 <= p.N;
        if (c + 1 < BN / 32) load_wu(c + 1, wb[(c + 1) & 1], ub[(c + 1) & 1]);
        float4 (&w)[4] = wb[c & 1];
        float4 (&u)[4] = ub[c & 1];
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          const int i = 4 * c + f, j = 8 * f + fc;
          // the same fmaf(acc, alpha, 0) the plain epilogue stores as G
          *reinterpret_cast<float2*>(wstage + fr * kPitch + j * 4) =
              make_float2(fmaf(acc[0][4 * i], p.alpha, 0.f), fmaf(acc[0][4 * i + 1], p.alpha, 0.f));
          *reinterpret_cast<float2*>(wstage + (fr + 8) * kPitch + j * 4) =
              make_float2(fmaf(acc[0][4 * i + 2], p.alpha, 0.f), fmaf(acc[0][4 * i + 3], p.alpha, 0.f));
        }
        __syncwarp();
        if (full) {
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rr = 4 * it + vr;
            const long long gm = (long long)mbase + rr;
            if (gm < p.M) {
              const long long e = gm * s.ldw + nb + 4 * vc;
              const float4 g = *reinterpret_cast<const float4*>(wstage + rr * kPitch + vc * 16);
              sgd4(w[it], u[it], g, h, s.lr_mult, s.wd);
              *reinterpret_cast<float4*>(s.W + e) = w[it];
              *reinterpret_cast<float4*>(s.U + e) = u[it];
              if (s.H) *reinterpret_cast<uint2*>(s.H + e) = pack_bf16x4(w[it]);
            }
          }
        } else if (nb < p.N) {
          // partial chunk at the right edge: lane = column, element by element
          const int n = nb + lane;
          if (n < p.N) {
            for (int rr = 0; rr < 16; ++rr) {
              const long long gm = (long long)mbase + rr;
              if (gm >= p.M) break;
              const long long e = gm * s.ldw + n;
              float4 w1 = make_float4(s.W[e], 0.f, 0.f, 0.f), u1 = make_float4(s.U[e], 0.f, 0.f, 0.f);
              const float4 g1 = make_float4(*reinterpret_cast<const float*>(wstage + rr * kPitch + lane * 4), 0.f, 0.f, 0.f);
              sgd4(w1, u1, g1, h, s.lr_mult, s.wd);
              s.W[e] = w1.x;
              s.U[e] = u1.x;
              if (s.H) s.H[e] = __float2bfloat16_rn(w1.x);
            }
          }
        }
        __syncwarp();                                          // staging region is free for the next chunk
      }
      continue;
    }

    // ---- epilogue: fragments → bias / ReLU → the warp's staging chunk (16 rows x 32 columns) → global
    uint8_t* const Cg_ptr = reinterpret_cast<uint8_t*>(grp ? p.C1 : p.C);
    const float* const bias_ptr = grp ? p.bias1 : p.bias;
#pragma unroll
    for (int u = 0; u < MT; ++u) {
      const int mbase = m0 + u * BM + 64 * cw + 16 * wi;       // first row of this warp's 16-row band
      if (mbase >= p.M) continue;                              // warp-uniform: whole band out of range
      float bm0 = 0.f, bm1 = 0.f;
      if (p.bias_mode == 2) {
        if (mbase + fr < p.M) bm0 = __ldg(bias_ptr + mbase + fr);
        if (mbase + fr + 8 < p.M) bm1 = __ldg(bias_ptr + mbase + fr + 8);
      }
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        int nb, n_end_c;
        chunk_cols(nti, n0, c, nb, n_end_c);
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          const int i = 4 * c + f;                             // 8-column fragment i of the tile
          const int j = 8 * f + fc;                            // column inside the chunk
          float v0 = acc[u][4 * i], v1 = acc[u][4 * i + 1], v2 = acc[u][4 * i + 2], v3 = acc[u][4 * i + 3];
          float b0 = bm0, b1 = bm0, b2 = bm1, b3 = bm1;
          if (p.bias_mode == 1) {
            if constexpr (kEarlyBias) {
              b0 = b2 = bcol[i][0]; b1 = b3 = bcol[i][1];
            } else {
              const int n = nb + j;
              b0 = b2 = (n < n_end_c) ? __ldg(bias_ptr + n) : 0.f;
              b1 = b3 = (n + 1 < n_end_c) ? __ldg(bias_ptr + n + 1) : 0.f;
            }
          }
          v0 = fmaf(v0, p.alpha, b0); v1 = fmaf(v1, p.alpha, b1); v2 = fmaf(v2, p.alpha, b2); v3 = fmaf(v3, p.alpha, b3);
          if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
          if (p.out_bf16) {
            *reinterpret_cast<__nv_bfloat162*>(wstage + fr * pitch + j * 2) = __floats2bfloat162_rn(v0, v1);
            *reinterpret_cast<__nv_bfloat162*>(wstage + (fr + 8) * pitch + j * 2) = __floats2bfloat162_rn(v2, v3);
          } else {
            *reinterpret_cast<float2*>(wstage + fr * pitch + j * 4) = make_float2(v0, v1);
            *reinterpret_cast<float2*>(wstage + (fr + 8) * pitch + j * 4) = make_float2(v2, v3);
          }
        }
        __syncwarp();
        // Fast path: chunk fully in range and 16-byte aligned → coalesced 16 B row-segment stores (plain, or vector
        // reductions red.global.add.v4.f32 for split-K); the fused reduce-scatter goes through the bulk copy engine.
        const bool staged = (nb + 32 <= n_end_c) && ld_ok && (((reinterpret_cast<uintptr_t>(Cg_ptr) + (long long)nb * esz) % 16) == 0);
        if (staged) {
          if (p.rs_world > 0) {
            // one row segment (32 columns) per lane, reduced into its owner's G as ONE bulk packet: the staging row is the
            // source; generic-proxy writes are fenced into the async proxy first
            fence_proxy_async();
            const long long gm = (long long)mbase + lane;
            if (lane < 16 && gm < p.M) {
              bool local;
              float* d = rs_addr(p, p.rs_e0 + gm * p.ldc + nb, local);
              bulk_reduce_add_f32(d, smem_u32(wstage + (size_t)lane * pitch), (uint32_t)(32 * esz));
            }
            bulk_commit();
            bulk_wait_read();                                  // staging row may be overwritten by the next chunk
          } else {
            uint8_t* gbase = Cg_ptr + (long long)nb * esz + (long long)lv * 16;
            for (int r0 = 0; r0 < 16; r0 += rows_per_it) {
              const int rr = r0 + lr;                          // row inside this warp's 16-row band
              const long long gm = (long long)mbase + rr;
              if (gm < p.M) {
                const uint4 val = *reinterpret_cast<const uint4*>(wstage + (size_t)rr * pitch + (size_t)lv * 16);
                uint8_t* gp = gbase + gm * p.ldc * esz;
                if (p.atomic_out) {
                  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(gp), "f"(__uint_as_float(val.x)),
                               "f"(__uint_as_float(val.y)), "f"(__uint_as_float(val.z)), "f"(__uint_as_float(val.w)) : "memory");
                } else {
                  *reinterpret_cast<uint4*>(gp) = val;
                }
              }
            }
          }
        } else if (nb < n_end_c) {
          // partial or unaligned chunk: lane = column, element by element
          const int n = nb + lane;
          if (n < n_end_c) {
            for (int rr = 0; rr < 16; ++rr) {
              const long long gm = (long long)mbase + rr;
              if (gm >= p.M) break;
              if (p.out_bf16) {
                reinterpret_cast<__nv_bfloat16*>(Cg_ptr)[gm * p.ldc + n] = *reinterpret_cast<const __nv_bfloat16*>(wstage + rr * pitch + lane * 2);
                continue;
              }
              const float v = *reinterpret_cast<const float*>(wstage + rr * pitch + lane * 4);
              if (p.rs_world > 0) { bool local; red_add_sys_f32(rs_addr(p, p.rs_e0 + gm * p.ldc + n, local), v); }
              else if (p.atomic_out) atomicAdd(reinterpret_cast<float*>(Cg_ptr) + gm * p.ldc + n, v);
              else reinterpret_cast<float*>(Cg_ptr)[gm * p.ldc + n] = v;
            }
          }
        }
        __syncwarp();                                          // staging region is free for the next chunk
      }
    }
  }
  if (p.rs_world > 0) bulk_wait_all();                         // bulk reductions have landed before the kernel retires
}


// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)f;
    (void)cudaGetLastError();
  });
  if (!fn) throw std::runtime_error("tmpi_native: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  return fn;
}

// Element type of a tensor map: fp32 operands of the tf32 path are described to the TMA unit as TFLOAT32, which rounds them
// (the tensor core alone would truncate the low 13 mantissa bits, a biased error that does not average out over K).
static CUtensorMapDataType map_type(int esz) {
  return esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
}

// 2-D tensor map (bf16 or fp32 elements): dims {inner, outer}, row pitch in bytes, box {128 bytes, box_outer}, 128B swizzle,
// zero OOB fill.
static CUtensorMap make_tmap(const void* ptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_outer, int esz = 2,
                             int mn_major = 0) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) throw std::runtime_error("tmpi_native: TMA operand base must be 16B aligned");
  if ((pitch_bytes & 15) != 0) throw std::runtime_error("tmpi_native: TMA operand row pitch must be a multiple of 16 bytes");
  using Key = std::tuple<const void*, uint64_t, uint64_t, uint64_t, uint32_t, int, int>;
  static std::map<Key, CUtensorMap> cache;
  static std::mutex mu;
  Key key{ptr, inner, outer, pitch_bytes, box_outer, esz, mn_major};
  const CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esz), box_outer};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = get_encode()(&m, map_type(esz), 2, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("tmpi_native: cuTensorMapEncodeTiled failed, code " + std::to_string((int)r));
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  return m;
}

extern int g_dbg;                  // gemm_set_debug()

template <typename OP, int BN, int MT>
static void launch(const CUtensorMap& ta, const CUtensorMap& tb, Params& p, int splits, cudaStream_t st,
                   const CUtensorMap* ta1 = nullptr, const CUtensorMap* tb1 = nullptr) {
  using T = typename Operand<OP>::Type;
  using C = Cfg<T, BN, MT>;
  p.dbg = g_dbg;
  if (!ta1) { p.groups = 1; p.C1 = nullptr; p.bias1 = nullptr; }
  static bool attr_set = false;
  if (!attr_set) {
    check_cuda(cudaFuncSetAttribute(gemm_wgmma<OP, BN, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES), "gemm smem attr");
    attr_set = true;
  }
  if (MT == 2 && sizeof(T) == 4 && (p.a_mn || p.b_mn)) throw std::runtime_error("tmpi_native: 256-row tf32 tiles need K-major operands");
  if (sizeof(T) == 4 && p.out_bf16) throw std::runtime_error("tmpi_native: the tf32 path stores fp32");
  const long long total = (long long)p.mt * p.nt * splits * p.groups;
  const int grid = (int)std::min<long long>(total, (long long)sm_count());
  gemm_wgmma<OP, BN, MT><<<grid, NUM_THREADS, C::SMEM_BYTES, st>>>(ta, tb, ta1 ? *ta1 : ta, tb1 ? *tb1 : tb, p);
  count_launch();
  TMPI_CHECK_LAUNCH("gemm_wgmma"); ::tmpi::check_capture(st, "gemm_wgmma");
}

}  // namespace wgmma
}  // namespace tmpi
