// Flat-arena optimizer + collective kernels (sm_90a, NVLink / NVSwitch peer memory).
//
// Every rank maps every peer's *symmetric arena* (W | G | U | R | H regions at identical byte offsets) and a
// small *signal pad* into its own address space (csrc/peer_arena.cpp).  The kernels below therefore issue
// plain ld/st (or multimem.* when a multicast mapping exists) on peer pointers — no NCCL/MPI call is on the
// path.  What the reference does in three separate stages per tensor
//     Barrier → ncclAllReduce(vels→vels2) → one elementwise update kernel per tensor
// (theanompi/lib/exchanger.py:120-134, exchanger_strategy.py:121-127, opt.py:181-268) is ONE launch here:
//     flag barrier → read all peers' gradients → average → weight-decay/momentum/lr update → bf16 shadow
//     [→ push the updated slice to the peers] → flag barrier.
//
//   flat_update_kernel<Rule>   k = 1 (no peers): one local optimizer pass over a block range (SGD = sgd4, Adam, RMSProp,
//                              Adadelta, centred RMSProp)
//   fused_oneshot_sgd   every rank reduces the whole range itself (latency-optimal, small buckets)
//   fused_twoshot_sgd   reduce-scatter → update owned slice → push updated weights to all peers (bandwidth-optimal)
//   fused_nvls_sgd      same with multimem.ld_reduce / multimem.st (reduction + broadcast inside the NVSwitch)
//   allreduce_*         plain sum/avg into a destination region (classic cdd vels→vels2, 'avg' weight averaging)
//   easgd_elastic       d = α(w − c); w −= d; c += d   on the center's memory over NVLink   (exchanger.py:188-211)
//   gosgd_*             push / merge / pull-merge of weights with push-sum weights α     (exchanger.py:450-462)
//   K1..K5 of the reference (float2half/half2float, sumfloats/sumhalfs, vecadd/vecaddhalf) for the legacy strategies.
#include <type_traits>
#include "common.cuh"
#include "api.h"

namespace tmpi {

constexpr int kThreads = 256;            // one float4 per thread per 1024-element arena block

// ------------------------------------------------------------------ memory helpers
__device__ __forceinline__ float4 ld_sys_f4(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ld_sys_u2(const void* p) {
  uint2 v;
  asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_f4(float* p, float4 v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_u2(void* p, uint2 v) {
  asm volatile("st.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ float4 mc_ld_reduce_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ uint2 mc_ld_reduce_bf16x4(const void* mc) {
  uint2 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v2.bf16x2 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_f4(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void mc_st_u2(void* mc, uint2 v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(mc), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)) : "memory");
}
__device__ __forceinline__ float4 unpack_bf16x4(uint2 u) {
  float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.x)), b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

template <typename T> __device__ __forceinline__ T* region(const CommCtx& c, int p, long long off) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(c.arena[p]) + off);
}

// ------------------------------------------------------------------ cross-rank per-block flag barrier
// Block b of every rank increments slot [b][my rank] on every peer (red.release.sys) and spins until its own
// slots [b][p] reach the block's epoch (ld.acquire.sys).  Epochs live in device memory, so the same captured
// CUDA graph can be replayed.  Bounded spin: a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void block_barrier(const CommCtx& c) {
  __syncthreads();
  uint32_t* ep = c.epoch + blockIdx.x;
  const uint32_t target = *ep + 1u;
  if ((int)threadIdx.x < c.world) {
    uint32_t* remote = c.sig[threadIdx.x] + (size_t)blockIdx.x * kMaxRanks + c.rank;
    asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(remote) : "memory");
    const uint32_t* mine = c.sig[c.rank] + (size_t)blockIdx.x * kMaxRanks + threadIdx.x;
    uint32_t v;
    long long t0 = clock64();
    while (true) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
      if ((int)(v - target) >= 0) break;
      if (clock64() - t0 > c.spin_limit) { __trap(); }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *ep = target;
}

// ============================================================================ k = 1: the local flat optimizers
// One kernel template walks the arena blocks [blk_lo, blk_hi): it looks up the block's group, loads W, G and the rule's kState
// state vectors as float4, lets the rule update them, stores them and refreshes the bf16 shadow.  lr is read from device memory
// once per launch, so a captured CUDA graph follows lr changes.  A rule holds its hyperparameters (built inside the kernel from
// scalar launch arguments, which keeps each instantiation's code identical to a hand-written kernel) and its per-element
// update; `prologue` computes per-launch constants, `skip` drops whole blocks by group, `enter_block` loads per-block constants
// through the block → tensor table (LARS, LAMB: the tensor's trust ratio).  A rule that takes its direction from state written by
// an earlier pass (LAMB) neither reads G (kReadsG) nor stores its state back (kWritesState).
// Global gradient-norm clipping (the kClip instantiations, grad_clip_norm below) makes the step use s·g: the kernel multiplies every
// loaded gradient by s, or, for a rule that already scales the gradient by a launch constant (kFoldsClip), folds s into it.
struct FlatRule {
  static constexpr bool kAdvancesStep = false;
  static constexpr bool kReadsG = true;
  static constexpr bool kWritesState = true;
  static constexpr bool kFoldsClip = false;
  __device__ __forceinline__ void prologue(const unsigned long long* step) {}
  __device__ __forceinline__ bool skip(const GroupTable& tab, int g) const { return false; }
  __device__ __forceinline__ void enter_block(long long b, const int* block_tensor, const float* tensor_scale) {}
  __device__ __forceinline__ void fold_clip(float s) {}
};

// filter: 0 all groups, 1 only non-exchanged (BN) groups, 2 only exchanged groups
__device__ __forceinline__ bool filtered_out(const GroupTable& tab, int g, int filter) {
  return (filter == 1 && tab.exch[g]) || (filter == 2 && !tab.exch[g]);
}

// momentum SGD, `common.cuh: sgd4` (the arithmetic of the GEMM SGD epilogue and the fused collectives).  State: U.  filter as above.
struct SgdRule : FlatRule {
  static constexpr int kState = 1;
  static constexpr bool kFoldsClip = true;                 // g·inv_k·s
  float mu, inv_k;
  int nesterov, filter;
  __device__ __forceinline__ SgdRule(float a, float b, float, int i, int j) : mu(a), inv_k(b), nesterov(i), filter(j) {}
  __device__ __forceinline__ bool skip(const GroupTable& tab, int g) const { return filtered_out(tab, g, filter); }
  __device__ __forceinline__ void fold_clip(float s) { inv_k = __fmul_rn(inv_k, s); }
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    sgd4(w, s[0], gg, Hyper{lr0, mu, inv_k, nesterov}, lrm, wd);
  }
};

// Adam (Wide-ResNet's optimizer, ref keras_model_zoo/wresnet.py:159).  State: M (the arena's U), V.
// m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  w -= lr * (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + eps), t read from a
// device counter that adam_advance_kernel bumps after the update (the captured CUDA graph keeps counting).
struct AdamRule : FlatRule {
  static constexpr int kState = 2;
  static constexpr bool kAdvancesStep = true;
  float b1, b2, eps, c1, c2;
  __device__ __forceinline__ AdamRule(float a, float b, float c, int, int) : b1(a), b2(b), eps(c) {}
  __device__ __forceinline__ void prologue(const unsigned long long* step) {
    const float t = (float)(*step + 1ull);
    c1 = 1.f / (1.f - __powf(b1, t)); c2 = 1.f / (1.f - __powf(b2, t));
  }
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    const float lr = lr0 * lrm;
    float4 &m = s[0], &v = s[1];
#define TMPI_ADAM1(Wc, Mc, Vc, Gc)                                    \
  {                                                                  \
    const float ge = Gc + wd * Wc;                                   \
    Mc = b1 * Mc + (1.f - b1) * ge;                                  \
    Vc = b2 * Vc + (1.f - b2) * ge * ge;                             \
    Wc -= lr * (Mc * c1) / (sqrtf(Vc * c2) + eps);                   \
  }
    TMPI_ADAM1(w.x, m.x, v.x, gg.x) TMPI_ADAM1(w.y, m.y, v.y, gg.y) TMPI_ADAM1(w.z, m.z, v.z, gg.z) TMPI_ADAM1(w.w, m.w, v.w, gg.w)
#undef TMPI_ADAM1
  }
};
__global__ void adam_advance_kernel(unsigned long long* step) { if (threadIdx.x == 0 && blockIdx.x == 0) *step += 1ull; }
// the same after a clipped step: a skipped step (non-finite gradient norm) does not advance the counter
__global__ void adam_advance_clip_kernel(unsigned long long* step, const ClipRecord* __restrict__ clip) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && clip->finite) *step += 1ull;
}

// Per-update learning-rate schedule (ops/reference.py: lr_at is the same formula on the host).  One thread: lr(u) for the update
// index u = *counter, in fp64 and rounded once to fp32, into *lr (the arena's hyper[0]), then *counter = u + 1.  Every operation
// with a correctly rounded result is spelled as an _rn intrinsic, so it is never contracted into an FMA (the build uses
// --use_fast_math): warm-up, constant and multistep values are bit-equal to the host's; cosine and poly go through cos / pow.
__global__ void lr_schedule_kernel(LrScheduleParams p, unsigned long long* __restrict__ counter, float* __restrict__ lr) {
  const long long u = (long long)*counter;
  double v = p.peak;
  if (u < p.warmup) {
    v = __dmul_rn(p.peak, __dadd_rn(p.start, __ddiv_rn(__dmul_rn(__dsub_rn(1.0, p.start), (double)u), (double)p.warmup)));
  } else if (p.policy == LR_MULTISTEP) {
    for (int k = 0; k < p.n_milestones; ++k)
      if (u >= p.milestones[k]) v = __dmul_rn(v, p.gamma);
  } else if (p.policy != LR_CONSTANT) {
    const double q = fmin(fmax(__ddiv_rn((double)(u - p.warmup), (double)(p.total - p.warmup)), 0.0), 1.0);
    const double f = p.policy == LR_COSINE ? __dmul_rn(0.5, __dadd_rn(1.0, cos(__dmul_rn(3.141592653589793, q))))
                                           : pow(__dsub_rn(1.0, q), p.power);
    v = __dadd_rn(p.final_lr, __dmul_rn(__dsub_rn(p.peak, p.final_lr), f));
  }
  *lr = __double2float_rn(v);
  *counter = (unsigned long long)u + 1ull;
}

void lr_schedule(const LrScheduleParams& p, void* counter, void* lr, cudaStream_t st) {
  if (p.policy < LR_CONSTANT || p.policy > LR_MULTISTEP) throw std::runtime_error("lr_schedule: unknown policy " + std::to_string(p.policy));
  if (p.n_milestones < 0 || p.n_milestones > kMaxLrMilestones) throw std::runtime_error("lr_schedule: at most 8 milestones");
  if (!counter || !lr) throw std::runtime_error("lr_schedule: needs the update counter and the lr slot");
  lr_schedule_kernel<<<1, 1, 0, st>>>(p, (unsigned long long*)counter, (float*)lr);
  count_launch(); TMPI_CHECK_LAUNCH("lr_schedule"); ::tmpi::check_capture(st, "lr_schedule");
}

// RMSProp (the GANs' optimizer, torch.optim.RMSprop without momentum).  State: V.
// v = alpha v + (1 - alpha) g^2;  w -= lr * g / (sqrt(v) + eps);  then, when clip > 0, w = clamp(w, -clip, clip) (the WGAN critic's
// weight clipping in the same pass).
struct RmspropRule : FlatRule {
  static constexpr int kState = 1;
  float alpha, eps, clip;
  __device__ __forceinline__ RmspropRule(float a, float b, float c, int, int) : alpha(a), eps(b), clip(c) {}
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    const float lr = lr0 * lrm;
    float4& v = s[0];
#define TMPI_RMS1(Wc, Vc, Gc)                                         \
  {                                                                  \
    const float ge = Gc + wd * Wc;                                   \
    Vc = alpha * Vc + (1.f - alpha) * ge * ge;                       \
    Wc -= lr * ge / (sqrtf(Vc) + eps);                               \
    if (clip > 0.f) Wc = fminf(fmaxf(Wc, -clip), clip);              \
  }
    TMPI_RMS1(w.x, v.x, gg.x) TMPI_RMS1(w.y, v.y, gg.y) TMPI_RMS1(w.z, v.z, gg.z) TMPI_RMS1(w.w, v.w, gg.w)
#undef TMPI_RMS1
  }
};

// Adadelta (the LSTM's default optimizer, torch.optim.Adadelta).  State: U (the arena's update accumulator), V.
// v = rho v + (1 - rho) g^2;  d = sqrt(u + eps) / sqrt(v + eps) * g;  u = rho u + (1 - rho) d^2;  w -= lr * d.
struct AdadeltaRule : FlatRule {
  static constexpr int kState = 2;
  float rho, eps;
  __device__ __forceinline__ AdadeltaRule(float a, float b, float, int, int) : rho(a), eps(b) {}
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    const float lr = lr0 * lrm;
    float4 &u = s[0], &v = s[1];
#define TMPI_ADADELTA1(Wc, Uc, Vc, Gc)                                \
  {                                                                  \
    const float ge = Gc + wd * Wc;                                   \
    Vc = rho * Vc + (1.f - rho) * ge * ge;                           \
    const float d = sqrtf(Uc + eps) / sqrtf(Vc + eps) * ge;          \
    Uc = rho * Uc + (1.f - rho) * d * d;                             \
    Wc -= lr * d;                                                    \
  }
    TMPI_ADADELTA1(w.x, u.x, v.x, gg.x) TMPI_ADADELTA1(w.y, u.y, v.y, gg.y) TMPI_ADADELTA1(w.z, u.z, v.z, gg.z)
    TMPI_ADADELTA1(w.w, u.w, v.w, gg.w)
#undef TMPI_ADADELTA1
  }
};

// centred RMSProp with momentum (the reference LSTM's rmsprop).  State: M (the arena's U), R, S; eps sits inside the square root.
// r = rho r + (1 - rho) g;  s = rho s + (1 - rho) g^2;  m = mu m - lr * g / sqrt(s - r^2 + eps);  w += m.
struct CenteredRmspropRule : FlatRule {
  static constexpr int kState = 3;
  float rho, mu, eps;
  __device__ __forceinline__ CenteredRmspropRule(float a, float b, float c, int, int) : rho(a), mu(b), eps(c) {}
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    const float lr = lr0 * lrm;
    float4 &m = s[0], &r = s[1], &sq = s[2];
#define TMPI_CRMS1(Wc, Mc, Rc, Sc, Gc)                                \
  {                                                                  \
    const float ge = Gc + wd * Wc;                                   \
    Rc = rho * Rc + (1.f - rho) * ge;                                \
    Sc = rho * Sc + (1.f - rho) * ge * ge;                           \
    Mc = mu * Mc - lr * ge / sqrtf(Sc - Rc * Rc + eps);              \
    Wc += Mc;                                                        \
  }
    TMPI_CRMS1(w.x, m.x, r.x, sq.x, gg.x) TMPI_CRMS1(w.y, m.y, r.y, sq.y, gg.y) TMPI_CRMS1(w.z, m.z, r.z, sq.z, gg.z)
    TMPI_CRMS1(w.w, m.w, r.w, sq.w, gg.w)
#undef TMPI_CRMS1
  }
};

// LARS (layer-wise adaptive rate scaling, You, Gitman and Ginsburg 2017): momentum SGD with the effective gradient of every tensor
// scaled by its trust ratio t (lars_trust below), i.e. sgd4 with inv_k·t and wd·t.  State: U.  filter as SgdRule.
struct LarsRule : SgdRule {
  float t_inv_k = 0.f, t = 0.f;
  __device__ __forceinline__ LarsRule(float a, float b, float c, int i, int j) : SgdRule(a, b, c, i, j) {}
  __device__ __forceinline__ void enter_block(long long b, const int* block_tensor, const float* tensor_scale) {
    t = tensor_scale[block_tensor[b]];
    t_inv_k = inv_k * t;
  }
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4& gg, float lr0, float lrm, float wd) const {
    sgd4(w, s[0], gg, Hyper{lr0, mu, t_inv_k, nesterov}, lrm, wd * t);
  }
};

// LAMB (You et al. 2019, "Large Batch Optimization for Deep Learning"): Adam moments, decoupled weight decay and a per-tensor trust
// ratio ‖W‖ / ‖r‖ on the update direction r.  A step is three passes: lamb_moments_kernel advances M and V and writes the per-block
// sums of squares of W and r, lars_finalize_kernel turns them into the trust ratios, and LambRule recomputes r from the new M, V
// (with the same helper) and applies it.  Both passes read the step counter before adam_advance_kernel bumps it.
// Bias corrections of step t = *step + 1, c1 = 1 / (1 − b1^t), c2 = 1 / (1 − b2^t), in fp64: 1 − b2^t of the first steps is small.
__device__ __forceinline__ void lamb_bias_corrections(const unsigned long long* step, float b1, float b2, float& c1, float& c2) {
  const double t = (double)(*step + 1ull);
  c1 = (float)(1.0 / (1.0 - pow((double)b1, t)));
  c2 = (float)(1.0 / (1.0 - pow((double)b2, t)));
}
// the update direction of one element from its advanced moments: r = (m·c1) / (sqrt(v·c2) + eps) + wd·w
__device__ __forceinline__ float lamb_dir(float w, float m, float v, float c1, float c2, float eps, float wd) {
  return (m * c1) / (sqrtf(v * c2) + eps) + wd * w;
}

// Pass 3 of a LAMB step: w -= lr·lr_mult·trust·r.  State: M (the arena's U), V, both only read here.  filter as SgdRule.
struct LambRule : FlatRule {
  static constexpr int kState = 2;
  static constexpr bool kAdvancesStep = true;              // after a pass with filter != 1 (launch_flat_update)
  static constexpr bool kReadsG = false;
  static constexpr bool kWritesState = false;
  float b1, b2, eps, c1 = 0.f, c2 = 0.f, t = 0.f;
  int filter;
  __device__ __forceinline__ LambRule(float a, float b, float c, int i, int) : b1(a), b2(b), eps(c), filter(i) {}
  __device__ __forceinline__ void prologue(const unsigned long long* step) { lamb_bias_corrections(step, b1, b2, c1, c2); }
  __device__ __forceinline__ bool skip(const GroupTable& tab, int g) const { return filtered_out(tab, g, filter); }
  __device__ __forceinline__ void enter_block(long long b, const int* block_tensor, const float* tensor_scale) {
    t = tensor_scale[block_tensor[b]];
  }
  __device__ __forceinline__ void apply(float4& w, float4* s, const float4&, float lr0, float lrm, float wd) const {
    const float lr = lr0 * lrm * t;
    const float4 &m = s[0], &v = s[1];
    w.x -= lr * lamb_dir(w.x, m.x, v.x, c1, c2, eps, wd);
    w.y -= lr * lamb_dir(w.y, m.y, v.y, c1, c2, eps, wd);
    w.z -= lr * lamb_dir(w.z, m.z, v.z, c1, c2, eps, wd);
    w.w -= lr * lamb_dir(w.w, m.w, v.w, c1, c2, eps, wd);
  }
};

// kClip: `clip` is the record grad_clip_norm wrote for this step.  A step whose gradient norm is not finite returns before it touches
// memory; otherwise the gradient is scaled by clip->scale.  __fmul_rn is never contracted into an FMA, so with s = 1 every later
// operation sees the same operands as without clipping and the step is bit-identical to the kClip = false instantiation.
template <class Rule, bool kClip = false>
__global__ void __launch_bounds__(kThreads) flat_update_kernel(float* __restrict__ W, const float* __restrict__ G, float* __restrict__ S0,
                                                               float* __restrict__ S1, float* __restrict__ S2, __nv_bfloat16* __restrict__ H,
                                                               const uint8_t* __restrict__ block_group, GroupTable tab,
                                                               const float* __restrict__ lr_ptr, const unsigned long long* __restrict__ step,
                                                               float ha, float hb, float hc, int ia, int ib, long long blk_lo,
                                                               long long blk_hi, const int* __restrict__ block_tensor,
                                                               const float* __restrict__ tensor_scale, const ClipRecord* __restrict__ clip) {
  Rule r(ha, hb, hc, ia, ib);
  float cs = 1.f;
  if constexpr (kClip) {
    const ClipRecord rec = *clip;
    if (!rec.finite) return;                              // skipped step: W, H and the state stay as they are
    cs = rec.scale;
    if constexpr (Rule::kFoldsClip) r.fold_clip(cs);
  }
  r.prologue(step);
  const float lr0 = *lr_ptr;
  for (long long b = blk_lo + blockIdx.x; b < blk_hi; b += gridDim.x) {
    const int g = block_group[b];
    if (r.skip(tab, g)) continue;
    r.enter_block(b, block_tensor, tensor_scale);
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    float4 w = *reinterpret_cast<const float4*>(W + i), s[Rule::kState];
    s[0] = *reinterpret_cast<const float4*>(S0 + i);
    if constexpr (Rule::kState > 1) s[1] = *reinterpret_cast<const float4*>(S1 + i);
    if constexpr (Rule::kState > 2) s[2] = *reinterpret_cast<const float4*>(S2 + i);
    float4 gg = {};
    if constexpr (Rule::kReadsG) gg = *reinterpret_cast<const float4*>(G + i);
    if constexpr (kClip && !Rule::kFoldsClip) {
      gg.x = __fmul_rn(gg.x, cs); gg.y = __fmul_rn(gg.y, cs); gg.z = __fmul_rn(gg.z, cs); gg.w = __fmul_rn(gg.w, cs);
    }
    r.apply(w, s, gg, lr0, tab.lr_mult[g], tab.wd[g]);
    *reinterpret_cast<float4*>(W + i) = w;
    if constexpr (Rule::kWritesState) {
      *reinterpret_cast<float4*>(S0 + i) = s[0];
      if constexpr (Rule::kState > 1) *reinterpret_cast<float4*>(S1 + i) = s[1];
      if constexpr (Rule::kState > 2) *reinterpret_cast<float4*>(S2 + i) = s[2];
    }
    if (H) *reinterpret_cast<uint2*>(H + i) = pack_bf16x4(w);
  }
}

// ha, hb, hc, ia, ib: the rule's hyperparameters, in the order of its constructor
template <class Rule, bool kClip = false>
static void launch_flat_update(const char* name, const FlatUpdateArgs& a, float ha, float hb, float hc, int ia, int ib, cudaStream_t st) {
  if (a.lo % kArenaBlock || a.hi % kArenaBlock) throw std::runtime_error(std::string(name) + ": range must be block aligned");
  const long long nb = (a.hi - a.lo) / kArenaBlock;
  if (nb <= 0) return;
  int grid = (int)std::min<long long>(nb, (long long)sm_count() * 8);
  flat_update_kernel<Rule, kClip><<<grid, kThreads, 0, st>>>((float*)a.W, (const float*)a.G, (float*)a.S[0], (float*)a.S[1],
                                                             (float*)a.S[2], (__nv_bfloat16*)a.H, (const uint8_t*)a.block_group, a.tab,
                                                             (const float*)a.lr_ptr, (const unsigned long long*)a.step, ha, hb, hc, ia, ib,
                                                             a.lo / kArenaBlock, a.hi / kArenaBlock, (const int*)a.block_tensor,
                                                             (const float*)a.tensor_scale, (const ClipRecord*)a.clip);
  // a filter-1 (batch-norm only) pass is followed by the filter-2 pass of the same step, which advances the counter
  const bool advance = Rule::kAdvancesStep && a.filter != 1;
  if (advance && kClip) adam_advance_clip_kernel<<<1, 32, 0, st>>>((unsigned long long*)a.step, (const ClipRecord*)a.clip);
  else if (advance) adam_advance_kernel<<<1, 32, 0, st>>>((unsigned long long*)a.step);
  count_launch(advance ? 2 : 1); TMPI_CHECK_LAUNCH(name); ::tmpi::check_capture(st, name);
}

template <class Rule>
static void launch_flat_update_clip(const char* name, const FlatUpdateArgs& a, float ha, float hb, float hc, int ia, int ib,
                                    cudaStream_t st) {
  if (a.clip) launch_flat_update<Rule, true>(name, a, ha, hb, hc, ia, ib, st);
  else launch_flat_update<Rule, false>(name, a, ha, hb, hc, ia, ib, st);
}

void flat_update(const FlatUpdateArgs& a, cudaStream_t st) {
  static const char* const names[] = {"sgd_flat", "adam_flat", "rmsprop_flat", "adadelta_flat", "rmsprop_centered_flat", "lars_flat",
                                      "lamb_flat"};
  static const int n_hp[] = {3, 3, 3, 2, 3, 3, 3};
  if (a.rule < FLAT_SGD || a.rule > FLAT_LAMB) throw std::runtime_error("flat_update: unknown rule " + std::to_string(a.rule));
  const char* name = names[a.rule];
  if (a.n_hp != n_hp[a.rule])
    throw std::runtime_error(std::string(name) + ": expected " + std::to_string(n_hp[a.rule]) + " hyperparameters");
  if (a.rule == FLAT_ADAM && !a.step) throw std::runtime_error("adam_flat: needs a step counter");
  if (a.rule == FLAT_LARS && (!a.block_tensor || !a.tensor_scale)) throw std::runtime_error("lars_flat: needs the block → tensor table and the trust ratios");
  if (a.rule == FLAT_LAMB && !a.step) throw std::runtime_error("lamb_flat: needs a step counter");
  if (a.rule == FLAT_LAMB && (!a.block_tensor || !a.tensor_scale)) throw std::runtime_error("lamb_flat: needs the block → tensor table and the trust ratios");
  if (a.clip && (a.rule == FLAT_LARS || a.rule == FLAT_LAMB))
    throw std::runtime_error(std::string(name) + ": gradient-norm clipping is for the sgd, adam, rmsprop, adadelta and rmsprop_centered rules");
  const float* h = a.hp;
  switch (a.rule) {
    case FLAT_SGD: launch_flat_update_clip<SgdRule>(name, a, h[0], h[2], 0.f, h[1] != 0.f, a.filter, st); break;
    case FLAT_ADAM: launch_flat_update_clip<AdamRule>(name, a, h[0], h[1], h[2], 0, 0, st); break;
    case FLAT_RMSPROP: launch_flat_update_clip<RmspropRule>(name, a, h[0], h[1], h[2], 0, 0, st); break;
    case FLAT_ADADELTA: launch_flat_update_clip<AdadeltaRule>(name, a, h[0], h[1], 0.f, 0, 0, st); break;
    case FLAT_RMSPROP_CENTERED: launch_flat_update_clip<CenteredRmspropRule>(name, a, h[0], h[1], h[2], 0, 0, st); break;
    case FLAT_LARS: launch_flat_update<LarsRule>(name, a, h[0], h[2], 0.f, h[1] != 0.f, a.filter, st); break;
    default: launch_flat_update<LambRule>(name, a, h[0], h[1], h[2], a.filter, 0, st); break;
  }
}

// ============================================================================ LARS trust ratios
// Pass 1: for every arena block of [blk_lo, blk_hi), the sums of squares of W and of the gradient over the block's real elements
// (those below the end of its tensor) → partial[b] = {Σw², Σg²}.  One block per CTA iteration, one float4 per thread, warp shuffles
// and a fixed-order sum over the 8 warps: no atomics, so the result does not depend on the grid.
// kW = false (gradient clipping): W is not read and partial[b] = Σg² alone, so the pass moves 4 B per element.
template <bool kW>
__global__ void __launch_bounds__(kThreads) lars_partial_kernel(const float* __restrict__ W, const float* __restrict__ G,
                                                                const int* __restrict__ block_tensor, const long long* __restrict__ tensor_span,
                                                                std::conditional_t<kW, float2, float>* __restrict__ partial,
                                                                long long blk_lo, long long blk_hi) {
  __shared__ float2 red[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long b = blk_lo + blockIdx.x; b < blk_hi; b += gridDim.x) {
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const int t = block_tensor[b];
    const long long end = tensor_span[2 * t] + tensor_span[2 * t + 1];
    float4 w = {}, g;
    if constexpr (kW) w = *reinterpret_cast<const float4*>(W + i);
    g = *reinterpret_cast<const float4*>(G + i);
    if (i + 4 > end) {                                   // the tensor's last block: zero the padding past its end
      if (i + 0 >= end) { w.x = 0.f; g.x = 0.f; }
      if (i + 1 >= end) { w.y = 0.f; g.y = 0.f; }
      if (i + 2 >= end) { w.z = 0.f; g.z = 0.f; }
      if (i + 3 >= end) { w.w = 0.f; g.w = 0.f; }
    }
    float sw = w.x * w.x + w.y * w.y + w.z * w.z + w.w * w.w;
    float sg = g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w;
    if constexpr (kW) sw = warp_sum(sw);
    sg = warp_sum(sg);
    if (lane == 0) red[warp] = make_float2(sw, sg);
    __syncthreads();
    if (threadIdx.x == 0) {
      float2 s = red[0];
#pragma unroll
      for (int k = 1; k < kThreads / 32; ++k) { s.x += red[k].x; s.y += red[k].y; }
      if constexpr (kW) partial[b] = s;
      else partial[b] = s.y;
    }
    __syncthreads();                                     // red[] is reused by the next block
  }
}

// Pass 2: one CTA per tensor sums its block partials in fp64 in a fixed order and writes norms[t] = {‖W‖, ‖g‖} (g = G·inv_k) and
// the trust ratio: eta·‖W‖ / (‖g‖ + wd·‖W‖) for the weight group when both norms are positive, else 1.
constexpr int kLarsGroupW = 0;                           // parallel/arena.py G_W
__global__ void __launch_bounds__(kThreads) lars_finalize_kernel(const float2* __restrict__ partial, const long long* __restrict__ tensor_span,
                                                                 const uint8_t* __restrict__ block_group, GroupTable tab, float inv_k, float eta,
                                                                 float2* __restrict__ norms, float* __restrict__ trust) {
  __shared__ double red[2][kThreads / 32];
  const int t = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long b0 = tensor_span[2 * t] / kArenaBlock, nb = ceil_div64(tensor_span[2 * t + 1], kArenaBlock);
  double sw = 0.0, sg = 0.0;
  for (long long k = threadIdx.x; k < nb; k += kThreads) {
    const float2 p = partial[b0 + k];
    sw += (double)p.x; sg += (double)p.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { sw += __shfl_xor_sync(0xffffffffu, sw, o); sg += __shfl_xor_sync(0xffffffffu, sg, o); }
  if (lane == 0) { red[0][warp] = sw; red[1][warp] = sg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    sw = red[0][0]; sg = red[1][0];
    for (int k = 1; k < kThreads / 32; ++k) { sw += red[0][k]; sg += red[1][k]; }
    const double wn = sqrt(sw), gn = sqrt(sg) * (double)inv_k;
    const int grp = nb > 0 ? block_group[b0] : -1;      // an empty tensor owns no block
    double tr = 1.0;
    if (grp == kLarsGroupW && wn > 0.0 && gn > 0.0) tr = (double)eta * wn / (gn + (double)tab.wd[grp] * wn);
    norms[t] = make_float2((float)wn, (float)gn);
    trust[t] = (float)tr;
  }
}

void lars_trust(const LarsTrustArgs& a, cudaStream_t st) {
  if (a.n_blocks <= 0 || a.n_tensors <= 0) return;
  const int grid = (int)std::min<long long>(a.n_blocks, (long long)sm_count() * 8);
  lars_partial_kernel<true><<<grid, kThreads, 0, st>>>((const float*)a.W, (const float*)a.G, (const int*)a.block_tensor,
                                                       (const long long*)a.tensor_span, (float2*)a.partial, 0, a.n_blocks);
  TMPI_CHECK_LAUNCH("lars_partial");
  lars_finalize_kernel<<<a.n_tensors, kThreads, 0, st>>>((const float2*)a.partial, (const long long*)a.tensor_span,
                                                         (const uint8_t*)a.block_group, a.tab, a.inv_k, a.eta, (float2*)a.norms,
                                                         (float*)a.trust);
  count_launch(2); TMPI_CHECK_LAUNCH("lars_finalize"); ::tmpi::check_capture(st, "lars_trust");
}

// ============================================================================ LAMB trust ratios
// Pass 1 of a LAMB step, over the blocks of [blk_lo, blk_hi) that `filter` keeps: with g = G·inv_k, advance the moments
// M = b1·M + (1 − b1)·g, V = b2·V + (1 − b2)·g² and write partial[b] = {Σw², Σr²} over the block's real elements, r = lamb_dir(...).
// W and G are only read.  A skipped block keeps the partial sums of the last pass that covered it.  The reduction is the one of
// lars_partial_kernel: no atomics, so the result does not depend on the grid.
__global__ void __launch_bounds__(kThreads) lamb_moments_kernel(const float* __restrict__ W, const float* __restrict__ G, float* __restrict__ M,
                                                                float* __restrict__ V, const uint8_t* __restrict__ block_group, GroupTable tab,
                                                                const unsigned long long* __restrict__ step, float b1, float b2, float eps,
                                                                float inv_k, int filter, const int* __restrict__ block_tensor,
                                                                const long long* __restrict__ tensor_span, float2* __restrict__ partial,
                                                                long long blk_lo, long long blk_hi) {
  __shared__ float2 red[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float c1, c2;
  lamb_bias_corrections(step, b1, b2, c1, c2);
  for (long long b = blk_lo + blockIdx.x; b < blk_hi; b += gridDim.x) {
    const int grp = block_group[b];
    if (filtered_out(tab, grp, filter)) continue;          // the same for the whole CTA
    const float wd = tab.wd[grp];
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const int t = block_tensor[b];
    const long long end = tensor_span[2 * t] + tensor_span[2 * t + 1];
    float4 w = *reinterpret_cast<const float4*>(W + i), m = *reinterpret_cast<const float4*>(M + i);
    float4 v = *reinterpret_cast<const float4*>(V + i);
    const float4 g = *reinterpret_cast<const float4*>(G + i);
#define TMPI_LAMB_MOM(c)                                                 \
  {                                                                     \
    const float ge = g.c * inv_k;                                       \
    m.c = b1 * m.c + (1.f - b1) * ge;                                   \
    v.c = b2 * v.c + (1.f - b2) * ge * ge;                              \
  }
    TMPI_LAMB_MOM(x) TMPI_LAMB_MOM(y) TMPI_LAMB_MOM(z) TMPI_LAMB_MOM(w)
#undef TMPI_LAMB_MOM
    *reinterpret_cast<float4*>(M + i) = m;
    *reinterpret_cast<float4*>(V + i) = v;
    float4 r = make_float4(lamb_dir(w.x, m.x, v.x, c1, c2, eps, wd), lamb_dir(w.y, m.y, v.y, c1, c2, eps, wd),
                           lamb_dir(w.z, m.z, v.z, c1, c2, eps, wd), lamb_dir(w.w, m.w, v.w, c1, c2, eps, wd));
    if (i + 4 > end) {                                     // the tensor's last block: zero the padding past its end
      if (i + 0 >= end) { w.x = 0.f; r.x = 0.f; }
      if (i + 1 >= end) { w.y = 0.f; r.y = 0.f; }
      if (i + 2 >= end) { w.z = 0.f; r.z = 0.f; }
      if (i + 3 >= end) { w.w = 0.f; r.w = 0.f; }
    }
    float sw = w.x * w.x + w.y * w.y + w.z * w.z + w.w * w.w;
    float sr = r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
    sw = warp_sum(sw); sr = warp_sum(sr);
    if (lane == 0) red[warp] = make_float2(sw, sr);
    __syncthreads();
    if (threadIdx.x == 0) {
      float2 s = red[0];
#pragma unroll
      for (int k = 1; k < kThreads / 32; ++k) { s.x += red[k].x; s.y += red[k].y; }
      partial[b] = s;
    }
    __syncthreads();                                       // red[] is reused by the next block
  }
}

void lamb_trust(const LambTrustArgs& a, cudaStream_t st) {
  if (a.n_blocks <= 0 || a.n_tensors <= 0) return;
  if (!a.step) throw std::runtime_error("lamb_trust: needs a step counter");
  const int grid = (int)std::min<long long>(a.n_blocks, (long long)sm_count() * 8);
  lamb_moments_kernel<<<grid, kThreads, 0, st>>>((const float*)a.W, (const float*)a.G, (float*)a.M, (float*)a.V,
                                                 (const uint8_t*)a.block_group, a.tab, (const unsigned long long*)a.step, a.b1, a.b2,
                                                 a.eps, a.inv_k, a.filter, (const int*)a.block_tensor, (const long long*)a.tensor_span,
                                                 (float2*)a.partial, 0, a.n_blocks);
  TMPI_CHECK_LAUNCH("lamb_moments");
  // the decay is already inside r: with eta = 1 and no wd, the LARS finalize writes {‖W‖, ‖r‖} and trust = ‖W‖ / ‖r‖
  GroupTable no_wd = a.tab;
  for (float& d : no_wd.wd) d = 0.f;
  lars_finalize_kernel<<<a.n_tensors, kThreads, 0, st>>>((const float2*)a.partial, (const long long*)a.tensor_span,
                                                         (const uint8_t*)a.block_group, no_wd, 1.f, 1.f, (float2*)a.norms,
                                                         (float*)a.trust);
  count_launch(2); TMPI_CHECK_LAUNCH("lars_finalize"); ::tmpi::check_capture(st, "lamb_trust");
}

// ============================================================================ global gradient-norm clipping
// Pass 1 is lars_partial_kernel<false>: partial[b] = Σg² over the real elements of block b.  Pass 2: one CTA sums the n_blocks partials
// in fp64 (every thread a fixed stride of them, then the warps in a fixed order: no atomics, the same result on every run) and writes
// the record the kClip flat_update pass reads.  torch.nn.utils.clip_grad_norm_ semantics: s = min(1, max_norm / (n + 1e-6)).
__global__ void __launch_bounds__(kThreads) clip_finalize_kernel(const float* __restrict__ partial, long long n_blocks, float max_norm,
                                                                 ClipRecord* __restrict__ rec, unsigned long long* __restrict__ skipped) {
  __shared__ double red[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s = 0.0;
  for (long long k = threadIdx.x; k < n_blocks; k += kThreads) s += (double)partial[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = red[0];
    for (int k = 1; k < kThreads / 32; ++k) s += red[k];
    const double n = sqrt(s);
    const bool finite = isfinite(n);
    ClipRecord r;
    r.norm = (float)n;
    r.scale = finite ? (float)fmin(1.0, (double)max_norm / (n + 1e-6)) : 0.f;
    r.finite = finite ? 1 : 0;
    r.pad = 0;
    *rec = r;
    if (!finite) *skipped += 1ull;
  }
}

void grad_clip_norm(const GradClipArgs& a, cudaStream_t st) {
  if (a.n_blocks <= 0) throw std::runtime_error("grad_clip_norm: empty arena");
  if (!(a.max_norm > 0.f)) throw std::runtime_error("grad_clip_norm: max_norm must be positive");
  const int grid = (int)std::min<long long>(a.n_blocks, (long long)sm_count() * 8);
  lars_partial_kernel<false><<<grid, kThreads, 0, st>>>(nullptr, (const float*)a.G, (const int*)a.block_tensor,
                                                        (const long long*)a.tensor_span, (float*)a.partial, 0, a.n_blocks);
  TMPI_CHECK_LAUNCH("clip_partial");
  clip_finalize_kernel<<<1, kThreads, 0, st>>>((const float*)a.partial, a.n_blocks, a.max_norm, (ClipRecord*)a.rec,
                                               (unsigned long long*)a.skipped);
  count_launch(2); TMPI_CHECK_LAUNCH("clip_finalize"); ::tmpi::check_capture(st, "grad_clip_norm");
}

// ============================================================================ fused collectives
__device__ __forceinline__ void local_block_update(const FusedArgs& a, const Hyper& h, long long b, int g) {
  const long long i = b * kArenaBlock + threadIdx.x * 4;
  float* W = region<float>(a.ctx, a.ctx.rank, a.w_off);
  float* U = region<float>(a.ctx, a.ctx.rank, a.u_off);
  const float* G = region<float>(a.ctx, a.ctx.rank, a.g_off);
  float4 w = *reinterpret_cast<const float4*>(W + i), u = *reinterpret_cast<const float4*>(U + i);
  const float4 gg = *reinterpret_cast<const float4*>(G + i);
  Hyper hl = h; hl.inv_k = 1.f;
  sgd4(w, u, gg, hl, a.tab.lr_mult[g], a.tab.wd[g]);
  *reinterpret_cast<float4*>(W + i) = w;
  *reinterpret_cast<float4*>(U + i) = u;
  if (a.h_off >= 0) *reinterpret_cast<uint2*>(region<__nv_bfloat16>(a.ctx, a.ctx.rank, a.h_off) + i) = pack_bf16x4(w);
}

// cast the caller's own gradient block to the bf16 wire region
__device__ __forceinline__ void cast_block_to_wire(const FusedArgs& a, long long b) {
  const long long i = b * kArenaBlock + threadIdx.x * 4;
  const float4 gg = *reinterpret_cast<const float4*>(region<float>(a.ctx, a.ctx.rank, a.g_off) + i);
  *reinterpret_cast<uint2*>(region<__nv_bfloat16>(a.ctx, a.ctx.rank, a.wire_off) + i) = pack_bf16x4(gg);
}

__device__ __forceinline__ float4 gather_grad(const FusedArgs& a, long long i) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (a.wire16) {
    uint2 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) v[p] = ld_sys_u2(region<__nv_bfloat16>(a.ctx, p, a.wire_off) + i);
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) acc = add4(acc, unpack_bf16x4(v[p]));
  } else {
    float4 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) v[p] = ld_sys_f4(region<float>(a.ctx, p, a.g_off) + i);
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) acc = add4(acc, v[p]);     // fixed order → bit-identical on all ranks
  }
  return acc;
}

// ---- one-shot: every rank reduces every block itself
// U arena blocks are in flight per CTA iteration (U x world independent 16 B peer loads per thread) — a single
// load per thread cannot cover the ~2 us NVLink round trip.
template <int U>
__global__ void __launch_bounds__(kThreads) fused_oneshot_sgd_kernel(const FusedArgs a) {
  const Hyper h{*a.lr_ptr, a.mu, a.inv_k, a.nesterov};
  const long long blo = a.lo / kArenaBlock, bhi = a.hi / kArenaBlock;
  if (a.wire16) {
    for (long long b = blo + blockIdx.x; b < bhi; b += gridDim.x)
      if (a.tab.exch[a.block_group[b]]) cast_block_to_wire(a, b);
  }
  block_barrier(a.ctx);                                  // peers' gradients (or wire copies) are complete
  float* W = region<float>(a.ctx, a.ctx.rank, a.w_off);
  float* U_ = region<float>(a.ctx, a.ctx.rank, a.u_off);
  for (long long b0 = blo + blockIdx.x; b0 < bhi; b0 += (long long)gridDim.x * U) {
    float4 gs[U]; int grp[U]; bool ex[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      ex[u] = false; grp[u] = -1;
      if (b < bhi) { grp[u] = a.block_group[b]; ex[u] = a.tab.exch[grp[u]] != 0; }
      if (ex[u]) gs[u] = gather_grad(a, b * kArenaBlock + threadIdx.x * 4);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      if (grp[u] < 0) continue;
      if (!ex[u]) { local_block_update(a, h, b, grp[u]); continue; }
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      float4 w = *reinterpret_cast<const float4*>(W + i), uu = *reinterpret_cast<const float4*>(U_ + i);
      sgd4(w, uu, gs[u], h, a.tab.lr_mult[grp[u]], a.tab.wd[grp[u]]);
      *reinterpret_cast<float4*>(W + i) = w;
      *reinterpret_cast<float4*>(U_ + i) = uu;
      if (a.h_off >= 0) *reinterpret_cast<uint2*>(region<__nv_bfloat16>(a.ctx, a.ctx.rank, a.h_off) + i) = pack_bf16x4(w);
    }
  }
  block_barrier(a.ctx);                                  // nobody overwrites G while a peer still reads it
}

// ---- two-shot: rank r owns a contiguous slice of the range; reduce → update → push W (+H) to every peer
template <int U>
__global__ void __launch_bounds__(kThreads) fused_twoshot_sgd_kernel(const FusedArgs a, int use_nvls) {
  const Hyper h{*a.lr_ptr, a.mu, a.inv_k, a.nesterov};
  const long long blo = a.lo / kArenaBlock, bhi = a.hi / kArenaBlock;
  const long long nb = bhi - blo;
  const long long per = (nb + a.ctx.world - 1) / a.ctx.world;
  const int R = a.ctx.rank, Wn = a.ctx.world;
  if (a.wire16 && !a.pre_reduced) {
    // block b casts, for every owner r, the strip of r's slice that block b of rank r will read
    for (int r = 0; r < Wn; ++r) {
      const long long s0 = blo + r * per, s1 = min(bhi, s0 + per);
      for (long long b = s0 + blockIdx.x; b < s1; b += gridDim.x)
        if (a.tab.exch[a.block_group[b]]) cast_block_to_wire(a, b);
    }
  }
  block_barrier(a.ctx);
  const long long s0 = blo + R * per, s1 = min(bhi, s0 + per);
  float* W = region<float>(a.ctx, R, a.w_off);
  float* U_ = region<float>(a.ctx, R, a.u_off);
  for (long long b0 = s0 + blockIdx.x; b0 < s1; b0 += (long long)gridDim.x * U) {
    float4 gs[U]; int grp[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      grp[u] = -1;
      if (b < s1) { const int g = a.block_group[b]; if (a.tab.exch[g]) grp[u] = g; }
      if (grp[u] >= 0) {
        const long long i = b * kArenaBlock + threadIdx.x * 4;
        if (a.pre_reduced) {
          // the wgrad GEMM epilogues of every rank already red.add-ed their tiles into THIS rank's G (reduce-scatter fused into
          // the producer): consume the sum and clear it for the next step (the closing barrier orders the clear before any
          // peer's next add)
          float* Gl = region<float>(a.ctx, R, a.g_off) + i;
          gs[u] = *reinterpret_cast<const float4*>(Gl);
          *reinterpret_cast<float4*>(Gl) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else if (use_nvls) {
          gs[u] = a.wire16 ? unpack_bf16x4(mc_ld_reduce_bf16x4(reinterpret_cast<char*>(a.ctx.mc_arena) + a.wire_off + i * 2))
                           : mc_ld_reduce_f4(reinterpret_cast<float*>(reinterpret_cast<char*>(a.ctx.mc_arena) + a.g_off) + i);
        } else {
          gs[u] = gather_grad(a, i);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (grp[u] < 0) continue;
      const long long b = b0 + (long long)u * gridDim.x;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      float4 w = *reinterpret_cast<const float4*>(W + i), uu = *reinterpret_cast<const float4*>(U_ + i);
      sgd4(w, uu, gs[u], h, a.tab.lr_mult[grp[u]], a.tab.wd[grp[u]]);
      *reinterpret_cast<float4*>(U_ + i) = uu;
      const uint2 wh = pack_bf16x4(w);
      // owner-keeps-master ships only the bf16 shadow — of plain WEIGHT blocks (group 0).  Biases (and anything else the
      // forward pass reads in fp32 straight from W) always travel as fp32 masters: they are a few KB.
      const bool push_w = a.push_master || a.h_off < 0 || grp[u] != 0;
      if (use_nvls) {
        if (push_w) mc_st_f4(reinterpret_cast<float*>(reinterpret_cast<char*>(a.ctx.mc_arena) + a.w_off) + i, w);
        else *reinterpret_cast<float4*>(W + i) = w;
        if (a.h_off >= 0) mc_st_u2(reinterpret_cast<char*>(a.ctx.mc_arena) + a.h_off + i * 2, wh);
      } else {
#pragma unroll
        for (int p = 0; p < kMaxRanks; ++p) {
          if (p < Wn) {
            if (push_w || p == R) st_f4(region<float>(a.ctx, p, a.w_off) + i, w);
            if (a.h_off >= 0) st_u2(region<__nv_bfloat16>(a.ctx, p, a.h_off) + i, wh);
          }
        }
      }
    }
  }
  // non-exchanged (BN) blocks: every rank updates all of them locally
  for (long long b = blo + blockIdx.x; b < bhi; b += gridDim.x) {
    const int g = a.block_group[b];
    if (!a.tab.exch[g]) local_block_update(a, h, b, g);
  }
  block_barrier(a.ctx);                                  // pushed weights are visible everywhere
}

static int pick_grid(long long nblocks, int max_blocks) {
  long long g = std::min<long long>(nblocks, (long long)max_blocks);
  if (g < 1) g = 1;
  if (g > kMaxCommBlocks) g = kMaxCommBlocks;
  return (int)g;
}

// algo: 0 one-shot, 1 two-shot (P2P), 2 two-shot NVLS
void fused_allreduce_sgd(const FusedArgs& a, int algo, int max_blocks, cudaStream_t st) {
  if (a.lo % kArenaBlock || a.hi % kArenaBlock) throw std::runtime_error("fused_allreduce_sgd: range must be block aligned");
  const long long nb = (a.hi - a.lo) / kArenaBlock;
  if (nb <= 0) return;
  if (algo == 2 && a.ctx.mc_arena == nullptr) throw std::runtime_error("fused_allreduce_sgd: NVLS requested without a multicast mapping");
  const bool wide = a.ctx.world > 4;                     // keep (U x world) peer loads per thread around 8..16
  if (a.pre_reduced && algo == 0) algo = a.ctx.mc_arena ? 2 : 1;     // ownership is the two-shot partition
  if (algo == 0) {
    if (wide) fused_oneshot_sgd_kernel<2><<<pick_grid(nb, max_blocks), kThreads, 0, st>>>(a);
    else fused_oneshot_sgd_kernel<4><<<pick_grid(nb, max_blocks), kThreads, 0, st>>>(a);
  } else {
    const long long per = (nb + a.ctx.world - 1) / a.ctx.world;
    const int nv = algo == 2 ? 1 : 0;
    // loads in flight per thread = U (NVLS: one multimem.ld_reduce per block) or U x world (P2P gather).  The exchange runs
    // next to the backward GEMMs on a few dozen co-resident CTAs, so its throughput is (bytes in flight) / (NVLink round trip):
    // keep 8..16 independent 16-byte loads per thread outstanding.  TMPI_FUSED_U overrides (2, 4 or 8).
    static const int u_env = [] { const char* e = getenv("TMPI_FUSED_U"); return e ? atoi(e) : 0; }();
    int U = nv ? 8 : (a.ctx.world <= 2 ? 8 : (wide ? 2 : 4));
    if (u_env == 2 || u_env == 4 || u_env == 8) U = u_env;
    if (U == 8) fused_twoshot_sgd_kernel<8><<<pick_grid(per, max_blocks), kThreads, 0, st>>>(a, nv);
    else if (U == 4) fused_twoshot_sgd_kernel<4><<<pick_grid(per, max_blocks), kThreads, 0, st>>>(a, nv);
    else fused_twoshot_sgd_kernel<2><<<pick_grid(per, max_blocks), kThreads, 0, st>>>(a, nv);
  }
  count_launch(); TMPI_CHECK_LAUNCH("fused_allreduce_sgd"); ::tmpi::check_capture(st, "fused_allreduce_sgd");
}

// every rank pushes the fp32 master of the slice it owns (two-shot partition of [lo, hi)) to all peers: re-synchronises W after
// steps that ran with push_master = 0 (before a checkpoint / weight averaging / anything that reads W on a non-owner)
__global__ void __launch_bounds__(kThreads) push_master_kernel(const FusedArgs a) {
  const long long blo = a.lo / kArenaBlock, bhi = a.hi / kArenaBlock;
  const long long per = (bhi - blo + a.ctx.world - 1) / a.ctx.world;
  const int R = a.ctx.rank;
  const long long s0 = blo + R * per, s1 = min(bhi, s0 + per);
  block_barrier(a.ctx);
  const float* W = region<float>(a.ctx, R, a.w_off);
  for (long long b = s0 + blockIdx.x; b < s1; b += gridDim.x) {
    if (!a.tab.exch[a.block_group[b]]) continue;
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const float4 w = *reinterpret_cast<const float4*>(W + i);
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p)
      if (p < a.ctx.world && p != R) st_f4(region<float>(a.ctx, p, a.w_off) + i, w);
  }
  block_barrier(a.ctx);
}
void push_master_slices(const FusedArgs& a, int max_blocks, cudaStream_t st) {
  if (a.lo % kArenaBlock || a.hi % kArenaBlock) throw std::runtime_error("push_master_slices: range must be block aligned");
  const long long nb = (a.hi - a.lo) / kArenaBlock;
  if (nb <= 0) return;
  const long long per = (nb + a.ctx.world - 1) / a.ctx.world;
  push_master_kernel<<<pick_grid(per, max_blocks), kThreads, 0, st>>>(a);
  count_launch(); TMPI_CHECK_LAUNCH("push_master_slices"); ::tmpi::check_capture(st, "push_master_slices");
}

// ============================================================================ plain flat allreduce (sum * scale) src region → dst region
__global__ void __launch_bounds__(kThreads) allreduce_oneshot_kernel(const ReduceArgs a) {
  const long long blo = a.lo / kArenaBlock, bhi = a.hi / kArenaBlock;
  block_barrier(a.ctx);
  float* D = region<float>(a.ctx, a.ctx.rank, a.dst_off);
  for (long long b = blo + blockIdx.x; b < bhi; b += gridDim.x) {
    if (a.skip_local_groups && !a.tab.exch[a.block_group[b]]) continue;
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    float4 v[kMaxRanks];
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) v[p] = ld_sys_f4(region<float>(a.ctx, p, a.src_off) + i);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) acc = add4(acc, v[p]);
    acc.x *= a.scale; acc.y *= a.scale; acc.z *= a.scale; acc.w *= a.scale;
    *reinterpret_cast<float4*>(D + i) = acc;
    if (a.h_off >= 0) *reinterpret_cast<uint2*>(region<__nv_bfloat16>(a.ctx, a.ctx.rank, a.h_off) + i) = pack_bf16x4(acc);
  }
  block_barrier(a.ctx);
}

__global__ void __launch_bounds__(kThreads) allreduce_twoshot_kernel(const ReduceArgs a, int use_nvls) {
  const long long blo = a.lo / kArenaBlock, bhi = a.hi / kArenaBlock;
  const long long per = (bhi - blo + a.ctx.world - 1) / a.ctx.world;
  const long long s0 = blo + a.ctx.rank * per, s1 = min(bhi, s0 + per);
  block_barrier(a.ctx);
  for (long long b = s0 + blockIdx.x; b < s1; b += gridDim.x) {
    if (a.skip_local_groups && !a.tab.exch[a.block_group[b]]) continue;
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (use_nvls) {
      acc = mc_ld_reduce_f4(reinterpret_cast<float*>(reinterpret_cast<char*>(a.ctx.mc_arena) + a.src_off) + i);
    } else {
      float4 v[kMaxRanks];
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) v[p] = ld_sys_f4(region<float>(a.ctx, p, a.src_off) + i);
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p) if (p < a.ctx.world) acc = add4(acc, v[p]);
    }
    acc.x *= a.scale; acc.y *= a.scale; acc.z *= a.scale; acc.w *= a.scale;
    const uint2 hh = pack_bf16x4(acc);
    if (use_nvls) {
      mc_st_f4(reinterpret_cast<float*>(reinterpret_cast<char*>(a.ctx.mc_arena) + a.dst_off) + i, acc);
      if (a.h_off >= 0) mc_st_u2(reinterpret_cast<char*>(a.ctx.mc_arena) + a.h_off + i * 2, hh);
    } else {
#pragma unroll
      for (int p = 0; p < kMaxRanks; ++p) {
        if (p < a.ctx.world) {
          st_f4(region<float>(a.ctx, p, a.dst_off) + i, acc);
          if (a.h_off >= 0) st_u2(region<__nv_bfloat16>(a.ctx, p, a.h_off) + i, hh);
        }
      }
    }
  }
  block_barrier(a.ctx);
}

void allreduce_flat(const ReduceArgs& a, int algo, int max_blocks, cudaStream_t st) {
  if (a.lo % kArenaBlock || a.hi % kArenaBlock) throw std::runtime_error("allreduce_flat: range must be block aligned");
  const long long nb = (a.hi - a.lo) / kArenaBlock;
  if (nb <= 0) return;
  if (algo == 0 && a.src_off == a.dst_off) throw std::runtime_error("allreduce_flat: one-shot cannot run in place");
  if (algo == 2 && a.ctx.mc_arena == nullptr) throw std::runtime_error("allreduce_flat: NVLS requested without a multicast mapping");
  if (algo == 0) allreduce_oneshot_kernel<<<pick_grid(nb, max_blocks), kThreads, 0, st>>>(a);
  else allreduce_twoshot_kernel<<<pick_grid((nb + a.ctx.world - 1) / a.ctx.world, max_blocks), kThreads, 0, st>>>(a, algo == 2 ? 1 : 0);
  count_launch(); TMPI_CHECK_LAUNCH("allreduce_flat"); ::tmpi::check_capture(st, "allreduce_flat");
}

// standalone device barrier (tests / stream alignment)
__global__ void barrier_kernel(const CommCtx c) { block_barrier(c); }
void device_barrier(const CommCtx& c, cudaStream_t st) {
  barrier_kernel<<<1, 32, 0, st>>>(c);
  count_launch(); TMPI_CHECK_LAUNCH("device_barrier"); ::tmpi::check_capture(st, "device_barrier");
}

// ============================================================================ device-side protocol words
// The 4 KiB tail of every rank's signal pad (peer-mapped like the rest of it) holds the words of the asynchronous rules:
//   [0] EASGD next ticket   [1] EASGD now serving   [2] EASGD exchanges served
//   [32 + 2*src], [33 + 2*src]   GOSGD inbox slot of sender `src`: {sequence number, push-sum weight bits}
//   [96 + dst]                   GOSGD acknowledgements: receiver `dst` writes the sequence number it merged (on the SENDER's pad)
__device__ __forceinline__ uint32_t* proto_words(const CommCtx& c, int p) {
  return c.sig[p] + (size_t)kMaxCommBlocks * kMaxRanks + kMaxCommBlocks;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_sys_v4(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ============================================================================ EASGD elastic exchange (worker side, center over NVLink)
// Reference: the server serialises workers with a blocking MPI recv and both sides broadcast their full model
// (easgd_server.py:152-164, lib/exchanger.py:214-261).  Here the workers queue on the DEVICE: a ticket lock in the center
// rank's signal pad (atom.acq_rel.sys take, st.release.sys hand-over) brackets ONE kernel on the worker's GPU that reads the
// center over NVLink, computes d = α(w − c) and updates both sides.  Three stream-ordered launches (acquire → elastic →
// release) instead of a grid-wide sync inside one kernel: no co-residency requirement, graph-capturable, and the host never
// waits.  lockfree = 1: no lock at all — the center update is a vector red.add (commutative, so no update can be lost) and
// the workers run fully concurrently.
__global__ void ticket_acquire_kernel(CommCtx c, int owner, uint32_t* local) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t* lock = proto_words(c, owner);
  uint32_t my;
  asm volatile("atom.acq_rel.sys.global.add.u32 %0, [%1], 1;" : "=r"(my) : "l"(lock) : "memory");
  local[0] = my;
  const long long t0 = clock64();
  while (ld_acquire_sys_u32(lock + 1) != my) {
    if (clock64() - t0 > c.spin_limit) __trap();
    __nanosleep(200);
  }
}
__global__ void ticket_release_kernel(CommCtx c, int owner, uint32_t* local) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t* lock = proto_words(c, owner);
  __threadfence_system();
  asm volatile("red.relaxed.sys.global.add.u32 [%0], 1;" ::"l"(lock + 2) : "memory");
  st_release_sys_u32(lock + 1, local[0] + 1u);
}

// U arena blocks in flight per CTA iteration: U independent 16 B NVLink loads per thread cover the ~2 us round trip
template <int U>
__global__ void __launch_bounds__(kThreads) easgd_elastic_kernel(float* __restrict__ w, __nv_bfloat16* __restrict__ h, float* c /*peer*/,
                                                                 float alpha, long long nblk, int lockfree) {
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)gridDim.x * U) {
    float4 cv[U], wv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      if (b < nblk) {
        const long long i = b * kArenaBlock + threadIdx.x * 4;
        cv[u] = ld_sys_f4(c + i);
        wv[u] = *reinterpret_cast<const float4*>(w + i);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      const float4 d = make_float4(alpha * (wv[u].x - cv[u].x), alpha * (wv[u].y - cv[u].y), alpha * (wv[u].z - cv[u].z),
                                   alpha * (wv[u].w - cv[u].w));
      wv[u].x -= d.x; wv[u].y -= d.y; wv[u].z -= d.z; wv[u].w -= d.w;
      *reinterpret_cast<float4*>(w + i) = wv[u];
      if (h) *reinterpret_cast<uint2*>(h + i) = pack_bf16x4(wv[u]);
      if (lockfree) red_add_sys_v4(c + i, d);
      else st_f4(c + i, add4(cv[u], d));
    }
  }
  __threadfence_system();
}

void easgd_elastic(void* w, void* h, void* center, float alpha, long long n, int max_blocks, int lockfree, cudaStream_t st) {
  if (n % kArenaBlock) throw std::runtime_error("easgd_elastic: n must be block aligned");
  const long long nb = n / kArenaBlock;
  if (nb <= 0) return;
  easgd_elastic_kernel<4><<<pick_grid((nb + 3) / 4, max_blocks), kThreads, 0, st>>>((float*)w, (__nv_bfloat16*)h, (float*)center, alpha, nb,
                                                                                lockfree);
  count_launch(); TMPI_CHECK_LAUNCH("easgd_elastic"); ::tmpi::check_capture(st, "easgd_elastic");
}
void ticket_acquire(const CommCtx& c, int owner, void* local_state, cudaStream_t st) {
  ticket_acquire_kernel<<<1, 32, 0, st>>>(c, owner, (uint32_t*)local_state);
  count_launch(); TMPI_CHECK_LAUNCH("ticket_acquire"); ::tmpi::check_capture(st, "ticket_acquire");
}
void ticket_release(const CommCtx& c, int owner, void* local_state, cudaStream_t st) {
  ticket_release_kernel<<<1, 32, 0, st>>>(c, owner, (uint32_t*)local_state);
  count_launch(); TMPI_CHECK_LAUNCH("ticket_release"); ::tmpi::check_capture(st, "ticket_release");
}

// dst = src (+ bf16 shadow) over peer memory: EASGD copy_to_local, GOSGD snapshot.  `gate` (optional, device word): the copy
// runs only when *gate != 0 (GOSGD: the push was admitted by gosgd_push_begin).
template <int U>
__global__ void __launch_bounds__(kThreads) copy_flat_kernel(float* dst, __nv_bfloat16* dst_h, const float* src, long long nblk,
                                                             const uint32_t* __restrict__ gate) {
  if (gate && *gate == 0u) return;
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)gridDim.x * U) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      if (b < nblk) v[u] = ld_sys_f4(src + b * kArenaBlock + threadIdx.x * 4);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long b = b0 + (long long)u * gridDim.x;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      st_f4(dst + i, v[u]);
      if (dst_h) *reinterpret_cast<uint2*>(dst_h + i) = pack_bf16x4(v[u]);
    }
  }
  __threadfence_system();
}
void copy_flat(void* dst, void* dst_h, const void* src, long long n, int max_blocks, const void* gate, cudaStream_t st) {
  if (n % kArenaBlock) throw std::runtime_error("copy_flat: n must be block aligned");
  const long long nb = n / kArenaBlock;
  if (nb <= 0) return;
  copy_flat_kernel<4><<<pick_grid((nb + 3) / 4, max_blocks), kThreads, 0, st>>>((float*)dst, (__nv_bfloat16*)dst_h, (const float*)src, nb,
                                                                            (const uint32_t*)gate);
  count_launch(); TMPI_CHECK_LAUNCH("copy_flat"); ::tmpi::check_capture(st, "copy_flat");
}

// ============================================================================ model EMA (utils/opt.py: ModelEma)
// state: uint64 {u, n_averaged, mode}.  ema_advance_kernel counts one more optimizer update and writes what ema_update_kernel does
// after it: nothing, E ← W, or E ← d·E + (1 − d)·W.  every, warmup, d and 1 − d are launch arguments, fixed when a step is captured;
// the counters live in device memory, so a captured CUDA graph keeps counting.
__global__ void ema_advance_kernel(unsigned long long* __restrict__ state, long long every, long long warmup) {
  const unsigned long long u = state[0] + 1ull;
  unsigned long long n = state[1], mode = EMA_SKIP;
  if (u % (unsigned long long)every == 0ull) {
    if (n == 0ull || u <= (unsigned long long)warmup) {
      n = 1ull; mode = EMA_COPY;
    } else {
      n += 1ull; mode = EMA_AVERAGE;
    }
  }
  state[0] = u; state[1] = n; state[2] = mode;
}

// fp32(d)·e + fp32(1 − d)·w with each product and the sum rounded once: mul.rn / add.rn are never contracted into an FMA, and without
// .ftz they keep subnormals (the build's --use_fast_math would flush them in __fmul_rn), so the result is bit-equal to torch's fp32
// expression d * e + (1 - d) * w on the CPU.
__device__ __forceinline__ float ema_avg(float e, float w, float d, float omd) {
  float a, b, r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(a) : "f"(d), "f"(e));
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(b) : "f"(omd), "f"(w));
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

constexpr int kEmaUnroll = 4;            // arena blocks in flight per CTA iteration
constexpr int kEmaSegCtas = 16;          // CTAs that walk the statistics segments

// CTAs [0, arena_ctas) walk the arena blocks of W / E with float4 loads and stores, the others the statistics segments {E part, the
// layer's tensor}.  A skip step returns before it touches memory; a copy step does not read E.
__global__ void __launch_bounds__(kThreads) ema_update_kernel(const float* __restrict__ W, float* __restrict__ E, long long nblk,
                                                              int arena_ctas, const EmaSegment* __restrict__ segs, int n_segs,
                                                              const unsigned long long* __restrict__ state, float d, float omd) {
  const unsigned long long mode = state[2];
  if (mode == EMA_SKIP) return;
  const bool copy = mode == EMA_COPY;
  if ((int)blockIdx.x >= arena_ctas) {
    for (int s = (int)blockIdx.x - arena_ctas; s < n_segs; s += (int)gridDim.x - arena_ctas) {
      const EmaSegment g = segs[s];
      for (long long i = threadIdx.x; i < g.n; i += kThreads) g.dst[i] = copy ? g.src[i] : ema_avg(g.dst[i], g.src[i], d, omd);
    }
    return;
  }
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)arena_ctas * kEmaUnroll) {
    float4 w[kEmaUnroll], e[kEmaUnroll];
#pragma unroll
    for (int u = 0; u < kEmaUnroll; ++u) {
      const long long b = b0 + (long long)u * arena_ctas;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      w[u] = *reinterpret_cast<const float4*>(W + i);
      if (!copy) e[u] = *reinterpret_cast<const float4*>(E + i);
    }
#pragma unroll
    for (int u = 0; u < kEmaUnroll; ++u) {
      const long long b = b0 + (long long)u * arena_ctas;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      const float4 o = copy ? w[u]
                            : make_float4(ema_avg(e[u].x, w[u].x, d, omd), ema_avg(e[u].y, w[u].y, d, omd),
                                          ema_avg(e[u].z, w[u].z, d, omd), ema_avg(e[u].w, w[u].w, d, omd));
      *reinterpret_cast<float4*>(E + i) = o;
    }
  }
}

// W ↔ E, H ← bf16-RN(new W) when there is a shadow, and every segment's two parts exchanged: applying it twice is the identity.
__global__ void __launch_bounds__(kThreads) ema_swap_kernel(float* __restrict__ W, float* __restrict__ E, __nv_bfloat16* __restrict__ H,
                                                            long long nblk, int arena_ctas, const EmaSegment* __restrict__ segs,
                                                            int n_segs) {
  if ((int)blockIdx.x >= arena_ctas) {
    for (int s = (int)blockIdx.x - arena_ctas; s < n_segs; s += (int)gridDim.x - arena_ctas) {
      const EmaSegment g = segs[s];
      for (long long i = threadIdx.x; i < g.n; i += kThreads) {
        const float a = g.dst[i];
        g.dst[i] = g.src[i];
        g.src[i] = a;
      }
    }
    return;
  }
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)arena_ctas * kEmaUnroll) {
    float4 w[kEmaUnroll], e[kEmaUnroll];
#pragma unroll
    for (int u = 0; u < kEmaUnroll; ++u) {
      const long long b = b0 + (long long)u * arena_ctas;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      w[u] = *reinterpret_cast<const float4*>(W + i);
      e[u] = *reinterpret_cast<const float4*>(E + i);
    }
#pragma unroll
    for (int u = 0; u < kEmaUnroll; ++u) {
      const long long b = b0 + (long long)u * arena_ctas;
      if (b >= nblk) continue;
      const long long i = b * kArenaBlock + threadIdx.x * 4;
      *reinterpret_cast<float4*>(W + i) = e[u];
      *reinterpret_cast<float4*>(E + i) = w[u];
      if (H) *reinterpret_cast<uint2*>(H + i) = pack_bf16x4(e[u]);
    }
  }
}

static void ema_grid(const EmaArgs& a, const char* name, long long& nb, int& arena_ctas, int& grid) {
  if (a.n <= 0 || a.n % kArenaBlock) throw std::runtime_error(std::string(name) + ": the arena size must be a positive multiple of the block");
  if (!a.W || !a.E || (a.n_segs > 0 && !a.segs) || a.n_segs < 0) throw std::runtime_error(std::string(name) + ": missing buffers");
  nb = a.n / kArenaBlock;
  arena_ctas = (int)std::min<long long>((nb + kEmaUnroll - 1) / kEmaUnroll, (long long)sm_count() * 8);
  grid = arena_ctas + std::min(a.n_segs, kEmaSegCtas);
}

void ema_advance(void* state, long long every, long long warmup, cudaStream_t st) {
  if (!state || every < 1 || warmup < 0) throw std::runtime_error("ema_advance: needs the state words, every >= 1 and warmup >= 0");
  ema_advance_kernel<<<1, 1, 0, st>>>((unsigned long long*)state, every, warmup);
  count_launch(); TMPI_CHECK_LAUNCH("ema_advance"); ::tmpi::check_capture(st, "ema_advance");
}

void ema_update(const EmaArgs& a, cudaStream_t st) {
  if (!a.state) throw std::runtime_error("ema_update: needs the state words");
  long long nb; int arena_ctas, grid;
  ema_grid(a, "ema_update", nb, arena_ctas, grid);
  ema_update_kernel<<<grid, kThreads, 0, st>>>((const float*)a.W, (float*)a.E, nb, arena_ctas, (const EmaSegment*)a.segs, a.n_segs,
                                               (const unsigned long long*)a.state, a.decay, a.one_minus_decay);
  count_launch(); TMPI_CHECK_LAUNCH("ema_update"); ::tmpi::check_capture(st, "ema_update");
}

void ema_swap(const EmaArgs& a, cudaStream_t st) {
  long long nb; int arena_ctas, grid;
  ema_grid(a, "ema_swap", nb, arena_ctas, grid);
  ema_swap_kernel<<<grid, kThreads, 0, st>>>((float*)a.W, (float*)a.E, (__nv_bfloat16*)a.H, nb, arena_ctas, (const EmaSegment*)a.segs,
                                             a.n_segs);
  count_launch(); TMPI_CHECK_LAUNCH("ema_swap"); ::tmpi::check_capture(st, "ema_swap");
}

// ============================================================================ sharpness-aware minimization (utils/opt.py: Sam)
// The products and sums below use mul.rn / add.rn / rcp.rn without .ftz (the build's --use_fast_math would flush subnormals in
// __fmul_rn and friends) and are never contracted into an FMA, so each is rounded once, as torch's fp32 CPU expressions are.
__device__ __forceinline__ float mul_rn(float a, float b) { float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float add_rn(float a, float b) { float r; asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }

// ASAM's pass 1: partial[b] = Σ(w·g)² over the real elements of block b, w·g rounded once; the reduction of lars_partial_kernel (no
// atomics, the result does not depend on the grid).  SAM's Σg² is lars_partial_kernel<false>.
__global__ void __launch_bounds__(kThreads) sam_partial_wg_kernel(const float* __restrict__ W, const float* __restrict__ G,
                                                                  const int* __restrict__ block_tensor,
                                                                  const long long* __restrict__ tensor_span, float* __restrict__ partial,
                                                                  long long n_blocks) {
  __shared__ float red[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const int t = block_tensor[b];
    const long long end = tensor_span[2 * t] + tensor_span[2 * t + 1];
    const float4 w = *reinterpret_cast<const float4*>(W + i), g = *reinterpret_cast<const float4*>(G + i);
    float4 p = make_float4(mul_rn(w.x, g.x), mul_rn(w.y, g.y), mul_rn(w.z, g.z), mul_rn(w.w, g.w));
    if (i + 4 > end) {                                   // the tensor's last block: zero the padding past its end
      if (i + 0 >= end) p.x = 0.f;
      if (i + 1 >= end) p.y = 0.f;
      if (i + 2 >= end) p.z = 0.f;
      if (i + 3 >= end) p.w = 0.f;
    }
    float s = warp_sum(p.x * p.x + p.y * p.y + p.z * p.z + p.w * p.w);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      s = red[0];
#pragma unroll
      for (int k = 1; k < kThreads / 32; ++k) s += red[k];
      partial[b] = s;
    }
    __syncthreads();                                     // red[] is reused by the next block
  }
}

// Pass 2: one CTA sums the n_blocks partials in fp64 in a fixed order (as clip_finalize_kernel) and writes the record:
// n = fp32(sqrt(Σ)), s = fp32(1 / fp32(n + 1e-12)) · fp32(rho), which is how torch evaluates rho / (grad_norm + 1e-12) on an fp32
// tensor (Tensor.__rtruediv__ is reciprocal() * other), and finite = n is neither NaN nor Inf.
__global__ void __launch_bounds__(kThreads) sam_finalize_kernel(const float* __restrict__ partial, long long n_blocks, float rho,
                                                                ClipRecord* __restrict__ rec) {
  __shared__ double red[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s = 0.0;
  for (long long k = threadIdx.x; k < n_blocks; k += kThreads) s += (double)partial[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = red[0];
    for (int k = 1; k < kThreads / 32; ++k) s += red[k];
    const float n = (float)sqrt(s);
    const bool finite = isfinite(n);
    float r;
    asm("rcp.rn.f32 %0, %1;" : "=f"(r) : "f"(add_rn(n, 1e-12f)));
    ClipRecord out;
    out.norm = n;
    out.scale = finite ? mul_rn(r, rho) : 0.f;
    out.finite = finite ? 1 : 0;
    out.pad = 0;
    *rec = out;
  }
}

// The ascent step, one pass: P ← W, then on the real elements W ← W + e with e = g·s (SAM) or ((w·w)·g)·s (ASAM), and H ← bf16-RN(W)
// when there is a shadow.  A non-finite record only copies W into P.  Reads W and G, writes P, W and H: 18 B per element.
template <bool kAdaptive>
__global__ void __launch_bounds__(kThreads) sam_perturb_kernel(float* __restrict__ W, const float* __restrict__ G, float* __restrict__ P,
                                                               __nv_bfloat16* __restrict__ H, const int* __restrict__ block_tensor,
                                                               const long long* __restrict__ tensor_span, long long n_blocks,
                                                               const ClipRecord* __restrict__ rec) {
  const float s = rec->scale;
  const bool finite = rec->finite != 0;
  for (long long b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const float4 w = *reinterpret_cast<const float4*>(W + i);
    *reinterpret_cast<float4*>(P + i) = w;
    if (!finite) continue;
    const int t = block_tensor[b];
    const long long end = tensor_span[2 * t] + tensor_span[2 * t + 1];
    const float4 g = *reinterpret_cast<const float4*>(G + i);
    float o[4] = {w.x, w.y, w.z, w.w};
    const float wv[4] = {w.x, w.y, w.z, w.w}, gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k >= end) continue;                        // padding past the tensor's end stays as it is
      const float d = kAdaptive ? mul_rn(mul_rn(wv[k], wv[k]), gv[k]) : gv[k];
      o[k] = add_rn(wv[k], mul_rn(d, s));
    }
    const float4 nw = make_float4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<float4*>(W + i) = nw;
    if (H) *reinterpret_cast<uint2*>(H + i) = pack_bf16x4(nw);
  }
}

// The restore: W ← P, H ← bf16-RN(P).  Reads P, writes W and H: 10 B per element.
__global__ void __launch_bounds__(kThreads) sam_restore_kernel(float* __restrict__ W, const float* __restrict__ P, __nv_bfloat16* __restrict__ H,
                                                               long long n_blocks) {
  for (long long b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const long long i = b * kArenaBlock + threadIdx.x * 4;
    const float4 p = *reinterpret_cast<const float4*>(P + i);
    *reinterpret_cast<float4*>(W + i) = p;
    if (H) *reinterpret_cast<uint2*>(H + i) = pack_bf16x4(p);
  }
}

static int sam_grid(const SamArgs& a, const char* name, bool ok) {
  if (a.n_blocks <= 0) throw std::runtime_error(std::string(name) + ": empty arena");
  if (!a.W || !ok) throw std::runtime_error(std::string(name) + ": missing buffers");
  return (int)std::min<long long>(a.n_blocks, (long long)sm_count() * 8);
}

void sam_norm(const SamArgs& a, cudaStream_t st) {
  const int grid = sam_grid(a, "sam_norm", a.G && a.partial && a.rec && a.block_tensor && a.tensor_span);
  if (!(a.rho > 0.f) || !std::isfinite(a.rho)) throw std::runtime_error("sam_norm: rho must be finite and positive");
  if (a.adaptive)
    sam_partial_wg_kernel<<<grid, kThreads, 0, st>>>((const float*)a.W, (const float*)a.G, (const int*)a.block_tensor,
                                                     (const long long*)a.tensor_span, (float*)a.partial, a.n_blocks);
  else
    lars_partial_kernel<false><<<grid, kThreads, 0, st>>>(nullptr, (const float*)a.G, (const int*)a.block_tensor,
                                                          (const long long*)a.tensor_span, (float*)a.partial, 0, a.n_blocks);
  TMPI_CHECK_LAUNCH("sam_partial");
  sam_finalize_kernel<<<1, kThreads, 0, st>>>((const float*)a.partial, a.n_blocks, a.rho, (ClipRecord*)a.rec);
  count_launch(2); TMPI_CHECK_LAUNCH("sam_finalize"); ::tmpi::check_capture(st, "sam_norm");
}

void sam_perturb(const SamArgs& a, cudaStream_t st) {
  const int grid = sam_grid(a, "sam_perturb", a.G && a.P && a.rec && a.block_tensor && a.tensor_span);
  auto k = a.adaptive ? sam_perturb_kernel<true> : sam_perturb_kernel<false>;
  k<<<grid, kThreads, 0, st>>>((float*)a.W, (const float*)a.G, (float*)a.P, (__nv_bfloat16*)a.H, (const int*)a.block_tensor,
                               (const long long*)a.tensor_span, a.n_blocks, (const ClipRecord*)a.rec);
  count_launch(); TMPI_CHECK_LAUNCH("sam_perturb"); ::tmpi::check_capture(st, "sam_perturb");
}

void sam_restore(const SamArgs& a, cudaStream_t st) {
  const int grid = sam_grid(a, "sam_restore", a.P != nullptr);
  sam_restore_kernel<<<grid, kThreads, 0, st>>>((float*)a.W, (const float*)a.P, (__nv_bfloat16*)a.H, a.n_blocks);
  count_launch(); TMPI_CHECK_LAUNCH("sam_restore"); ::tmpi::check_capture(st, "sam_restore");
}

// ============================================================================ GOSGD:  w ← (a_self·w + a_src·b) / (a_self + a_src)
// Host-driven form (CPU-mirrored semantics, tests): coefficients passed by value, `b` = local mailbox or a peer's snapshot.
template <int U>
__global__ void __launch_bounds__(kThreads) gosgd_merge_kernel(float* __restrict__ w, __nv_bfloat16* __restrict__ h, const float* b,
                                                               float ca, float cb, long long nblk) {
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)gridDim.x * U) {
    float4 bv[U], wv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long blk = b0 + (long long)u * gridDim.x;
      if (blk < nblk) {
        const long long i = blk * kArenaBlock + threadIdx.x * 4;
        bv[u] = ld_sys_f4(b + i);
        wv[u] = *reinterpret_cast<const float4*>(w + i);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long blk = b0 + (long long)u * gridDim.x;
      if (blk >= nblk) continue;
      const long long i = blk * kArenaBlock + threadIdx.x * 4;
      float4 o;
      o.x = ca * wv[u].x + cb * bv[u].x; o.y = ca * wv[u].y + cb * bv[u].y; o.z = ca * wv[u].z + cb * bv[u].z; o.w = ca * wv[u].w + cb * bv[u].w;
      *reinterpret_cast<float4*>(w + i) = o;
      if (h) *reinterpret_cast<uint2*>(h + i) = pack_bf16x4(o);
    }
  }
}
void gosgd_merge(void* w, void* h, const void* b, float a_self, float a_src, long long n, int max_blocks, cudaStream_t st) {
  if (n % kArenaBlock) throw std::runtime_error("gosgd_merge: n must be block aligned");
  const long long nb = n / kArenaBlock;
  if (nb <= 0) return;
  const float inv = 1.f / (a_self + a_src);
  gosgd_merge_kernel<4><<<pick_grid((nb + 3) / 4, max_blocks), kThreads, 0, st>>>((float*)w, (__nv_bfloat16*)h, (const float*)b, a_self * inv,
                                                                              a_src * inv, nb);
  count_launch(); TMPI_CHECK_LAUNCH("gosgd_merge"); ::tmpi::check_capture(st, "gosgd_merge");
}

// ---- device-side gossip protocol (no host message, no stream synchronisation on the path; ref lib/exchanger.py:484-584
//      blocks the sender inside ncclBcast until the receiver joins).
// Local state words (uint32 / float bits, one small device buffer per rank):
//   [0] alpha (float)  [1] push admitted flag  [2] last dest (+1; 0 = none)  [3] sequence of the outstanding push
//   [4] pushes done    [5] pushes skipped (previous snapshot still being pulled)  [6] merges done
//   [8] merge: chosen src (+1; 0 = none)  [9] merge: src's sequence  [10] ca (float)  [11] cb (float)
//   [16 + src] last sequence merged from src        [32 + dst] sequence counter of pushes sent to dst
__global__ void gosgd_push_begin_kernel(CommCtx c, uint32_t* st) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t ok = 1u;
  const uint32_t last = st[2];
  if (last != 0u) {
    // my snapshot region is single-buffered: the previous receiver must have pulled it (it acknowledges on MY pad)
    const uint32_t acked = ld_acquire_sys_u32(proto_words(c, c.rank) + 96 + (last - 1u));
    if (acked != st[3]) ok = 0u;
  }
  st[1] = ok;
  if (ok) {
    float a = __uint_as_float(st[0]) * 0.5f;                    // push-sum: keep half, ship half
    st[0] = __float_as_uint(a);
  } else {
    st[5] += 1u;
  }
}
__global__ void gosgd_push_end_kernel(CommCtx c, uint32_t* st, int dest) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (st[1] == 0u) return;
  __threadfence_system();                                       // the snapshot (copy_flat before me on this stream) is visible
  const uint32_t seq = st[32 + dest] + 1u;
  st[32 + dest] = seq; st[2] = (uint32_t)dest + 1u; st[3] = seq; st[4] += 1u;
  uint32_t* inbox = proto_words(c, dest) + 32 + 2 * c.rank;
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(inbox + 1), "r"(st[0]) : "memory");     // shipped weight = what I kept
  st_release_sys_u32(inbox, seq);
}
// receiver: pick at most one pending push (lowest rank first, fair enough for p << 1)
__global__ void gosgd_poll_kernel(CommCtx c, uint32_t* st) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  st[8] = 0u;
  const uint32_t* inbox = proto_words(c, c.rank) + 32;
  for (int s = 0; s < c.world; ++s) {
    if (s == c.rank) continue;
    const uint32_t seq = ld_acquire_sys_u32(inbox + 2 * s);
    if (seq != st[16 + s]) {
      const float a_src = __uint_as_float(ld_acquire_sys_u32(inbox + 2 * s + 1));
      const float a_self = __uint_as_float(st[0]);
      const float inv = 1.f / (a_self + a_src);
      st[8] = (uint32_t)s + 1u; st[9] = seq;
      st[10] = __float_as_uint(a_self * inv); st[11] = __float_as_uint(a_src * inv);
      st[0] = __float_as_uint(a_self + a_src);
      return;
    }
  }
}
template <int U>
__global__ void __launch_bounds__(kThreads) gosgd_pull_merge_kernel(CommCtx c, const uint32_t* __restrict__ st, long long w_off, long long h_off,
                                                                    long long snap_off, long long nblk) {
  const uint32_t chosen = st[8];
  if (chosen == 0u) return;
  const int src = (int)chosen - 1;
  const float ca = __uint_as_float(st[10]), cb = __uint_as_float(st[11]);
  float* w = region<float>(c, c.rank, w_off);
  __nv_bfloat16* h = h_off >= 0 ? region<__nv_bfloat16>(c, c.rank, h_off) : nullptr;
  const float* b = region<float>(c, src, snap_off);
  for (long long b0 = blockIdx.x; b0 < nblk; b0 += (long long)gridDim.x * U) {
    float4 bv[U], wv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long blk = b0 + (long long)u * gridDim.x;
      if (blk < nblk) {
        const long long i = blk * kArenaBlock + threadIdx.x * 4;
        bv[u] = ld_sys_f4(b + i);
        wv[u] = *reinterpret_cast<const float4*>(w + i);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long blk = b0 + (long long)u * gridDim.x;
      if (blk >= nblk) continue;
      const long long i = blk * kArenaBlock + threadIdx.x * 4;
      float4 o;
      o.x = ca * wv[u].x + cb * bv[u].x; o.y = ca * wv[u].y + cb * bv[u].y; o.z = ca * wv[u].z + cb * bv[u].z; o.w = ca * wv[u].w + cb * bv[u].w;
      *reinterpret_cast<float4*>(w + i) = o;
      if (h) *reinterpret_cast<uint2*>(h + i) = pack_bf16x4(o);
    }
  }
}
__global__ void gosgd_ack_kernel(CommCtx c, uint32_t* st) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const uint32_t chosen = st[8];
  if (chosen == 0u) return;
  const int src = (int)chosen - 1;
  st[16 + src] = st[9]; st[6] += 1u; st[8] = 0u;
  __threadfence_system();
  st_release_sys_u32(proto_words(c, src) + 96 + c.rank, st[9]);       // the sender may overwrite its snapshot now
}

void gosgd_push(const CommCtx& c, void* state, int dest, long long w_off, long long snap_off, long long n, int max_blocks, cudaStream_t st) {
  if (n % kArenaBlock) throw std::runtime_error("gosgd_push: n must be block aligned");
  if (dest < 0 || dest >= c.world || dest == c.rank) throw std::runtime_error("gosgd_push: bad destination");
  uint32_t* s = (uint32_t*)state;
  gosgd_push_begin_kernel<<<1, 32, 0, st>>>(c, s);
  char* base = reinterpret_cast<char*>(c.arena[c.rank]);
  const long long nb = n / kArenaBlock;
  copy_flat_kernel<4><<<pick_grid((nb + 3) / 4, max_blocks), kThreads, 0, st>>>((float*)(base + snap_off), nullptr, (const float*)(base + w_off), nb,
                                                                            s + 1);
  gosgd_push_end_kernel<<<1, 32, 0, st>>>(c, s, dest);
  count_launch(3); TMPI_CHECK_LAUNCH("gosgd_push"); ::tmpi::check_capture(st, "gosgd_push");
}
void gosgd_poll_merge(const CommCtx& c, void* state, long long w_off, long long h_off, long long snap_off, long long n, int max_blocks,
                      cudaStream_t st) {
  if (n % kArenaBlock) throw std::runtime_error("gosgd_poll_merge: n must be block aligned");
  uint32_t* s = (uint32_t*)state;
  const long long nb = n / kArenaBlock;
  gosgd_poll_kernel<<<1, 32, 0, st>>>(c, s);
  gosgd_pull_merge_kernel<4><<<pick_grid((nb + 3) / 4, max_blocks), kThreads, 0, st>>>(c, s, w_off, h_off, snap_off, nb);
  gosgd_ack_kernel<<<1, 32, 0, st>>>(c, s);
  count_launch(3); TMPI_CHECK_LAUNCH("gosgd_poll_merge"); ::tmpi::check_capture(st, "gosgd_poll_merge");
}

// ============================================================================ reference kernels K1..K5 (legacy strategies)
template <typename TI, typename TO> __global__ void cast_kernel(const TI* __restrict__ s, TO* __restrict__ d, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) d[i] = (TO)(float)s[i];
}
// kind: 0 f32→f16, 1 f16→f32, 2 f32→bf16, 3 bf16→f32     (K1/K5: float2half / half2float)
void cast_flat(const void* src, void* dst, long long n, int kind, cudaStream_t st) {
  const int g = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
  if (n <= 0) return;
  switch (kind) {
    case 0: cast_kernel<float, __half><<<g, 256, 0, st>>>((const float*)src, (__half*)dst, n); break;
    case 1: cast_kernel<__half, float><<<g, 256, 0, st>>>((const __half*)src, (float*)dst, n); break;
    case 2: cast_kernel<float, __nv_bfloat16><<<g, 256, 0, st>>>((const float*)src, (__nv_bfloat16*)dst, n); break;
    case 3: cast_kernel<__nv_bfloat16, float><<<g, 256, 0, st>>>((const __nv_bfloat16*)src, (float*)dst, n); break;
    default: throw std::runtime_error("cast_flat: bad kind");
  }
  count_launch(); TMPI_CHECK_LAUNCH("cast_flat"); ::tmpi::check_capture(st, "cast_flat");
}

// K2/K3 sumfloats / sumhalfs with the reference's loop bug fixed (SURVEY §2.9 #1): dst[i] = Σ_j src[i + chunk*j], fp32 accumulate
template <typename T> __global__ void sum_chunks_kernel(const T* __restrict__ s, T* __restrict__ d, long long chunk, int nchunks) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < chunk; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < nchunks; ++j) acc += (float)s[i + chunk * j];
    d[i] = (T)acc;
  }
}
void sum_chunks(const void* src, void* dst, long long chunk, int nchunks, int is_half, cudaStream_t st) {
  if (chunk <= 0) return;
  const int g = (int)std::min<long long>((chunk + 255) / 256, (long long)sm_count() * 16);
  if (is_half) sum_chunks_kernel<__half><<<g, 256, 0, st>>>((const __half*)src, (__half*)dst, chunk, nchunks);
  else sum_chunks_kernel<float><<<g, 256, 0, st>>>((const float*)src, (float*)dst, chunk, nchunks);
  count_launch(); TMPI_CHECK_LAUNCH("sum_chunks"); ::tmpi::check_capture(st, "sum_chunks");
}

// K4/K5 vecadd / vecaddhalf: cur[i] += tmp[i]
template <typename T> __global__ void vecadd_kernel(T* __restrict__ cur, const T* __restrict__ tmp, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    cur[i] = (T)((float)cur[i] + (float)tmp[i]);
}
void vecadd(void* cur, const void* tmp, long long n, int is_half, cudaStream_t st) {
  if (n <= 0) return;
  const int g = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
  if (is_half) vecadd_kernel<__half><<<g, 256, 0, st>>>((__half*)cur, (const __half*)tmp, n);
  else vecadd_kernel<float><<<g, 256, 0, st>>>((float*)cur, (const float*)tmp, n);
  count_launch(); TMPI_CHECK_LAUNCH("vecadd"); ::tmpi::check_capture(st, "vecadd");
}

}  // namespace tmpi
