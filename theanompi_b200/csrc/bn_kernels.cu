// Batch normalisation (+ residual add)(+ ReLU) forward / backward and the residual `add`, NHWC, bf16 or fp32 activations, fp32
// statistics / parameters.  The reference takes these from Lasagne / Keras (lasagne_model_zoo/resnet50.py:14-77 batch_norm +
// ElemwiseSumLayer + rectify; keras_model_zoo/wresnet.py:37-82 BatchNormalization / merge) and special-cases parameters NAMED
// gamma / beta in its optimizer and exchanger (lib/opt.py:207-226, lib/exchanger.py:35-43).
//
//   forward (training)   stats:    per-channel Σx, Σx² (row slabs per CTA, column sums in registers → smem → one atomic per CTA)
//                        finalize: mean, rstd, running statistics (momentum update, unbiased variance)
//                        apply:    y = γ·(x − mean)·rstd + β  [+ residual] [ReLU]
//   backward             reduce:   g = dy ⊙ [y > 0];  dβ = Σ g,  dγ = Σ g·x̂           (x̂ = (x − mean)·rstd)
//                        apply:    dx = γ·rstd·(g − dβ/M − x̂·dγ/M);  d residual = g
// M = N·H·W rows.  Each pass is one streaming kernel over the activation tensor (16-byte vectors).
//
// Drop-path (stochastic depth) is a compile-time variant (kDrop) of the apply pass and of both backward passes: with a row s of
// the step's drop table (one fp32 scale per sample, ops/drop_path.py), y = act(s_n·(γ·x̂ + β) + residual), and the backward uses
// g̃ = s_n·g in Σg, Σg·x̂ and dx while the residual still receives g.  The statistics stay those of the whole batch.
#include "common.cuh"
#include "api.h"
#include <algorithm>

namespace tmpi {

static inline int grid1(long long n, int block) { return (int)((n + block - 1) / block); }

// Sample index n = r / hw of the rows a thread walks with a fixed stride: one division when the walk starts, then one carry per
// step (the stride split once into whole samples q and leftover rows m), never a division per 16-byte vector.
struct SampleWalk {
  unsigned n, p, hw, q, m;
  __device__ __forceinline__ void init(long long r, int hw_, int stride) {
    hw = (unsigned)hw_;
    n = (unsigned)(r / hw_); p = (unsigned)(r - (long long)n * hw_);
    q = (unsigned)stride / hw; m = (unsigned)stride % hw;
  }
  __device__ __forceinline__ void step() { n += q; p += m; if (p >= hw) { p -= hw; ++n; } }
};

// ---------------------------------------------------------------- column reductions over row slabs
// MODE 0: a = Σ x, b = Σ x²            (forward statistics)
// MODE 1: a = Σ g, b = Σ g·x̂          (backward: g = dy ⊙ [y > 0] when relu; g = act'(y) ⊙ dy for ACT_LEAKY / ACT_SIGMOID)
//         kDrop: g ← drop[r / hw]·g    (the drop-path scale of the row's sample)
template <typename T, int MODE, int ACT, bool kDrop = false>
__global__ void __launch_bounds__(256) bn_colreduce_kernel(const T* __restrict__ x, const T* __restrict__ dy, const T* __restrict__ y,
                                                          const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ out_a,
                                                          float* __restrict__ out_b, long long R, int C, int relu, int VT, int rows_per_cta,
                                                          float slope, const float* __restrict__ drop, int hw) {
  static_assert(!kDrop || (MODE == 1 && ACT == ACT_FLAG), "drop-path: backward reduction with ReLU / identity only");
  constexpr int N = VecIO<T>::N;
  extern __shared__ float sm[];                       // [2][RL][VT*N]
  const int nvec = C / N;
  const int RL = blockDim.x / VT;
  const int tv = threadIdx.x % VT, tr = threadIdx.x / VT;
  const int cv = blockIdx.y * VT + tv;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  float a[N], b[N], mu[N], rs[N];
#pragma unroll
  for (int i = 0; i < N; ++i) { a[i] = 0.f; b[i] = 0.f; mu[i] = 0.f; rs[i] = 1.f; }
  const bool on = tr < RL && cv < nvec;
  if (on) {
    if (MODE == 1) {
#pragma unroll
      for (int i = 0; i < N; ++i) { mu[i] = mean[cv * N + i]; rs[i] = rstd[cv * N + i]; }
    }
    const long long rend = min(R, r0 + rows_per_cta);
    // UR rows per trip, all (raw 16-byte) loads issued before any use — this pass is pure streaming, memory-level parallelism
    // is everything; the vectors stay packed until they are consumed so the trip fits in ~64 registers
    constexpr int UR = MODE == 0 ? 4 : 2;
    SampleWalk w;
    if constexpr (kDrop) w.init(r0 + tr, hw, RL);
    for (long long r = r0 + tr; r < rend; r += UR * RL) {
      uint4 xr[UR], gr[UR], yr[UR];
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < rend) {
          xr[u] = *reinterpret_cast<const uint4*>(x + rr * C + cv * N);
          if (MODE == 1) {
            gr[u] = *reinterpret_cast<const uint4*>(dy + rr * C + cv * N);
            if (ACT != ACT_FLAG || relu) yr[u] = *reinterpret_cast<const uint4*>(y + rr * C + cv * N);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < rend) {
          float xv[N];
          VecIO<T>::ld(reinterpret_cast<const T*>(&xr[u]), xv);
          if (MODE == 0) {
#pragma unroll
            for (int i = 0; i < N; ++i) { a[i] += xv[i]; b[i] += xv[i] * xv[i]; }
          } else {
            float gv[N], yv[N];
            VecIO<T>::ld(reinterpret_cast<const T*>(&gr[u]), gv);
            if (ACT != ACT_FLAG || relu) VecIO<T>::ld(reinterpret_cast<const T*>(&yr[u]), yv);
            float s = 1.f;
            if constexpr (kDrop) s = __ldg(drop + w.n);
#pragma unroll
            for (int i = 0; i < N; ++i) {
              float g = gv[i];
              if (ACT == ACT_FLAG) { if (relu && !(yv[i] > 0.f)) g = 0.f; }
              else g = act_bwd<ACT>(g, yv[i], slope);
              if constexpr (kDrop) g *= s;
              a[i] += g; b[i] += g * (xv[i] - mu[i]) * rs[i];
            }
          }
        }
        if constexpr (kDrop) w.step();
      }
    }
  }
  float* sa = sm;
  float* sb = sm + RL * VT * N;
  if (tr < RL) {
#pragma unroll
    for (int i = 0; i < N; ++i) { sa[(tr * VT + tv) * N + i] = a[i]; sb[(tr * VT + tv) * N + i] = b[i]; }
  }
  __syncthreads();
  if (threadIdx.x < VT * N) {
    const int v = threadIdx.x / N, i = threadIdx.x % N;
    const int c = (blockIdx.y * VT + v) * N + i;
    if (c < C) {
      float s0 = 0.f, s1 = 0.f;
      for (int t = 0; t < RL; ++t) { s0 += sa[(t * VT + v) * N + i]; s1 += sb[(t * VT + v) * N + i]; }
      atomicAdd(out_a + c, s0);
      atomicAdd(out_b + c, s1);
    }
  }
}

template <typename T, int MODE, int ACT = ACT_FLAG, bool kDrop = false>
static void colreduce(const void* x, const void* dy, const void* y, const float* mean, const float* rstd, float* a, float* b, long long R,
                      int C, int relu, cudaStream_t st, float slope = 0.f, const float* drop = nullptr, int hw = 1) {
  constexpr int N = VecIO<T>::N;
  if (C % N) throw std::runtime_error("batch_norm: C must be a multiple of the 16-byte vector width");
  const int nvec = C / N;
  const int VT = nvec < 32 ? nvec : 32;
  const int RL = 256 / VT;
  // enough CTAs to fill the machine a few times, few enough that the atomics stay cheap
  long long slabs = std::max<long long>(1, std::min<long long>((R + RL - 1) / RL, (long long)sm_count() * 8 / std::max(1, (nvec + VT - 1) / VT)));
  if (deterministic_mode()) slabs = 1;                     // one CTA per channel group: fixed summation order, no atomics race
  const int rows_per_cta = (int)((R + slabs - 1) / slabs);
  dim3 grid((unsigned)((R + rows_per_cta - 1) / rows_per_cta), (unsigned)((nvec + VT - 1) / VT));
  const size_t smem = (size_t)2 * RL * VT * N * sizeof(float);
  check_cuda(cudaMemsetAsync(a, 0, (size_t)C * 4, st), "bn memset");
  check_cuda(cudaMemsetAsync(b, 0, (size_t)C * 4, st), "bn memset");
  bn_colreduce_kernel<T, MODE, ACT, kDrop><<<grid, 256, smem, st>>>((const T*)x, (const T*)dy, (const T*)y, mean, rstd, a, b, R, C, relu, VT,
                                                                    rows_per_cta, slope, drop, hw);
}

// mean / rstd from the sums (training) or from the running statistics (eval); momentum update of the running statistics;
// per-channel affine of the apply pass written over the (consumed) sums:  y = x * scale + shift
__global__ void bn_finalize_kernel(float* __restrict__ sum, float* __restrict__ sumsq, float* __restrict__ mean,
                                   float* __restrict__ rstd, float* __restrict__ run_mean, float* __restrict__ run_var,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, int C, float inv_m,
                                   float unbias, float momentum, float eps, int training) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float m, r;
  if (training) {
    m = sum[c] * inv_m;
    const float v = fmaxf(sumsq[c] * inv_m - m * m, 0.f);
    r = rsqrtf(v + eps);
    if (run_mean) {
      run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * m;
      run_var[c] = (1.f - momentum) * run_var[c] + momentum * v * unbias;
    }
  } else {
    m = run_mean[c];
    r = rsqrtf(run_var[c] + eps);
  }
  mean[c] = m; rstd[c] = r;
  const float sc = gamma[c] * r;
  sum[c] = sc;                       // scale
  sumsq[c] = beta[c] - m * sc;       // shift
}

// Elementwise passes: thread = (channel vector cv, row lane); the per-channel coefficients are loaded ONCE per thread and the
// thread then walks rows with a fixed stride — no per-element division (the first version did a 64-bit modulo per 16 bytes and
// was issue-bound at ~5x the memory roofline), 32-bit offsets inside a row slab.
// kDrop: y = act(drop[r / hw]·(scale·x + shift) + res); the launcher guarantees a residual
template <typename T, int ACT, bool kDrop = false>
__global__ void __launch_bounds__(256) bn_apply_kernel(const T* __restrict__ x, const T* __restrict__ res, T* __restrict__ y,
                                                      const float* __restrict__ scale, const float* __restrict__ shift, long long R, int C,
                                                      int relu, int VT, int rows_per_cta, float slope, const float* __restrict__ drop, int hw) {
  static_assert(!kDrop || ACT == ACT_FLAG, "drop-path: ReLU / identity only");
  constexpr int N = VecIO<T>::N;
  const int nvec = C / N;
  const int RL = blockDim.x / VT;
  const int tv = threadIdx.x % VT, tr = threadIdx.x / VT;
  const int cv = blockIdx.y * VT + tv;
  if (tr >= RL || cv >= nvec) return;
  float sc[N], sh[N];
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    *reinterpret_cast<float4*>(sc + i) = __ldg(reinterpret_cast<const float4*>(scale + cv * N + i));
    *reinterpret_cast<float4*>(sh + i) = __ldg(reinterpret_cast<const float4*>(shift + cv * N + i));
  }
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long rend = min(R, r0 + rows_per_cta);
  const T* xp = x + r0 * C + cv * N;
  const T* rp = res ? res + r0 * C + cv * N : nullptr;
  T* yp = y + r0 * C + cv * N;
  const int nrows = (int)(rend - r0);
  SampleWalk w;
  if constexpr (kDrop) w.init(r0 + tr, hw, RL);
  for (int r = tr; r < nrows; r += 2 * RL) {
    // two rows in flight per trip
    const int r2 = r + RL;
    const bool two = r2 < nrows;
    float a[N], b[N], ra[N], rb[N];
    float sa = 1.f, sb = 1.f;
    if constexpr (kDrop) { sa = __ldg(drop + w.n); w.step(); if (two) sb = __ldg(drop + w.n); w.step(); }
    VecIO<T>::ld(xp + (unsigned)r * (unsigned)C, a);
    if (two) VecIO<T>::ld(xp + (unsigned)r2 * (unsigned)C, b);
    if (rp) { VecIO<T>::ld(rp + (unsigned)r * (unsigned)C, ra); if (two) VecIO<T>::ld(rp + (unsigned)r2 * (unsigned)C, rb); }
#pragma unroll
    for (int i = 0; i < N; ++i) {
      a[i] = fmaf(a[i], sc[i], sh[i]);
      if constexpr (kDrop) a[i] = fmaf(sa, a[i], ra[i]);
      else if (rp) a[i] += ra[i];
      if (ACT == ACT_FLAG) { if (relu) a[i] = fmaxf(a[i], 0.f); }
      else a[i] = act_fwd<ACT>(a[i], slope);
    }
    VecIO<T>::st(yp + (unsigned)r * (unsigned)C, a);
    if (two) {
#pragma unroll
      for (int i = 0; i < N; ++i) {
        b[i] = fmaf(b[i], sc[i], sh[i]);
        if constexpr (kDrop) b[i] = fmaf(sb, b[i], rb[i]);
        else if (rp) b[i] += rb[i];
        if (ACT == ACT_FLAG) { if (relu) b[i] = fmaxf(b[i], 0.f); }
        else b[i] = act_fwd<ACT>(b[i], slope);
      }
      VecIO<T>::st(yp + (unsigned)r2 * (unsigned)C, b);
    }
  }
}

// per-channel coefficients of the backward apply pass:  dx = k1 * g + k2 * x + k3
//   k1 = γ·rstd,  k2 = −k1·rstd·dγ/M,  k3 = −k1·dβ/M − k2·mean      (from dx = γ·rstd·(g − dβ/M − x̂·dγ/M), x̂ = (x − mean)·rstd)
__global__ void bn_bwd_coef_kernel(const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                                   const float* __restrict__ dgamma, const float* __restrict__ dbeta, float* __restrict__ k, int C, float inv_m) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float k1 = gamma[c] * rstd[c];
  const float k2 = -k1 * rstd[c] * dgamma[c] * inv_m;
  k[c] = k1; k[C + c] = k2; k[2 * C + c] = -k1 * dbeta[c] * inv_m - k2 * mean[c];
}

// accumulate mode: the same coefficients from THIS batch's sums (sb = Σg, sg = Σg·x̂ in the scratch), which one thread per channel
// then adds into the accumulated dβ / dγ (one fp32 add per element: deterministic)
__global__ void bn_bwd_coef_accum_kernel(const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                                         const float* __restrict__ sg, const float* __restrict__ sb, float* __restrict__ dgamma,
                                         float* __restrict__ dbeta, float* __restrict__ k, int C, float inv_m) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float g = sg[c], b = sb[c];
  const float k1 = gamma[c] * rstd[c];
  const float k2 = -k1 * rstd[c] * g * inv_m;
  k[c] = k1; k[C + c] = k2; k[2 * C + c] = -k1 * b * inv_m - k2 * mean[c];
  dgamma[c] += g;
  dbeta[c] += b;
}

// kDrop: dx from g̃ = drop[r / hw]·g (the coefficients k come from the Σ of g̃), dres = g
template <typename T, int ACT, bool kDrop = false>
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const T* __restrict__ x, const T* __restrict__ dy, const T* __restrict__ y,
                                                          T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ k, long long R, int C,
                                                          int relu, int VT, int rows_per_cta, float slope, const float* __restrict__ drop,
                                                          int hw) {
  static_assert(!kDrop || ACT == ACT_FLAG, "drop-path: ReLU / identity only");
  constexpr int N = VecIO<T>::N;
  const int nvec = C / N;
  const int RL = blockDim.x / VT;
  const int tv = threadIdx.x % VT, tr = threadIdx.x / VT;
  const int cv = blockIdx.y * VT + tv;
  if (tr >= RL || cv >= nvec) return;
  float k1[N], k2[N], k3[N];
#pragma unroll
  for (int i = 0; i < N; i += 4) {
    *reinterpret_cast<float4*>(k1 + i) = __ldg(reinterpret_cast<const float4*>(k + cv * N + i));
    *reinterpret_cast<float4*>(k2 + i) = __ldg(reinterpret_cast<const float4*>(k + C + cv * N + i));
    *reinterpret_cast<float4*>(k3 + i) = __ldg(reinterpret_cast<const float4*>(k + 2 * C + cv * N + i));
  }
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const int nrows = (int)(min(R, r0 + rows_per_cta) - r0);
  const long long base = r0 * C + cv * N;
  SampleWalk w;
  if constexpr (kDrop) w.init(r0 + tr, hw, RL);
  for (int r = tr; r < nrows; r += RL) {
    const unsigned o = (unsigned)r * (unsigned)C;
    float xv[N], g[N], out[N];
    float s = 1.f;
    if constexpr (kDrop) { s = __ldg(drop + w.n); w.step(); }
    VecIO<T>::ld(x + base + o, xv);
    VecIO<T>::ld(dy + base + o, g);
    if (ACT != ACT_FLAG || relu) {
      float yv[N];
      VecIO<T>::ld(y + base + o, yv);
#pragma unroll
      for (int i = 0; i < N; ++i) {
        if (ACT == ACT_FLAG) { if (!(yv[i] > 0.f)) g[i] = 0.f; }
        else g[i] = act_bwd<ACT>(g[i], yv[i], slope);
      }
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if constexpr (kDrop) out[i] = fmaf(k1[i], s * g[i], fmaf(k2[i], xv[i], k3[i]));
      else out[i] = fmaf(k1[i], g[i], fmaf(k2[i], xv[i], k3[i]));
    }
    VecIO<T>::st(dx + base + o, out);
    if (dres) VecIO<T>::st(dres + base + o, g);
  }
}

// y = a + b (the residual merge of pre-activation blocks)
template <typename T>
__global__ void __launch_bounds__(256) add_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, long long total_vec) {
  constexpr int N = VecIO<T>::N;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_vec) return;
  float av[N], bv[N];
  VecIO<T>::ld(a + idx * N, av);
  VecIO<T>::ld(b + idx * N, bv);
#pragma unroll
  for (int i = 0; i < N; ++i) av[i] += bv[i];
  VecIO<T>::st(y + idx * N, av);
}

// y = s_n·a + b per sample n = blockIdx.y (b absent: y = s_n·a) — the drop-path merge of a pre-activation block and its branch
// gradient; the 2-D grid gives the sample index without any division
template <typename T>
__global__ void __launch_bounds__(256) add_scaled_kernel(const T* __restrict__ a, const T* __restrict__ b, const float* __restrict__ s,
                                                        T* __restrict__ y, int vec_per_sample) {
  constexpr int N = VecIO<T>::N;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= vec_per_sample) return;
  const long long e = ((long long)blockIdx.y * vec_per_sample + v) * N;
  const float sn = __ldg(s + blockIdx.y);
  float av[N], bv[N];
  VecIO<T>::ld(a + e, av);
  if (b) {
    VecIO<T>::ld(b + e, bv);
#pragma unroll
    for (int i = 0; i < N; ++i) av[i] = fmaf(sn, av[i], bv[i]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) av[i] *= sn;
  }
  VecIO<T>::st(y + e, av);
}

// y = a + b + c + d (gradient merge of the four inception branches)
template <typename T>
__global__ void __launch_bounds__(256) add4_kernel(const T* __restrict__ a, const T* __restrict__ b, const T* __restrict__ c, const T* __restrict__ d,
                                                  T* __restrict__ y, long long total_vec) {
  constexpr int N = VecIO<T>::N;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_vec) return;
  float av[N], bv[N], cv[N], dv[N];
  VecIO<T>::ld(a + idx * N, av); VecIO<T>::ld(b + idx * N, bv); VecIO<T>::ld(c + idx * N, cv); VecIO<T>::ld(d + idx * N, dv);
#pragma unroll
  for (int i = 0; i < N; ++i) av[i] = (av[i] + bv[i]) + (cv[i] + dv[i]);
  VecIO<T>::st(y + idx * N, av);
}

// (row slab, channel-vector group) launch geometry shared by the elementwise passes
struct RowGeom { dim3 grid; int VT, rows_per_cta; };
static RowGeom row_geom(long long R, int nvec) {
  RowGeom g;
  g.VT = nvec < 32 ? nvec : 32;
  const int RL = 256 / g.VT;
  const int gy = (nvec + g.VT - 1) / g.VT;
  // ~16 row trips per thread, at least ~4 CTAs per SM in flight, row slabs small enough for 32-bit in-slab offsets
  long long slabs = std::max<long long>(1, std::min<long long>((R + RL - 1) / RL, std::max<long long>((long long)sm_count() * 8 / gy, (R + RL * 16 - 1) / (RL * 16))));
  g.rows_per_cta = (int)((R + slabs - 1) / slabs);
  g.grid = dim3((unsigned)((R + g.rows_per_cta - 1) / g.rows_per_cta), (unsigned)gy);
  return g;
}

// ---------------------------------------------------------------- launchers (f32 = 1: fp32 activations, else bf16)
template <typename T>
static void bn_apply_t(const void* x, const void* res, void* y, const float* s0, const float* s1, long long R, int C, int act, float slope,
                       const float* drop, int hw, const RowGeom& g, cudaStream_t st) {
#define BNA(A) bn_apply_kernel<T, A><<<g.grid, 256, 0, st>>>((const T*)x, (const T*)res, (T*)y, s0, s1, R, C, act, g.VT, g.rows_per_cta, slope, \
                                                             nullptr, 1)
  if (drop) bn_apply_kernel<T, ACT_FLAG, true><<<g.grid, 256, 0, st>>>((const T*)x, (const T*)res, (T*)y, s0, s1, R, C, act, g.VT,
                                                                        g.rows_per_cta, slope, drop, hw);
  else if (act == ACT_NONE || act == ACT_RELU) BNA(ACT_FLAG);
  else if (act == ACT_LEAKY) BNA(ACT_LEAKY);
  else if (act == ACT_SIGMOID) BNA(ACT_SIGMOID);
  else throw std::runtime_error("batch_norm: unknown activation");
#undef BNA
}

template <typename T>
static void bn_bwd_t(const void* x, const void* dy, const void* y, void* dx, void* dres, const float* mean, const float* rstd, void* dgamma,
                     void* dbeta, const float* gamma, float* k, long long R, int C, int act, float slope, int accumulate, const float* drop,
                     int hw, cudaStream_t st) {
  constexpr int N = VecIO<T>::N;
  // accumulate: this batch's sums go to the scratch after the coefficients (k[3C, 5C)), not into the accumulated dγ / dβ
  float* sb = accumulate ? k + 3 * C : (float*)dbeta;
  float* sg = accumulate ? k + 4 * C : (float*)dgamma;
  if (drop) colreduce<T, 1, ACT_FLAG, true>(x, dy, y, mean, rstd, sb, sg, R, C, act, st, 0.f, drop, hw);
  else if (act == ACT_NONE || act == ACT_RELU) colreduce<T, 1>(x, dy, y, mean, rstd, sb, sg, R, C, act, st);
  else if (act == ACT_LEAKY) colreduce<T, 1, ACT_LEAKY>(x, dy, y, mean, rstd, sb, sg, R, C, act, st, slope);
  else if (act == ACT_SIGMOID) colreduce<T, 1, ACT_SIGMOID>(x, dy, y, mean, rstd, sb, sg, R, C, act, st, slope);
  else throw std::runtime_error("batch_norm: unknown activation");
  if (accumulate)
    bn_bwd_coef_accum_kernel<<<grid1(C, 256), 256, 0, st>>>(gamma, mean, rstd, sg, sb, (float*)dgamma, (float*)dbeta, k, C, 1.f / (float)R);
  else
    bn_bwd_coef_kernel<<<grid1(C, 256), 256, 0, st>>>(gamma, mean, rstd, (const float*)dgamma, (const float*)dbeta, k, C, 1.f / (float)R);
  const RowGeom g = row_geom(R, C / N);
  if ((long long)g.rows_per_cta * C >= (1LL << 32)) throw std::runtime_error("batch_norm: row slab too large for 32-bit offsets");
#define BNB(A) bn_bwd_apply_kernel<T, A><<<g.grid, 256, 0, st>>>((const T*)x, (const T*)dy, (const T*)y, (T*)dx, (T*)dres, k, R, C, act, g.VT, \
                                                                g.rows_per_cta, slope, nullptr, 1)
  if (drop) bn_bwd_apply_kernel<T, ACT_FLAG, true><<<g.grid, 256, 0, st>>>((const T*)x, (const T*)dy, (const T*)y, (T*)dx, (T*)dres, k, R, C,
                                                                            act, g.VT, g.rows_per_cta, slope, drop, hw);
  else if (act == ACT_LEAKY) BNB(ACT_LEAKY);
  else if (act == ACT_SIGMOID) BNB(ACT_SIGMOID);
  else BNB(ACT_FLAG);
#undef BNB
}

// act: ACT_NONE / ACT_RELU / ACT_LEAKY (slope) / ACT_SIGMOID after the affine (and the residual add)
// drop-path: the rows of sample n = r / (R / batch) are scaled by drop_scale[n] (one row of the step's table); ReLU / identity only
static int drop_hw(const void* drop_scale, long long R, int batch, int act, const char* who) {
  if (!drop_scale) return 1;
  if (batch < 1 || R % batch || R / batch > 0x7FFFFFFF)
    throw std::runtime_error(std::string(who) + ": a drop-path scale row needs R = batch * rows-per-sample");
  if (act != ACT_NONE && act != ACT_RELU) throw std::runtime_error(std::string(who) + ": drop-path takes ReLU or no activation");
  return (int)(R / batch);
}

void bn_forward(const void* x, const void* res, void* y, const void* gamma, const void* beta, void* mean, void* rstd, void* run_mean,
                void* run_var, void* scratch /*2*C floats*/, long long R, int C, float momentum, float eps, int training, int act, float slope,
                const void* drop_scale, int batch, int f32, cudaStream_t st) {
  float* s0 = (float*)scratch; float* s1 = s0 + C;
  if (C % 4) throw std::runtime_error("batch_norm: C must be a multiple of 4");
  if (drop_scale && !res) throw std::runtime_error("batch_norm: a drop-path scale row scales the branch of a residual add: needs res");
  const int hw = drop_hw(drop_scale, R, batch, act, "batch_norm");
  auto D = (const float*)drop_scale;
  if (training) {
    if (f32) colreduce<float, 0>(x, nullptr, nullptr, nullptr, nullptr, s0, s1, R, C, 0, st);
    else colreduce<__nv_bfloat16, 0>(x, nullptr, nullptr, nullptr, nullptr, s0, s1, R, C, 0, st);
  }
  bn_finalize_kernel<<<grid1(C, 256), 256, 0, st>>>(s0, s1, (float*)mean, (float*)rstd, (float*)run_mean, (float*)run_var, (const float*)gamma,
                                                    (const float*)beta, C, 1.f / (float)R, R > 1 ? (float)R / (float)(R - 1) : 1.f, momentum, eps,
                                                    training);
  const int N = f32 ? 4 : 8;
  if (C % N) throw std::runtime_error("batch_norm: C must be a multiple of the 16-byte vector width");
  const RowGeom g = row_geom(R, C / N);
  if ((long long)g.rows_per_cta * C >= (1LL << 32)) throw std::runtime_error("batch_norm: row slab too large for 32-bit offsets");
  if (f32) bn_apply_t<float>(x, res, y, s0, s1, R, C, act, slope, D, hw, g, st);
  else bn_apply_t<__nv_bfloat16>(x, res, y, s0, s1, R, C, act, slope, D, hw, g, st);
  count_launch(training ? 3 : 2); TMPI_CHECK_LAUNCH("bn_forward"); ::tmpi::check_capture(st, "bn_forward");
}

// scratch: 3*C floats (the coefficients of the apply pass), 5*C with accumulate (+ this batch's Σg, Σg·x̂)
void bn_backward(const void* x, const void* dy, const void* y, void* dx, void* dres, const void* gamma, const void* mean, const void* rstd,
                 void* dgamma, void* dbeta, void* scratch, long long R, int C, int act, float slope, int accumulate, const void* drop_scale,
                 int batch, int f32, cudaStream_t st) {
  auto M = (const float*)mean; auto RS = (const float*)rstd; auto G = (const float*)gamma; auto K = (float*)scratch;
  const int hw = drop_hw(drop_scale, R, batch, act, "batch_norm");
  auto D = (const float*)drop_scale;
  if (f32) bn_bwd_t<float>(x, dy, y, dx, dres, M, RS, dgamma, dbeta, G, K, R, C, act, slope, accumulate, D, hw, st);
  else bn_bwd_t<__nv_bfloat16>(x, dy, y, dx, dres, M, RS, dgamma, dbeta, G, K, R, C, act, slope, accumulate, D, hw, st);
  count_launch(3); TMPI_CHECK_LAUNCH("bn_backward"); ::tmpi::check_capture(st, "bn_backward");
}

void add_tensors(const void* a, const void* b, void* y, long long n, int f32, cudaStream_t st) {
  const int N = f32 ? 4 : 8;
  if (n % N) throw std::runtime_error("add_tensors: numel must be a multiple of the 16-byte vector width");
  const long long tv = n / N;
  if (f32) add_kernel<float><<<grid1(tv, 256), 256, 0, st>>>((const float*)a, (const float*)b, (float*)y, tv);
  else add_kernel<__nv_bfloat16><<<grid1(tv, 256), 256, 0, st>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, tv);
  count_launch(); TMPI_CHECK_LAUNCH("add_tensors"); ::tmpi::check_capture(st, "add_tensors");
}

void add_scaled(const void* a, const void* b, const void* scale, void* y, long long n, int batch, int f32, cudaStream_t st) {
  const int N = f32 ? 4 : 8;
  if (!scale || batch < 1 || batch > 65535 || n % batch || (n / batch) % N || n / batch / N > 0x7FFFFFFF)
    throw std::runtime_error("add_scaled: needs a scale row and 1 <= batch <= 65535 samples of a multiple of 16 bytes each");
  const int vps = (int)(n / batch / N);
  const dim3 grid((unsigned)grid1(vps, 256), (unsigned)batch);
  auto S = (const float*)scale;
  if (f32) add_scaled_kernel<float><<<grid, 256, 0, st>>>((const float*)a, (const float*)b, S, (float*)y, vps);
  else add_scaled_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, S, (__nv_bfloat16*)y, vps);
  count_launch(); TMPI_CHECK_LAUNCH("add_scaled"); ::tmpi::check_capture(st, "add_scaled");
}

void add4_tensors(const void* a, const void* b, const void* c, const void* d, void* y, long long n, int f32, cudaStream_t st) {
  const int N = f32 ? 4 : 8;
  if (n % N) throw std::runtime_error("add4_tensors: numel must be a multiple of the 16-byte vector width");
  const long long tv = n / N;
  if (f32) add4_kernel<float><<<grid1(tv, 256), 256, 0, st>>>((const float*)a, (const float*)b, (const float*)c, (const float*)d, (float*)y, tv);
  else add4_kernel<__nv_bfloat16><<<grid1(tv, 256), 256, 0, st>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, (const __nv_bfloat16*)c,
                                                                  (const __nv_bfloat16*)d, (__nv_bfloat16*)y, tv);
  count_launch(); TMPI_CHECK_LAUNCH("add4_tensors"); ::tmpi::check_capture(st, "add4_tensors");
}

}  // namespace tmpi
