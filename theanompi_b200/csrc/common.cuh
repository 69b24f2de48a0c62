// Common helpers for the sm_90a extension (torch-free: raw pointers + cudaStream_t).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>
#include <atomic>
#include <stdexcept>
#include <string>

namespace tmpi {

// every launcher bumps this; Python reads it for bench.py's "gpu_launches"
extern std::atomic<unsigned long long> g_launch_count;
inline void count_launch(int n = 1) { g_launch_count.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

inline void check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    throw std::runtime_error(std::string("tmpi_native: ") + what + ": " + cudaGetErrorString(e));
  }
}
#define TMPI_CHECK_LAUNCH(name) ::tmpi::check_cuda(cudaGetLastError(), name)

// TMPI_DEBUG_CAPTURE=1: after every launch verify that an ongoing stream capture is still valid and name the
// first op that invalidated it (CUDA only reports "a previous error" at capture end).
inline void check_capture(cudaStream_t st, const char* name) {
  static int dbg = -1;
  if (dbg < 0) { const char* e = getenv("TMPI_DEBUG_CAPTURE"); dbg = (e && e[0] == '1') ? 1 : 0; }
  if (!dbg) return;
  cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
  cudaError_t e = cudaStreamIsCapturing(st, &s);
  if (e != cudaSuccess || s == cudaStreamCaptureStatusInvalidated)
    throw std::runtime_error(std::string("tmpi_native: stream capture invalidated at/before ") + name + ": " + cudaGetErrorString(e));
}

constexpr int kArenaBlock = 1024;   // must match parallel/arena.py BLOCK
constexpr int kMaxGroups = 8;

struct GroupTable {
  float lr_mult[kMaxGroups];
  float wd[kMaxGroups];
  int exch[kMaxGroups];
};

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

#ifdef __CUDACC__
__device__ __forceinline__ float bf16_to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ __nv_bfloat16 f_to_bf16(float v) { return __float2bfloat16_rn(v); }

// 16-byte vector of 8 bf16
struct __align__(16) bf16x8 { __nv_bfloat162 v[4]; };

__device__ __forceinline__ void unpack8(const bf16x8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(p.v[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

// 16-byte vectors of bf16 (8) or fp32 (4) activations, unpacked to / packed from fp32 registers: the kernels that run in both
// precision modes are templates on the storage type T
template <typename T> struct VecIO;
// (Raw: the 16-byte register type, for kernels that keep vectors packed between load and store; LOG2N: C >> LOG2N vectors per row)
template <> struct VecIO<__nv_bfloat16> {
  static constexpr int N = 8, LOG2N = 3;
  using Raw = bf16x8;
  static __device__ __forceinline__ void unpack(const Raw& r, float* f) { unpack8(r, f); }
  static __device__ __forceinline__ Raw pack(const float* f) { return pack8(f); }
  static __device__ __forceinline__ void ld(const __nv_bfloat16* p, float* f) { unpack8(*reinterpret_cast<const bf16x8*>(p), f); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, const float* f) { *reinterpret_cast<bf16x8*>(p) = pack8(f); }
};
template <> struct VecIO<float> {
  static constexpr int N = 4, LOG2N = 2;
  using Raw = float4;
  static __device__ __forceinline__ void unpack(const Raw& v, float* f) { f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w; }
  static __device__ __forceinline__ Raw pack(const float* f) { return make_float4(f[0], f[1], f[2], f[3]); }
  static __device__ __forceinline__ void ld(const float* p, float* f) {
    const float4 v = *reinterpret_cast<const float4*>(p); f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  static __device__ __forceinline__ void st(float* p, const float* f) { *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]); }
};
// N one-byte flags (argmax window indices, dropout keep bits) with one 8- or 4-byte load; .y is 0 for N = 4
template <int N> __device__ __forceinline__ uint2 ld_flags(const uint8_t* p) {
  if (N == 8) return *reinterpret_cast<const uint2*>(p);
  return make_uint2(*reinterpret_cast<const uint32_t*>(p), 0u);
}
// scalar conversions between the storage type and fp32
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return bf16_to_f(v); }
__device__ __forceinline__ float to_f(float v) { return v; }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return f_to_bf16(v); }
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }

// Activation of a fused elementwise pass.  ACT_FLAG: identity or ReLU chosen by the kernel's runtime `relu` argument (the
// instantiation every pre-existing launch uses, its code unchanged); the others are compile-time variants.  The backward mask is
// computed from the activation's OUTPUT y: ReLU / leaky ReLU keep the sign of their input, sigmoid' = y (1 - y).
enum : int { ACT_FLAG = -1, ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2, ACT_SIGMOID = 3 };
template <int ACT> __device__ __forceinline__ float act_fwd(float v, float slope) {
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_LEAKY) return v > 0.f ? v : v * slope;
  if (ACT == ACT_SIGMOID) return 1.f / (1.f + __expf(-v));
  return v;
}
template <int ACT> __device__ __forceinline__ float act_bwd(float d, float y, float slope) {
  if (ACT == ACT_RELU) return y > 0.f ? d : 0.f;
  if (ACT == ACT_LEAKY) return y > 0.f ? d : d * slope;
  if (ACT == ACT_SIGMOID) return d * y * (1.f - y);
  return d;
}

__device__ __forceinline__ uint2 pack_bf16x4(float4 v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  uint2 r; r.x = *reinterpret_cast<uint32_t*>(&a); r.y = *reinterpret_cast<uint32_t*>(&b); return r;
}

// ------------------------------------------------------------------ the SGD math (one float4)
// Shared by the flat optimizer kernels (comm_kernels.cu) and the SGD epilogue of the wgrad GEMM (gemm_wgmma.cu): both must
// produce the same bits for the same (W, U, G).
struct Hyper { float lr, mu, inv_k; int nesterov; };

__device__ __forceinline__ void sgd4(float4& w, float4& u, const float4& gsum, const Hyper& h, float lrm, float wd) {
  const float lr = h.lr * lrm;
#define TMPI_SGD1(W, U, G)                                   \
  {                                                          \
    const float ge = G * h.inv_k + wd * W;                   \
    U = h.mu * U + ge;                                       \
    W -= lr * (h.nesterov ? (ge + h.mu * U) : U);            \
  }
  TMPI_SGD1(w.x, u.x, gsum.x) TMPI_SGD1(w.y, u.y, gsum.y) TMPI_SGD1(w.z, u.z, gsum.z) TMPI_SGD1(w.w, u.w, gsum.w)
#undef TMPI_SGD1
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif

// TMPI_DETERMINISTIC=1: bit-reproducible training steps — no split-K (gradient tiles are otherwise combined with fp32 atomics in
// arrival order) and every cross-CTA atomic reduction (bias gradients, batch-norm statistics) collapses to one CTA per channel
// group with a fixed summation order.  Slower; meant for debugging / regression runs.
inline bool deterministic_mode() {
  static const bool v = [] { const char* e = getenv("TMPI_DETERMINISTIC"); return e && e[0] == '1'; }();
  return v;
}

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace tmpi
