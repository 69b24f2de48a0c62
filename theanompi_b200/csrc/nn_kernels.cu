// Fused non-GEMM layer kernels for sm_90a: LRN fwd/bwd, max/avg pooling fwd/bwd, dropout (Philox),
// softmax + NLL + top-1/top-5 error (+ dlogits), ReLU-mask + bias-gradient reduction, NHWC im2col /
// col2im-gather for the implicit-GEMM convolutions, normalise+crop+mirror for the loader.
// Activations are NHWC bf16 (C % 8 == 0) or, in the tf32 precision mode, fp32 (C % 4 == 0): 16-byte vectors unless noted;
// math is fp32.  Each op has one entry point taking `f32`; kernels that do the same arithmetic for both storage types are
// templates on VecIO<T>, the packed-bf16 tricks (max-pool forward, fused conv→max-pool backward) are bf16-only.
// Reference ops: theanompi/models/layers2.py (LRN :753-809, Pool :402-428, Dropout :864-908,
// Softmax :937-997, Crop/Subtract :223-347) and data/utils.py:42-129 (crop_and_mirror).
#include "common.cuh"
#include "api.h"
#include <algorithm>
#include <cfloat>
#include <type_traits>

namespace tmpi {

static inline int grid_for(long long n, int block) { return (int)((n + block - 1) / block); }

// ============================================================================ LRN
template <int HALF>
__global__ void lrn_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long rows, int C,
                               float k, float alpha, float beta) {
  const int nvec = C >> 3;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;           // host guarantees rows * nvec < 2^32
  if (idx >= (unsigned)rows * (unsigned)nvec) return;
  const long long r = idx / (unsigned)nvec;
  const int cv = (int)(idx - (unsigned)r * (unsigned)nvec);
  const __nv_bfloat16* row = x + r * C;
  float xs[24];
#pragma unroll
  for (int v = 0; v < 3; ++v) {
    const int c = (cv - 1 + v) * 8;
    if (c >= 0 && c < C) unpack8(*reinterpret_cast<const bf16x8*>(row + c), xs + 8 * v);
    else {
#pragma unroll
      for (int i = 0; i < 8; ++i) xs[8 * v + i] = 0.f;
    }
  }
  float out[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float s = 0.f;
#pragma unroll
    for (int j = -HALF; j <= HALF; ++j) { float t = xs[8 + i + j]; s += t * t; }
    const float scale = k + alpha * s;
    out[i] = xs[8 + i] * exp2f(-beta * __log2f(scale));
  }
  *reinterpret_cast<bf16x8*>(y + r * C + cv * 8) = pack8(out);
}

template <int HALF>
__global__ void lrn_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                               __nv_bfloat16* __restrict__ dx, long long rows, int C, float k, float alpha, float beta) {
  const int nvec = C >> 3;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;           // host guarantees rows * nvec < 2^32
  if (idx >= (unsigned)rows * (unsigned)nvec) return;
  const long long r = idx / (unsigned)nvec;
  const int cv = (int)(idx - (unsigned)r * (unsigned)nvec);
  float xs[24], ds[24];
#pragma unroll
  for (int v = 0; v < 3; ++v) {
    const int c = (cv - 1 + v) * 8;
    if (c >= 0 && c < C) {
      unpack8(*reinterpret_cast<const bf16x8*>(x + r * C + c), xs + 8 * v);
      unpack8(*reinterpret_cast<const bf16x8*>(dy + r * C + c), ds + 8 * v);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) { xs[8 * v + i] = 0.f; ds[8 * v + i] = 0.f; }
    }
  }
  // t_i = dy_i * x_i * s_i^(-beta-1) for i in [8-HALF, 16+HALF); p_i = s_i^-beta for the centre 8
  float t[8 + 2 * HALF];
  float pc[8];
#pragma unroll
  for (int a = 0; a < 8 + 2 * HALF; ++a) {
    const int L = 8 - HALF + a;
    float s = 0.f;
#pragma unroll
    for (int j = -HALF; j <= HALF; ++j) { float q = xs[L + j]; s += q * q; }
    const float scale = k + alpha * s;
    const float p = exp2f(-beta * __log2f(scale));
    t[a] = ds[L] * xs[L] * p / scale;
    if (a >= HALF && a < HALF + 8) pc[a - HALF] = p;
  }
  float out[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j <= 2 * HALF; ++j) acc += t[i + j];
    out[i] = ds[8 + i] * pc[i] - 2.f * alpha * beta * xs[8 + i] * acc;
  }
  *reinterpret_cast<bf16x8*>(dx + r * C + cv * 8) = pack8(out);
}

// fp32: one thread per element, any C and any window (the vector kernels above need C % 8 == 0 and n <= 9)
__global__ void lrn_fwd_f32_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int C, int half, float k,
                                   float alpha, float beta) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * C) return;
  const long long r = idx / C; const int c = (int)(idx - r * C);
  const float* row = x + r * C;
  float s = 0.f;
  for (int j = max(0, c - half); j <= min(C - 1, c + half); ++j) s += row[j] * row[j];
  y[idx] = row[c] * exp2f(-beta * __log2f(k + alpha * s));
}
__global__ void lrn_bwd_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, long long rows, int C,
                                   int half, float k, float alpha, float beta) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * C) return;
  const long long r = idx / C; const int c = (int)(idx - r * C);
  const float* xr = x + r * C; const float* dr = dy + r * C;
  // dx_c = dy_c * s_c^-beta - 2 alpha beta x_c * sum_{i : |i - c| <= half} dy_i x_i s_i^(-beta-1)
  float acc = 0.f, pc = 0.f;
  for (int i = max(0, c - half); i <= min(C - 1, c + half); ++i) {
    float s = 0.f;
    for (int j = max(0, i - half); j <= min(C - 1, i + half); ++j) s += xr[j] * xr[j];
    const float scale = k + alpha * s;
    const float p = exp2f(-beta * __log2f(scale));
    acc += dr[i] * xr[i] * p / scale;
    if (i == c) pc = p;
  }
  dx[idx] = dr[c] * pc - 2.f * alpha * beta * xr[c] * acc;
}

void lrn_fwd(const void* x, void* y, long long rows, int C, int n, float k, float alpha, float beta, int f32, cudaStream_t st) {
  if (f32) {
    lrn_fwd_f32_kernel<<<grid_for(rows * C, 256), 256, 0, st>>>((const float*)x, (float*)y, rows, C, n / 2, k, alpha, beta);
    count_launch(); TMPI_CHECK_LAUNCH("lrn_fwd"); ::tmpi::check_capture(st, "lrn_fwd");
    return;
  }
  if (C % 8) throw std::runtime_error("lrn: C must be a multiple of 8");
  const int half = n / 2;
  long long total = rows * (C / 8);
  if (total >= (1LL << 32)) throw std::runtime_error("lrn: tensor too large for 32-bit indexing");
  const int B = 256;
  auto X = (const __nv_bfloat16*)x; auto Y = (__nv_bfloat16*)y;
  switch (half) {
    case 1: lrn_fwd_kernel<1><<<grid_for(total, B), B, 0, st>>>(X, Y, rows, C, k, alpha, beta); break;
    case 2: lrn_fwd_kernel<2><<<grid_for(total, B), B, 0, st>>>(X, Y, rows, C, k, alpha, beta); break;
    case 3: lrn_fwd_kernel<3><<<grid_for(total, B), B, 0, st>>>(X, Y, rows, C, k, alpha, beta); break;
    case 4: lrn_fwd_kernel<4><<<grid_for(total, B), B, 0, st>>>(X, Y, rows, C, k, alpha, beta); break;
    default: throw std::runtime_error("lrn: window n must be 3,5,7 or 9");
  }
  count_launch(); TMPI_CHECK_LAUNCH("lrn_fwd"); ::tmpi::check_capture(st, "lrn_fwd");
}

void lrn_bwd(const void* x, const void* dy, void* dx, long long rows, int C, int n, float k, float alpha, float beta, int f32, cudaStream_t st) {
  if (f32) {
    lrn_bwd_f32_kernel<<<grid_for(rows * C, 256), 256, 0, st>>>((const float*)x, (const float*)dy, (float*)dx, rows, C, n / 2, k, alpha, beta);
    count_launch(); TMPI_CHECK_LAUNCH("lrn_bwd"); ::tmpi::check_capture(st, "lrn_bwd");
    return;
  }
  if (C % 8) throw std::runtime_error("lrn: C must be a multiple of 8");
  const int half = n / 2;
  long long total = rows * (C / 8);
  if (total >= (1LL << 32)) throw std::runtime_error("lrn: tensor too large for 32-bit indexing");
  const int B = 256;
  auto X = (const __nv_bfloat16*)x; auto DY = (const __nv_bfloat16*)dy; auto DX = (__nv_bfloat16*)dx;
  switch (half) {
    case 1: lrn_bwd_kernel<1><<<grid_for(total, B), B, 0, st>>>(X, DY, DX, rows, C, k, alpha, beta); break;
    case 2: lrn_bwd_kernel<2><<<grid_for(total, B), B, 0, st>>>(X, DY, DX, rows, C, k, alpha, beta); break;
    case 3: lrn_bwd_kernel<3><<<grid_for(total, B), B, 0, st>>>(X, DY, DX, rows, C, k, alpha, beta); break;
    case 4: lrn_bwd_kernel<4><<<grid_for(total, B), B, 0, st>>>(X, DY, DX, rows, C, k, alpha, beta); break;
    default: throw std::runtime_error("lrn: window n must be 3,5,7 or 9");
  }
  count_launch(); TMPI_CHECK_LAUNCH("lrn_bwd"); ::tmpi::check_capture(st, "lrn_bwd");
}

// ============================================================================ pooling
struct PoolGeom { int N, H, W, C, Ho, Wo, k, s, p; };

template <int MAXW, bool FUSE>      // defined with the fused conv→pool backward further down
__global__ void maxpool_relu_bias_bwd_kernel(const __nv_bfloat16* __restrict__ dyp, const uint8_t* __restrict__ arg,
                                             const __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ dym,
                                             float* __restrict__ db0, float* __restrict__ db1, int c_split, PoolGeom g, int VT);

// One CTA per output row (n, ho): (n, ho) come from blockIdx, threads sweep (wo, channel vector) — no per-thread
// division chain, 32-bit offsets inside the row (the one-thread-per-output version was instruction bound at 2.5x the
// memory roofline).  K > 0: compile-time window size (unrolled), K == 0: generic.
template <int K>
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                          uint8_t* __restrict__ arg, PoolGeom g) {
  const int k = K > 0 ? K : g.k;
  const int nvec = g.C >> 3;
  const int ho = blockIdx.x % g.Ho, n = blockIdx.x / g.Ho;
  const int h0 = ho * g.s - g.p;
  const __nv_bfloat16* xin = x + (long long)n * g.H * g.W * g.C;
  const long long orow = ((long long)n * g.Ho + ho) * g.Wo * g.C;
  const int items = g.Wo * nvec;
  for (int it = threadIdx.x; it < items; it += blockDim.x) {
    const int wo = it / nvec, cv = it - wo * nvec;
    const int w0 = wo * g.s - g.p;
    // running max and its window index stay PACKED (two bf16 / two 16-bit indices per register): one __hgt2_mask and two
    // bit-selects per register and tap instead of unpack + compare + two selects per channel
    uint32_t best[4], bidx[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { best[i] = 0xFF80FF80u; bidx[i] = 0u; }          // -inf, index 0
#pragma unroll
    for (int kh = 0; kh < (K > 0 ? K : 1); ++kh) {
      for (int kh2 = (K > 0 ? kh : 0); kh2 < (K > 0 ? kh + 1 : k); ++kh2) {
        const int h = h0 + kh2;
        if (h < 0 || h >= g.H) continue;
#pragma unroll
        for (int kw = 0; kw < (K > 0 ? K : 1); ++kw) {
          for (int kw2 = (K > 0 ? kw : 0); kw2 < (K > 0 ? kw + 1 : k); ++kw2) {
            const int w = w0 + kw2;
            if (w < 0 || w >= g.W) continue;
            const bf16x8 v = *reinterpret_cast<const bf16x8*>(xin + ((unsigned)(h * g.W + w) * (unsigned)g.C + cv * 8));
            const uint32_t* vw = reinterpret_cast<const uint32_t*>(&v);
            const uint32_t tt = (uint32_t)(kh2 * k + kw2) * 0x00010001u;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const uint32_t m = __hgt2_mask(*reinterpret_cast<const __nv_bfloat162*>(&vw[i]), *reinterpret_cast<const __nv_bfloat162*>(&best[i]));
              best[i] = (vw[i] & m) | (best[i] & ~m);
              bidx[i] = (tt & m) | (bidx[i] & ~m);
            }
          }
        }
      }
    }
    const long long o = orow + (unsigned)(wo * g.C + cv * 8);
    *reinterpret_cast<uint4*>(y + o) = make_uint4(best[0], best[1], best[2], best[3]);
    uint2 packed;                                   // 8 window indices, one byte per channel
    packed.x = __byte_perm(bidx[0], bidx[1], 0x6420);
    packed.y = __byte_perm(bidx[2], bidx[3], 0x6420);
    *reinterpret_cast<uint2*>(arg + o) = packed;
  }
}

// fp32 max pooling: one thread per output vector with plain compares (the packed-bf16 compare above has no fp32 counterpart)
__global__ void maxpool_fwd_f32_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ arg, PoolGeom g) {
  const int nvec = g.C >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)g.N * g.Ho * g.Wo * nvec;
  if (idx >= total) return;
  const int cv = (int)(idx % nvec); long long t = idx / nvec;
  const int wo = (int)(t % g.Wo); t /= g.Wo;
  const int ho = (int)(t % g.Ho); const int n = (int)(t / g.Ho);
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  uint32_t bi[4] = {0u, 0u, 0u, 0u};
  for (int kh = 0; kh < g.k; ++kh) {
    const int h = ho * g.s - g.p + kh;
    if (h < 0 || h >= g.H) continue;
    for (int kw = 0; kw < g.k; ++kw) {
      const int w = wo * g.s - g.p + kw;
      if (w < 0 || w >= g.W) continue;
      float v[4];
      VecIO<float>::ld(x + (((long long)n * g.H + h) * g.W + w) * g.C + cv * 4, v);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (v[i] > best[i]) { best[i] = v[i]; bi[i] = (uint32_t)(kh * g.k + kw); }
    }
  }
  const long long o = (((long long)n * g.Ho + ho) * g.Wo + wo) * g.C + cv * 4;
  VecIO<float>::st(y + o, best);
  *reinterpret_cast<uint32_t*>(arg + o) = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
}

template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ arg, T* __restrict__ dx, PoolGeom g) {
  constexpr int N = VecIO<T>::N;
  const int nvec = g.C >> VecIO<T>::LOG2N;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;             // host guarantees total < 2^32
  const unsigned total = (unsigned)g.N * g.H * g.W * nvec;
  if (idx >= total) return;
  const int cv = (int)(idx % (unsigned)nvec); unsigned t = idx / (unsigned)nvec;
  const int w = (int)(t % g.W); t /= g.W;
  const int h = (int)(t % g.H); const int n = (int)(t / g.H);
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  // outputs whose window covers (h, w): ho*s - p <= h < ho*s - p + k
  int ho_lo = (h + g.p - g.k + g.s) / g.s; if (h + g.p - g.k + 1 <= 0) ho_lo = 0;
  int wo_lo = (w + g.p - g.k + g.s) / g.s; if (w + g.p - g.k + 1 <= 0) wo_lo = 0;
  const int ho_hi = min(g.Ho - 1, (h + g.p) / g.s);
  const int wo_hi = min(g.Wo - 1, (w + g.p) / g.s);
  for (int ho = ho_lo; ho <= ho_hi; ++ho) {
    const int kh = h + g.p - ho * g.s;
    if (kh < 0 || kh >= g.k) continue;
    for (int wo = wo_lo; wo <= wo_hi; ++wo) {
      const int kw = w + g.p - wo * g.s;
      if (kw < 0 || kw >= g.k) continue;
      const long long o = (((long long)n * g.Ho + ho) * g.Wo + wo) * g.C + cv * N;
      const uint2 a = ld_flags<N>(arg + o);
      float d[N];
      VecIO<T>::ld(dy + o, d);
      const uint32_t me = (uint32_t)(kh * g.k + kw);
#pragma unroll
      for (int i = 0; i < N; ++i) {
        const uint32_t ai = ((i < 4 ? a.x : a.y) >> (8 * (i & 3))) & 0xFFu;
        if (ai == me) acc[i] += d[i];
      }
    }
  }
  VecIO<T>::st(dx + (((long long)n * g.H + h) * g.W + w) * g.C + cv * N, acc);
}

__device__ __forceinline__ int avg_count(const PoolGeom& g, int ho, int wo) {
  const int h0 = max(0, ho * g.s - g.p), h1 = min(g.H, ho * g.s - g.p + g.k);
  const int w0 = max(0, wo * g.s - g.p), w1 = min(g.W, wo * g.s - g.p + g.k);
  return max(1, (h1 - h0) * (w1 - w0));
}

template <typename T>
__global__ void avgpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, PoolGeom g) {
  constexpr int N = VecIO<T>::N;
  const int nvec = g.C >> VecIO<T>::LOG2N;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;             // host guarantees total < 2^32
  const unsigned total = (unsigned)g.N * g.Ho * g.Wo * nvec;
  if (idx >= total) return;
  const int cv = (int)(idx % (unsigned)nvec); unsigned t = idx / (unsigned)nvec;
  const int wo = (int)(t % g.Wo); t /= g.Wo;
  const int ho = (int)(t % g.Ho); const int n = (int)(t / g.Ho);
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  for (int kh = 0; kh < g.k; ++kh) {
    const int h = ho * g.s - g.p + kh;
    if (h < 0 || h >= g.H) continue;
    for (int kw = 0; kw < g.k; ++kw) {
      const int w = wo * g.s - g.p + kw;
      if (w < 0 || w >= g.W) continue;
      float v[N];
      VecIO<T>::ld(x + (((long long)n * g.H + h) * g.W + w) * g.C + cv * N, v);
#pragma unroll
      for (int i = 0; i < N; ++i) acc[i] += v[i];
    }
  }
  const float inv = 1.f / (float)avg_count(g, ho, wo);
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] *= inv;
  VecIO<T>::st(y + (((long long)n * g.Ho + ho) * g.Wo + wo) * g.C + cv * N, acc);
}

template <typename T>
__global__ void avgpool_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, PoolGeom g) {
  constexpr int N = VecIO<T>::N;
  const int nvec = g.C >> VecIO<T>::LOG2N;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;             // host guarantees total < 2^32
  const unsigned total = (unsigned)g.N * g.H * g.W * nvec;
  if (idx >= total) return;
  const int cv = (int)(idx % (unsigned)nvec); unsigned t = idx / (unsigned)nvec;
  const int w = (int)(t % g.W); t /= g.W;
  const int h = (int)(t % g.H); const int n = (int)(t / g.H);
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  const int ho_hi = min(g.Ho - 1, (h + g.p) / g.s);
  const int wo_hi = min(g.Wo - 1, (w + g.p) / g.s);
  for (int ho = 0; ho <= ho_hi; ++ho) {
    const int kh = h + g.p - ho * g.s;
    if (kh < 0 || kh >= g.k) continue;
    for (int wo = 0; wo <= wo_hi; ++wo) {
      const int kw = w + g.p - wo * g.s;
      if (kw < 0 || kw >= g.k) continue;
      float d[N];
      VecIO<T>::ld(dy + (((long long)n * g.Ho + ho) * g.Wo + wo) * g.C + cv * N, d);
      const float inv = 1.f / (float)avg_count(g, ho, wo);
#pragma unroll
      for (int i = 0; i < N; ++i) acc[i] += d[i] * inv;
    }
  }
  VecIO<T>::st(dx + (((long long)n * g.H + h) * g.W + w) * g.C + cv * N, acc);
}

static void need_vec(int C, int f32, const char* what) {
  if (C % (f32 ? 4 : 8)) throw std::runtime_error(std::string(what) + (f32 ? ": C must be a multiple of 4" : ": C must be a multiple of 8"));
}

void pool_fwd(const void* x, void* y, void* arg, int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p, int is_max, int f32,
              cudaStream_t st) {
  need_vec(C, f32, "pool");
  PoolGeom g{N, H, W, C, Ho, Wo, k, s, p};
  const int nvec = f32 ? C / 4 : C / 8;
  const long long total = (long long)N * Ho * Wo * nvec;
  if ((long long)N * H * W * nvec >= (1LL << 32)) throw std::runtime_error("pool: tensor too large for 32-bit indexing");
  if (!f32 && (long long)H * W * C >= (1LL << 31)) throw std::runtime_error("pool: image too large for 32-bit in-image offsets");
  if (is_max && f32) {
    maxpool_fwd_f32_kernel<<<grid_for(total, 256), 256, 0, st>>>((const float*)x, (float*)y, (uint8_t*)arg, g);
  } else if (is_max) {
    const unsigned rows = (unsigned)N * Ho;
    auto X = (const __nv_bfloat16*)x; auto Y = (__nv_bfloat16*)y; auto A = (uint8_t*)arg;
    if (k == 3) maxpool_fwd_kernel<3><<<rows, 256, 0, st>>>(X, Y, A, g);
    else if (k == 2) maxpool_fwd_kernel<2><<<rows, 256, 0, st>>>(X, Y, A, g);
    else maxpool_fwd_kernel<0><<<rows, 256, 0, st>>>(X, Y, A, g);
  } else if (f32) {
    avgpool_fwd_kernel<float><<<grid_for(total, 256), 256, 0, st>>>((const float*)x, (float*)y, g);
  } else {
    avgpool_fwd_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, g);
  }
  count_launch(); TMPI_CHECK_LAUNCH("pool_fwd"); ::tmpi::check_capture(st, "pool_fwd");
}

void pool_bwd(const void* dy, const void* arg, void* dx, int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p, int is_max, int f32,
              cudaStream_t st) {
  need_vec(C, f32, "pool");
  PoolGeom g{N, H, W, C, Ho, Wo, k, s, p};
  const long long total = (long long)N * H * W * (f32 ? C / 4 : C / 8);
  const int maxw = (k + s - 1) / s;
  const auto A = (const uint8_t*)arg;
  if (f32) {
    if (is_max) maxpool_bwd_kernel<float><<<grid_for(total, 256), 256, 0, st>>>((const float*)dy, A, (float*)dx, g);
    else avgpool_bwd_kernel<float><<<grid_for(total, 256), 256, 0, st>>>((const float*)dy, (float*)dx, g);
  } else if (is_max && maxw <= 3 && (long long)H * W * C < (1LL << 31)) {
    // row-per-CTA kernel shared with the fused conv→pool backward (all candidate windows in flight at once)
    const int nvec = C / 8;
    const int VT = nvec < 32 ? nvec : 32;
    dim3 grid((unsigned)N * H, (unsigned)((nvec + VT - 1) / VT));
    auto DY = (const __nv_bfloat16*)dy; auto DX = (__nv_bfloat16*)dx;
    if (maxw == 1) maxpool_relu_bias_bwd_kernel<1, false><<<grid, 256, 0, st>>>(DY, A, nullptr, DX, nullptr, nullptr, C, g, VT);
    else if (maxw == 2) maxpool_relu_bias_bwd_kernel<2, false><<<grid, 256, 0, st>>>(DY, A, nullptr, DX, nullptr, nullptr, C, g, VT);
    else maxpool_relu_bias_bwd_kernel<3, false><<<grid, 256, 0, st>>>(DY, A, nullptr, DX, nullptr, nullptr, C, g, VT);
  } else if (is_max) {
    maxpool_bwd_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, st>>>((const __nv_bfloat16*)dy, A, (__nv_bfloat16*)dx, g);
  } else {
    avgpool_bwd_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, st>>>((const __nv_bfloat16*)dy, (__nv_bfloat16*)dx, g);
  }
  count_launch(); TMPI_CHECK_LAUNCH("pool_bwd"); ::tmpi::check_capture(st, "pool_bwd");
}

// ============================================================================ dropout (Philox4x32-10)
__device__ __forceinline__ void philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// y = x * keep; keep drawn with P(keep) = 1 - p_drop from Philox keyed by (seed, layer) and counter (idx, *step).  One counter
// draws 8 keep bits, so a thread handles 8 elements in both storage types (one bf16 vector or two fp32 vectors).
template <typename T>
__global__ void dropout_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, uint8_t* __restrict__ mask,
                                   long long n8, float p_drop, unsigned long long seed, uint32_t layer,
                                   const unsigned long long* __restrict__ step) {
  constexpr int N = VecIO<T>::N;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n8) return;
  const unsigned long long stp = *step;
  uint32_t r[4];
  philox4x32((uint32_t)idx, (uint32_t)(idx >> 32), (uint32_t)stp, (uint32_t)(stp >> 32), (uint32_t)seed,
             (uint32_t)(seed >> 32) ^ (layer * 0x9E3779B9u), r);
  const uint32_t thr = (uint32_t)(p_drop * 65536.f);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; j += N) VecIO<T>::ld(x + idx * 8 + j, v + j);
  uint32_t mlo = 0, mhi = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t u = (r[i >> 1] >> (16 * (i & 1))) & 0xFFFFu;
    const uint32_t keep = u >= thr ? 1u : 0u;
    v[i] = keep ? v[i] : 0.f;
    if (i < 4) mlo |= keep << (8 * i); else mhi |= keep << (8 * (i - 4));
  }
#pragma unroll
  for (int j = 0; j < 8; j += N) VecIO<T>::st(y + idx * 8 + j, v + j);
  *reinterpret_cast<uint2*>(mask + idx * 8) = make_uint2(mlo, mhi);
}

template <typename T>
__global__ void dropout_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ mask, T* __restrict__ dx, long long nv) {
  constexpr int N = VecIO<T>::N;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nv) return;
  float v[N];
  VecIO<T>::ld(dy + idx * N, v);
  const uint2 m = ld_flags<N>(mask + idx * N);
#pragma unroll
  for (int i = 0; i < N; ++i) { const uint32_t k = ((i < 4 ? m.x : m.y) >> (8 * (i & 3))) & 0xFFu; if (!k) v[i] = 0.f; }
  VecIO<T>::st(dx + idx * N, v);
}

__global__ void advance_step_kernel(unsigned long long* step) { if (threadIdx.x == 0 && blockIdx.x == 0) *step += 1ull; }

void dropout_fwd(const void* x, void* y, void* mask, long long n, float p_drop, unsigned long long seed, int layer, const void* step, int f32,
                 cudaStream_t st) {
  if (n % 8) throw std::runtime_error("dropout: numel must be a multiple of 8");
  auto M = (uint8_t*)mask; auto S = (const unsigned long long*)step;
  if (f32) dropout_fwd_kernel<float><<<grid_for(n / 8, 256), 256, 0, st>>>((const float*)x, (float*)y, M, n / 8, p_drop, seed, (uint32_t)layer, S);
  else dropout_fwd_kernel<__nv_bfloat16><<<grid_for(n / 8, 256), 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, M, n / 8, p_drop,
                                                                                 seed, (uint32_t)layer, S);
  count_launch(); TMPI_CHECK_LAUNCH("dropout_fwd"); ::tmpi::check_capture(st, "dropout_fwd");
}
void dropout_bwd(const void* dy, const void* mask, void* dx, long long n, int f32, cudaStream_t st) {
  auto M = (const uint8_t*)mask;
  if (f32) dropout_bwd_kernel<float><<<grid_for(n / 4, 256), 256, 0, st>>>((const float*)dy, M, (float*)dx, n / 4);
  else dropout_bwd_kernel<__nv_bfloat16><<<grid_for(n / 8, 256), 256, 0, st>>>((const __nv_bfloat16*)dy, M, (__nv_bfloat16*)dx, n / 8);
  count_launch(); TMPI_CHECK_LAUNCH("dropout_bwd"); ::tmpi::check_capture(st, "dropout_bwd");
}
void advance_step(void* step, cudaStream_t st) {
  advance_step_kernel<<<1, 32, 0, st>>>((unsigned long long*)step);
  count_launch(); TMPI_CHECK_LAUNCH("advance_step"); ::tmpi::check_capture(st, "advance_step");
}

// Uniform [0, 1) noise (GAN generator input): element i is word i % 4 of Philox(counter = (i / 4, *step), key = (seed, stream)),
// scaled by 2^-24 after dropping the low 8 bits — ops/reference.py: uniform_noise draws the same numbers on the CPU.  The step is
// read from device memory, so a replayed CUDA graph draws fresh noise.
template <typename T>
__global__ void uniform_noise_kernel(T* __restrict__ out, long long n, unsigned long long seed, uint32_t stream,
                                     const unsigned long long* __restrict__ step) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q * 4 >= n) return;
  const unsigned long long stp = *step;
  uint32_t r[4];
  philox4x32((uint32_t)q, (uint32_t)(q >> 32), (uint32_t)stp, (uint32_t)(stp >> 32), (uint32_t)seed, (uint32_t)(seed >> 32) ^ stream, r);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (q * 4 + j < n) out[q * 4 + j] = from_f<T>((float)(r[j] >> 8) * (1.f / 16777216.f));
}
void uniform_noise(void* out, long long n, unsigned long long seed, int stream, const void* step, int f32, cudaStream_t st) {
  const int g = grid_for((n + 3) / 4, 256);
  auto S = (const unsigned long long*)step;
  if (f32) uniform_noise_kernel<float><<<g, 256, 0, st>>>((float*)out, n, seed, (uint32_t)stream, S);
  else uniform_noise_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((__nv_bfloat16*)out, n, seed, (uint32_t)stream, S);
  count_launch(); TMPI_CHECK_LAUNCH("uniform_noise"); ::tmpi::check_capture(st, "uniform_noise");
}

// ============================================================================ GAN losses over a [B] score vector, + dscores
// kind 0 (Wasserstein):   loss = a * mean(o),               d = a / B          (a = +1 fake / -1 real for the critic, -1 generator)
// kind 1 (least squares): loss = 0.5 * mean((o - a)^2),     d = (o - a) / B    (a = target: 1 real / 0 fake, generator 1)
// One CTA: B is the batch size.  out[0] = loss (device scalar, no host sync).
template <typename T>
__global__ void __launch_bounds__(256) gan_loss_kernel(const T* __restrict__ o, T* __restrict__ d, float* __restrict__ out, int B, int kind,
                                                       float a) {
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float invB = 1.f / (float)B;
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float v = to_f(o[i]);
    if (kind == 0) { s += v; d[i] = from_f<T>(a * invB); }
    else { const float e = v - a; s += e * e; d[i] = from_f<T>(e * invB); }
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (warp == 0) {
    float v = lane < nw ? red[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) out[0] = kind == 0 ? a * v * invB : 0.5f * v * invB;
  }
}
void gan_loss(const void* scores, void* dscores, void* out, int B, int kind, float a, int f32, cudaStream_t st) {
  if (kind != 0 && kind != 1) throw std::runtime_error("gan_loss: kind must be 0 (wgan) or 1 (lsgan)");
  if (f32) gan_loss_kernel<float><<<1, 256, 0, st>>>((const float*)scores, (float*)dscores, (float*)out, B, kind, a);
  else gan_loss_kernel<__nv_bfloat16><<<1, 256, 0, st>>>((const __nv_bfloat16*)scores, (__nv_bfloat16*)dscores, (float*)out, B, kind, a);
  count_launch(); TMPI_CHECK_LAUNCH("gan_loss"); ::tmpi::check_capture(st, "gan_loss");
}

// ============================================================================ softmax + NLL + errors + dlogits
// one CTA per row; rowstat[b] = {nll, err1, err5}; dlogits = (softmax - onehot) * scale
// kSmooth (label smoothing ε): the target is q = on·onehot + off with on = 1 − ε, off = ε / C, so rowstat[3b] is the soft-target
// cross-entropy −Σ q·log p = log se − on·(z_y − max) − off·Σ(z − max) and dlogits = (softmax − q) * scale; err1 / err5 are unchanged
template <typename T, bool kSmooth>
__global__ void softmax_xent_kernel(const T* __restrict__ logits, const long long* __restrict__ labels,
                                    T* __restrict__ dlogits, float* __restrict__ rowstat, int C, float scale, float on, float off) {
  const int b = blockIdx.x;
  const T* row = logits + (long long)b * C;
  const int label = (int)labels[b];
  __shared__ float red[32];
  __shared__ float bcast;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, to_f(row[c]));
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : -INFINITY; v = warp_max(v); if (lane == 0) bcast = v; }
  __syncthreads();
  mx = bcast;
  __syncthreads();
  const float lab = to_f(row[label]);
  float se = 0.f, gt = 0.f, sz = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = to_f(row[c]);
    se += __expf(v - mx);
    gt += (v > lab || (v == lab && c < label)) ? 1.f : 0.f;     // rank of the label's logit
    if constexpr (kSmooth) sz += v - mx;
  }
  se = warp_sum(se); gt = warp_sum(gt);
  if (lane == 0) { red[warp] = se; }
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; v = warp_sum(v); if (lane == 0) bcast = v; }
  __syncthreads();
  se = bcast;
  __syncthreads();
  if (lane == 0) { red[warp] = gt; }
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; v = warp_sum(v); if (lane == 0) bcast = v; }
  __syncthreads();
  gt = bcast;
  if constexpr (kSmooth) {                                      // Σ(z − max) to thread 0 (red is free: its last readers passed the barrier)
    sz = warp_sum(sz);
    if (lane == 0) red[warp] = sz;
    __syncthreads();
    if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; sz = warp_sum(v); }
  }
  const float inv = 1.f / se;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float pr = __expf(to_f(row[c]) - mx) * inv;
    if constexpr (kSmooth) { pr -= off; if (c == label) pr -= on; }
    else { if (c == label) pr -= 1.f; }
    dlogits[(long long)b * C + c] = from_f<T>(pr * scale);
  }
  if (threadIdx.x == 0) {
    if constexpr (kSmooth) rowstat[3 * b + 0] = __logf(se) - on * (lab - mx) - off * sz;
    else rowstat[3 * b + 0] = -(lab - mx - __logf(se));
    rowstat[3 * b + 1] = gt >= 1.f ? 1.f : 0.f;
    rowstat[3 * b + 2] = gt >= 5.f ? 1.f : 0.f;
  }
}

__global__ void rowstat_mean_kernel(const float* __restrict__ rowstat, float* __restrict__ out, int B, float weight) {
  __shared__ float red[3][32];
  float a = 0.f, b = 0.f, c = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) { a += rowstat[3 * i]; b += rowstat[3 * i + 1]; c += rowstat[3 * i + 2]; }
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { red[0][warp] = a; red[1][warp] = b; red[2][warp] = c; }
  __syncthreads();
  if (warp == 0) {
    a = lane < nw ? red[0][lane] : 0.f; b = lane < nw ? red[1][lane] : 0.f; c = lane < nw ? red[2][lane] : 0.f;
    a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
    if (lane == 0) { out[0] = weight * a / B; out[1] = b / B; out[2] = c / B; }
  }
}

// the reported loss carries `weight`, the gradient `grad_weight` (weight / n under gradient accumulation over n micro-batches);
// label_smoothing ε = 0 runs the plain NLL instantiation, ε in (0, 1] the soft-target one
void softmax_xent(const void* logits, const void* labels, void* dlogits, void* rowstat, void* out3, int B, int C, float weight,
                  float grad_weight, float label_smoothing, int f32, cudaStream_t st) {
  if (!(label_smoothing >= 0.f && label_smoothing <= 1.f)) throw std::runtime_error("softmax_xent: label_smoothing must be in [0, 1]");
  auto LB = (const long long*)labels; auto RS = (float*)rowstat;
  const float scale = grad_weight / (float)B;
  const bool smooth = label_smoothing != 0.f;
  const float on = 1.f - label_smoothing, off = label_smoothing / (float)C;
  if (f32) {
    auto k = smooth ? softmax_xent_kernel<float, true> : softmax_xent_kernel<float, false>;
    k<<<B, 256, 0, st>>>((const float*)logits, LB, (float*)dlogits, RS, C, scale, on, off);
  } else {
    auto k = smooth ? softmax_xent_kernel<__nv_bfloat16, true> : softmax_xent_kernel<__nv_bfloat16, false>;
    k<<<B, 256, 0, st>>>((const __nv_bfloat16*)logits, LB, (__nv_bfloat16*)dlogits, RS, C, scale, on, off);
  }
  count_launch(); TMPI_CHECK_LAUNCH("softmax_xent"); ::tmpi::check_capture(st, "softmax_xent");
  rowstat_mean_kernel<<<1, 256, 0, st>>>((const float*)rowstat, (float*)out3, B, weight);
  count_launch(); TMPI_CHECK_LAUNCH("rowstat_mean"); ::tmpi::check_capture(st, "rowstat_mean");
}

// ============================================================================ multi-view validation: averaged softmax + metrics
// One CTA per row b.  View v's max-shifted fp32 softmax p_v of the logits is stored into (v = 0) or added to (v > 0) the fp32
// accumulator acc[b, :], each element by the thread that owns column c in every view, so the sum runs in view order.  On the last view
// the same launch divides by V (an IEEE division), leaving p̄ = (1/V)·Σ p_v in acc, and writes rowstat[b] = {−log max(p̄_y, FLT_MIN),
// rank ≥ 1, rank ≥ 5} with rank = #{p̄_c > p̄_y} + #{c < y : p̄_c = p̄_y}, the rank rule of softmax_xent_kernel.
template <typename T>
__global__ void view_softmax_accum_kernel(const T* __restrict__ logits, const long long* __restrict__ labels, float* __restrict__ acc,
                                          float* __restrict__ rowstat, int C, int v, int V) {
  const int b = blockIdx.x;
  const T* row = logits + (long long)b * C;
  float* a = acc + (long long)b * C;
  __shared__ float red[32];
  __shared__ float bcast;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, to_f(row[c]));
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? red[lane] : -INFINITY; t = warp_max(t); if (lane == 0) bcast = t; }
  __syncthreads();
  mx = bcast;
  __syncthreads();
  float se = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) se += __expf(to_f(row[c]) - mx);
  se = warp_sum(se);
  if (lane == 0) red[warp] = se;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? red[lane] : 0.f; t = warp_sum(t); if (lane == 0) bcast = t; }
  __syncthreads();
  const float inv = 1.f / bcast;
  const bool last = v == V - 1;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = __expf(to_f(row[c]) - mx) * inv;
    if (v > 0) s += a[c];
    if (last) s = __fdiv_rn(s, (float)V);
    a[c] = s;
  }
  if (!last) return;                                            // CTA-uniform
  __syncthreads();                                              // p̄ of the whole row written (global writes visible to the CTA)
  const int label = (int)labels[b];
  const float py = a[label];
  float gt = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float p = a[c];
    gt += (p > py || (p == py && c < label)) ? 1.f : 0.f;
  }
  gt = warp_sum(gt);
  if (lane == 0) red[warp] = gt;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nw ? red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) {
      rowstat[3 * b + 0] = -__logf(fmaxf(py, FLT_MIN));
      rowstat[3 * b + 1] = t >= 1.f ? 1.f : 0.f;
      rowstat[3 * b + 2] = t >= 5.f ? 1.f : 0.f;
    }
  }
}

void view_softmax_accum(const void* logits, const void* labels, void* acc, void* rowstat, void* out3, int B, int C, int v, int V, int f32,
                        cudaStream_t st) {
  if (!(V >= 1 && v >= 0 && v < V)) throw std::runtime_error("view_softmax_accum: needs 0 <= v < V");
  auto LB = (const long long*)labels; auto A = (float*)acc; auto RS = (float*)rowstat;
  if (f32) view_softmax_accum_kernel<float><<<B, 256, 0, st>>>((const float*)logits, LB, A, RS, C, v, V);
  else view_softmax_accum_kernel<__nv_bfloat16><<<B, 256, 0, st>>>((const __nv_bfloat16*)logits, LB, A, RS, C, v, V);
  count_launch(); TMPI_CHECK_LAUNCH("view_softmax_accum"); ::tmpi::check_capture(st, "view_softmax_accum");
  if (v != V - 1) return;
  rowstat_mean_kernel<<<1, 256, 0, st>>>((const float*)rowstat, (float*)out3, B, 1.f);
  count_launch(); TMPI_CHECK_LAUNCH("rowstat_mean"); ::tmpi::check_capture(st, "rowstat_mean");
}

// ============================================================================ Mixup / CutMix
// The draw of one step (ops/reference.py: mix_draw is the same on the host).  Philox4x32-10 with key (seed_lo, seed_hi ^ rank) and
// counter (j, 0xFFFFFFFF, step_lo, step_hi), j the block index within the step.  Dropout's and uniform_noise's second counter word
// is the high word of a non-negative 64-bit element index, at most 0x7FFFFFFF, so none of their blocks is ever one of these,
// whatever the keys.  Blocks: j = 0 the gate, switch and centre words; j = 1 the two U^(1/α) boosts; j = 2 + k attempt k of the
// Gamma draw X, j = 2 + kMixAttempts + k attempt k of Y.  Every correctly rounded fp64 operation is an _rn intrinsic, so
// --use_fast_math cannot contract it; log, cos and pow are the libdevice functions.
constexpr int kMixAttempts = 16;         // Marsaglia–Tsang accepts ≥ 95 % of attempts: running out is ~1e-21 per variate
constexpr uint32_t kMixCounterTag = 0xFFFFFFFFu;

__device__ __forceinline__ double mix_u01(uint32_t w) { return __dmul_rn(__dadd_rn((double)w, 0.5), 2.3283064365386963e-10); }  // (0, 1)

// Gamma(a) by Marsaglia–Tsang from Box–Muller normals (a < 1: Gamma(a + 1)·U^(1/a)); false if every attempt was rejected
__device__ bool mix_gamma(double a, double boost_u, uint32_t j0, uint32_t s_lo, uint32_t s_hi, uint32_t k0, uint32_t k1, double* out) {
  const double ae = a < 1.0 ? __dadd_rn(a, 1.0) : a;
  const double d = __dsub_rn(ae, 1.0 / 3.0);
  const double c = __ddiv_rn(1.0, __dsqrt_rn(__dmul_rn(9.0, d)));
  for (int k = 0; k < kMixAttempts; ++k) {
    uint32_t r[4];
    philox4x32(j0 + (uint32_t)k, kMixCounterTag, s_lo, s_hi, k0, k1, r);
    const double x = __dmul_rn(__dsqrt_rn(__dmul_rn(-2.0, log(mix_u01(r[0])))), cos(__dmul_rn(6.283185307179586, mix_u01(r[1]))));
    double v = __dadd_rn(1.0, __dmul_rn(c, x));
    if (v <= 0.0) continue;
    v = __dmul_rn(__dmul_rn(v, v), v);
    const double u = mix_u01(r[2]), x2 = __dmul_rn(x, x);
    if (u < __dsub_rn(1.0, __dmul_rn(__dmul_rn(0.0331, x2), x2)) ||
        log(u) < __dadd_rn(__dmul_rn(0.5, x2), __dmul_rn(d, __dadd_rn(__dsub_rn(1.0, v), log(v))))) {
      double g = __dmul_rn(d, v);
      if (a < 1.0) g = __dmul_rn(g, pow(boost_u, __ddiv_rn(1.0, a)));
      *out = g;
      return true;
    }
  }
  return false;
}

__global__ void mix_draw_kernel(MixParams p, const unsigned long long* __restrict__ step, MixRecord* __restrict__ rec, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long s = *step + (unsigned long long)t;
  const uint32_t s_lo = (uint32_t)s, s_hi = (uint32_t)(s >> 32);
  const uint32_t k0 = (uint32_t)p.seed, k1 = (uint32_t)(p.seed >> 32) ^ (uint32_t)p.rank;
  MixRecord r = {};
  r.mode = MIX_NONE; r.lam = 1.f; r.lam_raw = 1.0; r.H = p.H; r.W = p.W;
  uint32_t w0[4], w1[4];
  philox4x32(0u, kMixCounterTag, s_lo, s_hi, k0, k1, w0);
  if (mix_u01(w0[0]) < p.prob) {
    const bool both = p.alpha > 0.0 && p.cutmix_alpha > 0.0;
    const int mode = both ? (mix_u01(w0[1]) < p.switch_prob ? MIX_CUTMIX : MIX_MIXUP) : (p.cutmix_alpha > 0.0 ? MIX_CUTMIX : MIX_MIXUP);
    const double a = mode == MIX_CUTMIX ? p.cutmix_alpha : p.alpha;
    philox4x32(1u, kMixCounterTag, s_lo, s_hi, k0, k1, w1);
    double gx, gy;
    if (mix_gamma(a, mix_u01(w1[0]), 2u, s_lo, s_hi, k0, k1, &gx) &&
        mix_gamma(a, mix_u01(w1[1]), 2u + kMixAttempts, s_lo, s_hi, k0, k1, &gy)) {
      const double sum = __dadd_rn(gx, gy);
      const double lam = sum > 0.0 ? __ddiv_rn(gx, sum) : 0.5;
      r.mode = mode; r.lam_raw = lam;
      if (mode == MIX_MIXUP) {
        r.lam = __double2float_rn(lam);
      } else {
        const double cut = __dsqrt_rn(__dsub_rn(1.0, lam));
        const int ch = (int)__dmul_rn((double)p.H, cut), cw = (int)__dmul_rn((double)p.W, cut);
        r.cy = (int)(((unsigned long long)w0[2] * (unsigned)p.H) >> 32);
        r.cx = (int)(((unsigned long long)w0[3] * (unsigned)p.W) >> 32);
        r.y0 = min(max(r.cy - ch / 2, 0), p.H); r.y1 = min(max(r.cy + ch / 2, 0), p.H);
        r.x0 = min(max(r.cx - cw / 2, 0), p.W); r.x1 = min(max(r.cx + cw / 2, 0), p.W);
        const long long area = (long long)(r.y1 - r.y0) * (r.x1 - r.x0);
        r.lam = __double2float_rn(__dsub_rn(1.0, __ddiv_rn((double)area, (double)((long long)p.H * p.W))));
      }
    }
  }
  rec[t] = r;
}

void mix_draw(const MixParams& p, const void* step, void* rec, int n, cudaStream_t st) {
  if (n < 1 || p.H < 1 || p.W < 1) throw std::runtime_error("mix_draw: needs n >= 1 and a positive image size");
  mix_draw_kernel<<<grid_for(n, 128), 128, 0, st>>>(p, (const unsigned long long*)step, (MixRecord*)rec, n);
  count_launch(); TMPI_CHECK_LAUNCH("mix_draw"); ::tmpi::check_capture(st, "mix_draw");
}

// ============================================================================ drop-path (stochastic depth) draw
// out[l·B + n] = 0 if block l drops sample n this step, else keep_scale[l] (ops/reference.py: drop_path_draw is the same on the
// host).  Philox4x32-10 with key (seed_lo, seed_hi ^ rank) and counter (n, l ^ kDropPathTag, step_lo, step_hi); the decision is
// (word0 >> 8) < thresh[l], i.e. u = (word0 >> 8)·2^-24 < p_l with thresh[l] = ⌈p_l·2^24⌉ computed exactly on the host.  The tag
// keeps the second counter word in [0xC0000000, 0xC000FFFF] (L < 2^16): dropout's and uniform_noise's second word is the high word
// of a non-negative 64-bit index (at most 0x7FFFFFFF) and the mix draw's is 0xFFFFFFFF, so no block of another stream is ever one
// of these, whatever the keys.
constexpr uint32_t kDropPathTag = 0xC0000000u;

__global__ void drop_path_draw_kernel(const uint32_t* __restrict__ thresh, const float* __restrict__ keep_scale, int L, int B,
                                      unsigned long long seed, uint32_t rank, const unsigned long long* __restrict__ step,
                                      float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= L * B) return;
  const int l = t / B, n = t - l * B;
  const unsigned long long s = *step;
  uint32_t r[4];
  philox4x32((uint32_t)n, (uint32_t)l ^ kDropPathTag, (uint32_t)s, (uint32_t)(s >> 32), (uint32_t)seed, (uint32_t)(seed >> 32) ^ rank, r);
  out[t] = (r[0] >> 8) < thresh[l] ? 0.f : keep_scale[l];
}

void drop_path_draw(const void* thresh, const void* keep_scale, int L, int B, unsigned long long seed, int rank, const void* step, void* out,
                    cudaStream_t st) {
  if (L < 1 || L > 65535 || B < 1 || (long long)L * B > 0x7FFFFFFF) throw std::runtime_error("drop_path_draw: needs 1 <= L <= 65535 blocks and B >= 1");
  drop_path_draw_kernel<<<grid_for((long long)L * B, 256), 256, 0, st>>>((const uint32_t*)thresh, (const float*)keep_scale, L, B, seed,
                                                                          (uint32_t)rank, (const unsigned long long*)step, (float*)out);
  count_launch(); TMPI_CHECK_LAUNCH("drop_path_draw"); ::tmpi::check_capture(st, "drop_path_draw");
}

// ============================================================================ CIFAR augmentation draw (cifar_augment)
// Image n's pad-and-crop offsets, flip and Cutout box of one step (ops/cifar_augment.py owns the layout; ops/reference.py:
// cifar_augment_draw is the same on the host).  Philox4x32-10 with key (seed_lo, seed_hi ^ rank): block 0 has counter
// (n, kCifarAugTag, step_lo, step_hi), block 1 (n, kCifarAugTag + 1, ...).  Each value is ⌊w·k / 2^32⌋: oy, ox ∈ [0, 2·pad] from
// block 0 words 0 and 1, flip = word 2 >> 31, Cutout centre cy ∈ [0, H) from word 3 and cx ∈ [0, W) from block 1 word 0.  The tag
// is neither dropout's / uniform_noise's second word (at most 0x7FFFFFFF), nor the mix draw's 0xFFFFFFFF, nor in drop-path's
// [0xC0000000, 0xC000FFFF], so no block of another stream is ever one of these.
// offs[n] = (oy − pad, ox − pad); box[n] = (y1, x1, y2 − y1, x2 − x1) with y1 = clamp(cy − L/2, 0, H), y2 = clamp(cy + L/2, 0, H)
// and the same for x (DeVries & Taylor's Cutout: an odd L cuts an (L − 1)-wide hole).
constexpr uint32_t kCifarAugTag = 0xA0000000u;

__global__ void cifar_augment_draw_kernel(int B, int pad, int L, int H, int W, unsigned long long seed, uint32_t rank,
                                          const unsigned long long* __restrict__ step, int2* __restrict__ offs,
                                          uint8_t* __restrict__ flips, int4* __restrict__ boxes) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= B) return;
  const unsigned long long s = *step;
  const uint32_t s_lo = (uint32_t)s, s_hi = (uint32_t)(s >> 32), k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32) ^ rank;
  uint32_t a[4], b[4];
  philox4x32((uint32_t)n, kCifarAugTag, s_lo, s_hi, k0, k1, a);
  philox4x32((uint32_t)n, kCifarAugTag + 1u, s_lo, s_hi, k0, k1, b);
  const unsigned k = 2u * (unsigned)pad + 1u;
  const int oy = (int)(((unsigned long long)a[0] * k) >> 32), ox = (int)(((unsigned long long)a[1] * k) >> 32);
  const int cy = (int)(((unsigned long long)a[3] * (unsigned)H) >> 32), cx = (int)(((unsigned long long)b[0] * (unsigned)W) >> 32);
  const int y1 = min(max(cy - L / 2, 0), H), y2 = min(max(cy + L / 2, 0), H);
  const int x1 = min(max(cx - L / 2, 0), W), x2 = min(max(cx + L / 2, 0), W);
  offs[n] = make_int2(oy - pad, ox - pad);
  flips[n] = (uint8_t)(a[2] >> 31);
  boxes[n] = make_int4(y1, x1, y2 - y1, x2 - x1);
}

void cifar_augment_draw(int B, int pad, int L, int H, int W, unsigned long long seed, int rank, const void* step, void* offs, void* flips,
                        void* boxes, cudaStream_t st) {
  if (B < 1 || H < 1 || W < 1 || pad < 0 || pad >= H || pad >= W || L < 0 || L > H || L > W)
    throw std::runtime_error("cifar_augment_draw: needs B >= 1, 0 <= pad < H, W and 0 <= cutout <= H, W");
  cifar_augment_draw_kernel<<<grid_for(B, 128), 128, 0, st>>>(B, pad, L, H, W, seed, (uint32_t)rank, (const unsigned long long*)step,
                                                              (int2*)offs, (uint8_t*)flips, (int4*)boxes);
  count_launch(); TMPI_CHECK_LAUNCH("cifar_augment_draw"); ::tmpi::check_capture(st, "cifar_augment_draw");
}

// One thread per element position of a pair (i, j = B − 1 − i), blockIdx.y = i: it reads both rows and writes both, so the mix is
// in place.  kVec: N-element 16-byte vectors (the row length n = H·W·C times sizeof(T) is a multiple of 16), else one element.  The
// grid is sized for Mixup; CutMix CTAs whose elements lie outside the box rows return before touching the batch.
template <typename T, bool kVec>
__global__ void __launch_bounds__(256) mix_batch_kernel(T* __restrict__ x, const MixRecord* __restrict__ rec, int B, int H, int W, int C) {
  constexpr int N = kVec ? VecIO<T>::N : 1;
  __shared__ MixRecord r;
  if (threadIdx.x == 0) r = *rec;
  __syncthreads();
  if (r.mode == MIX_NONE) return;
  const long long rowlen = (long long)W * C, n = rowlen * H;
  const long long cta0 = (long long)blockIdx.x * blockDim.x * N;
  if (r.mode == MIX_CUTMIX) {
    const long long cta1 = min(n, cta0 + (long long)blockDim.x * N) - 1;
    if (cta1 / rowlen < r.y0 || cta0 / rowlen >= r.y1) return;
  }
  const long long e0 = cta0 + (long long)threadIdx.x * N;
  if (e0 >= n) return;
  const int i = blockIdx.y, j = B - 1 - i;
  T* xi = x + (long long)i * n + e0;
  T* xj = x + (long long)j * n + e0;
  float a[N], b[N];
  if constexpr (kVec) { VecIO<T>::ld(xi, a); VecIO<T>::ld(xj, b); }
  else { a[0] = to_f(*xi); b[0] = to_f(*xj); }
  bool any = false;
  if (r.mode == MIX_MIXUP) {
    const float lam = r.lam, oml = __fsub_rn(1.f, lam);
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const float na = __fadd_rn(__fmul_rn(lam, a[k]), __fmul_rn(oml, b[k]));
      const float nb = __fadd_rn(__fmul_rn(lam, b[k]), __fmul_rn(oml, a[k]));
      a[k] = na; b[k] = nb;
    }
    any = true;
  } else {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const long long e = e0 + k;
      const int h = (int)(e / rowlen), w = (int)((e - (long long)h * rowlen) / C);
      if (h >= r.y0 && h < r.y1 && w >= r.x0 && w < r.x1) { const float t = a[k]; a[k] = b[k]; b[k] = t; any = true; }
    }
  }
  if (!any) return;
  if constexpr (kVec) { VecIO<T>::st(xi, a); if (j != i) VecIO<T>::st(xj, b); }
  else { *xi = from_f<T>(a[0]); if (j != i) *xj = from_f<T>(b[0]); }
}

void mix_batch(void* x, const void* rec, int B, int H, int W, int C, int f32, cudaStream_t st) {
  const int pairs = (B + 1) / 2;
  if (B < 1 || H < 1 || W < 1 || C < 1 || pairs > 65535) throw std::runtime_error("mix_batch: needs 1 <= B <= 131070 and a non-empty image");
  const long long n = (long long)H * W * C;
  const int esz = f32 ? 4 : 2;
  const bool vec = (n * esz) % 16 == 0 && ((uintptr_t)x & 15) == 0;
  const long long units = vec ? n * esz / 16 : n;
  const dim3 grid((unsigned)grid_for(units, 256), (unsigned)pairs);
  auto R = (const MixRecord*)rec;
  if (f32) {
    if (vec) mix_batch_kernel<float, true><<<grid, 256, 0, st>>>((float*)x, R, B, H, W, C);
    else mix_batch_kernel<float, false><<<grid, 256, 0, st>>>((float*)x, R, B, H, W, C);
  } else {
    if (vec) mix_batch_kernel<__nv_bfloat16, true><<<grid, 256, 0, st>>>((__nv_bfloat16*)x, R, B, H, W, C);
    else mix_batch_kernel<__nv_bfloat16, false><<<grid, 256, 0, st>>>((__nv_bfloat16*)x, R, B, H, W, C);
  }
  count_launch(); TMPI_CHECK_LAUNCH("mix_batch"); ::tmpi::check_capture(st, "mix_batch");
}

// softmax_xent_kernel against the mixed soft target q = on·(λ·onehot(y_i) + (1 − λ)·onehot(y_j)) + off (on = 1 − ε, off = ε / C;
// ε = 0 gives off = 0 exactly), with λ = 1 when the record's mode is MIX_NONE:
//   rowstat[3b] = log se − on·(λ·(z_i − max) + (1 − λ)·(z_j − max)) − off·Σ(z − max),   dlogits = (softmax − q) * scale,
// and err1 / err5 rank the logit of the larger-weight label (y_i when λ ≥ ½, else y_j).
template <typename T>
__global__ void softmax_xent_mix_kernel(const T* __restrict__ logits, const long long* __restrict__ labels,
                                        const MixRecord* __restrict__ rec, T* __restrict__ dlogits, float* __restrict__ rowstat, int C,
                                        float scale, float on, float off) {
  const int b = blockIdx.x;
  const T* row = logits + (long long)b * C;
  const int yi = (int)labels[b], yj = (int)labels[gridDim.x - 1 - b];
  const float lam = rec->mode != MIX_NONE ? rec->lam : 1.f, oml = 1.f - lam;
  const int label = lam >= 0.5f ? yi : yj;                      // the errors' label
  __shared__ float red[32];
  __shared__ float bcast;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, to_f(row[c]));
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : -INFINITY; v = warp_max(v); if (lane == 0) bcast = v; }
  __syncthreads();
  mx = bcast;
  __syncthreads();
  const float lab = to_f(row[label]);
  float se = 0.f, gt = 0.f, sz = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = to_f(row[c]);
    se += __expf(v - mx);
    gt += (v > lab || (v == lab && c < label)) ? 1.f : 0.f;     // rank of the errors' label's logit
    sz += v - mx;
  }
  se = warp_sum(se); gt = warp_sum(gt); sz = warp_sum(sz);
  if (lane == 0) red[warp] = se;
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; v = warp_sum(v); if (lane == 0) bcast = v; }
  __syncthreads();
  se = bcast;
  __syncthreads();
  if (lane == 0) red[warp] = gt;
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; v = warp_sum(v); if (lane == 0) bcast = v; }
  __syncthreads();
  gt = bcast;
  __syncthreads();
  if (lane == 0) red[warp] = sz;                                // Σ(z − max) to thread 0
  __syncthreads();
  if (warp == 0) { float v = lane < nw ? red[lane] : 0.f; sz = warp_sum(v); }
  const float inv = 1.f / se;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float pr = __expf(to_f(row[c]) - mx) * inv - off;
    if (c == yi) pr -= on * lam;
    if (c == yj) pr -= on * oml;
    dlogits[(long long)b * C + c] = from_f<T>(pr * scale);
  }
  if (threadIdx.x == 0) {
    rowstat[3 * b + 0] = __logf(se) - on * (lam * (to_f(row[yi]) - mx) + oml * (to_f(row[yj]) - mx)) - off * sz;
    rowstat[3 * b + 1] = gt >= 1.f ? 1.f : 0.f;
    rowstat[3 * b + 2] = gt >= 5.f ? 1.f : 0.f;
  }
}

void softmax_xent_mix(const void* logits, const void* labels, const void* rec, void* dlogits, void* rowstat, void* out3, int B, int C,
                      float weight, float grad_weight, float label_smoothing, int f32, cudaStream_t st) {
  if (!(label_smoothing >= 0.f && label_smoothing <= 1.f)) throw std::runtime_error("softmax_xent_mix: label_smoothing must be in [0, 1]");
  if (!rec) throw std::runtime_error("softmax_xent_mix: needs the step's mix record");
  auto LB = (const long long*)labels; auto RS = (float*)rowstat; auto R = (const MixRecord*)rec;
  const float scale = grad_weight / (float)B;
  const float on = 1.f - label_smoothing, off = label_smoothing / (float)C;
  if (f32) softmax_xent_mix_kernel<float><<<B, 256, 0, st>>>((const float*)logits, LB, R, (float*)dlogits, RS, C, scale, on, off);
  else softmax_xent_mix_kernel<__nv_bfloat16><<<B, 256, 0, st>>>((const __nv_bfloat16*)logits, LB, R, (__nv_bfloat16*)dlogits, RS, C,
                                                                   scale, on, off);
  count_launch(); TMPI_CHECK_LAUNCH("softmax_xent_mix"); ::tmpi::check_capture(st, "softmax_xent_mix");
  rowstat_mean_kernel<<<1, 256, 0, st>>>((const float*)rowstat, (float*)out3, B, weight);
  count_launch(); TMPI_CHECK_LAUNCH("rowstat_mean"); ::tmpi::check_capture(st, "rowstat_mean");
}

// Knowledge distillation: the student's logits z against the hard target q (one-hot, smoothed, or the mixed target of rec when kMix)
// and the teacher's logits t of the same batch at temperature T.  One CTA per row, three passes over it as softmax_xent_kernel:
//   1. m = max z, m_t = max t (max z/T = m/T since T > 0);
//   2. se = Σ e^(z−m), sT = Σ e^((z−m)/T), st = Σ e_t with e_t = e^((t−m_t)/T), sd = Σ e_t·((t−m_t) − (z−m)), sz = Σ (z−m), the rank;
//   3. dlogits = scale·[(1 − α)·(p − q) + α·T·(softmax(z/T) − softmax(t/T))].
// KL(softmax(t/T) ‖ softmax(z/T)) = sd / (T·st) − log st + log sT in closed form, so
//   rowstat[3b] = (1 − α)·(log se − on·(λ·(z_i − m) + (1 − λ)·(z_j − m)) − off·sz) + α·T²·KL,
// and err1 / err5 rank the student's logit of the label with the larger weight (y_i when λ ≥ ½, else y_j).
template <typename T, bool kMix>
__global__ void __launch_bounds__(256) softmax_xent_kd_kernel(const T* __restrict__ logits, const T* __restrict__ teacher,
                                                              const long long* __restrict__ labels, const MixRecord* __restrict__ rec,
                                                              T* __restrict__ dlogits, float* __restrict__ rowstat, int C, float scale,
                                                              float on, float off, float alpha, float temp) {
  const int b = blockIdx.x;
  const T* row = logits + (long long)b * C;
  const T* trow = teacher + (long long)b * C;
  const int yi = (int)labels[b];
  const int yj = kMix ? (int)labels[gridDim.x - 1 - b] : yi;
  const float lam = (kMix && rec->mode != MIX_NONE) ? rec->lam : 1.f, oml = 1.f - lam;
  const int label = lam >= 0.5f ? yi : yj;                      // the errors' label
  __shared__ float red[6][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float mx = -INFINITY, mt = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { mx = fmaxf(mx, to_f(row[c])); mt = fmaxf(mt, to_f(trow[c])); }
  mx = warp_max(mx); mt = warp_max(mt);
  if (lane == 0) { red[0][warp] = mx; red[1][warp] = mt; }
  __syncthreads();
  mx = red[0][0]; mt = red[1][0];
  for (int w = 1; w < nw; ++w) { mx = fmaxf(mx, red[0][w]); mt = fmaxf(mt, red[1][w]); }
  __syncthreads();
  const float invT = 1.f / temp;
  const float lab = to_f(row[label]);
  float se = 0.f, sT = 0.f, st = 0.f, sd = 0.f, sz = 0.f, gt = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float zc = to_f(row[c]), v = zc - mx, u = to_f(trow[c]) - mt;
    const float et = __expf(u * invT);
    se += __expf(v);
    sT += __expf(v * invT);
    st += et;
    sd += et * (u - v);
    sz += v;
    gt += (zc > lab || (zc == lab && c < label)) ? 1.f : 0.f;     // rank of the errors' label's logit
  }
  se = warp_sum(se); sT = warp_sum(sT); st = warp_sum(st); sd = warp_sum(sd); sz = warp_sum(sz); gt = warp_sum(gt);
  if (lane == 0) { red[0][warp] = se; red[1][warp] = sT; red[2][warp] = st; red[3][warp] = sd; red[4][warp] = sz; red[5][warp] = gt; }
  __syncthreads();
  se = red[0][0]; sT = red[1][0]; st = red[2][0]; sd = red[3][0]; sz = red[4][0]; gt = red[5][0];
  for (int w = 1; w < nw; ++w) { se += red[0][w]; sT += red[1][w]; st += red[2][w]; sd += red[3][w]; sz += red[4][w]; gt += red[5][w]; }
  const float hw = 1.f - alpha, sw = alpha * temp;              // weights of (p − q) and of (softmax(z/T) − softmax(t/T))
  const float inv = 1.f / se, invsT = 1.f / sT, invst = 1.f / st;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = to_f(row[c]) - mx;
    float pq = __expf(v) * inv - off;
    if (c == yi) pq -= on * lam;
    if (kMix && c == yj) pq -= on * oml;
    const float kd = __expf(v * invT) * invsT - __expf((to_f(trow[c]) - mt) * invT) * invst;
    dlogits[(long long)b * C + c] = from_f<T>((hw * pq + sw * kd) * scale);
  }
  if (threadIdx.x == 0) {
    const float hard = __logf(se) - on * (lam * (to_f(row[yi]) - mx) + oml * (to_f(row[yj]) - mx)) - off * sz;
    const float kl = sd * invT * invst - __logf(st) + __logf(sT);
    rowstat[3 * b + 0] = hw * hard + sw * temp * kl;
    rowstat[3 * b + 1] = gt >= 1.f ? 1.f : 0.f;
    rowstat[3 * b + 2] = gt >= 5.f ? 1.f : 0.f;
  }
}

void softmax_xent_kd(const void* logits, const void* teacher, const void* labels, const void* rec, void* dlogits, void* rowstat, void* out3,
                     int B, int C, float grad_weight, float label_smoothing, float alpha, float temperature, int f32, cudaStream_t st) {
  if (!(label_smoothing >= 0.f && label_smoothing <= 1.f)) throw std::runtime_error("softmax_xent_kd: label_smoothing must be in [0, 1]");
  if (!(alpha > 0.f && alpha <= 1.f)) throw std::runtime_error("softmax_xent_kd: alpha must be in (0, 1]");
  if (!(temperature > 0.f && temperature <= 3.4e38f)) throw std::runtime_error("softmax_xent_kd: temperature must be finite and > 0");
  auto LB = (const long long*)labels; auto RS = (float*)rowstat; auto R = (const MixRecord*)rec;
  const float scale = grad_weight / (float)B;
  const float on = 1.f - label_smoothing, off = label_smoothing / (float)C;
  if (f32) {
    auto k = rec ? softmax_xent_kd_kernel<float, true> : softmax_xent_kd_kernel<float, false>;
    k<<<B, 256, 0, st>>>((const float*)logits, (const float*)teacher, LB, R, (float*)dlogits, RS, C, scale, on, off, alpha, temperature);
  } else {
    auto k = rec ? softmax_xent_kd_kernel<__nv_bfloat16, true> : softmax_xent_kd_kernel<__nv_bfloat16, false>;
    k<<<B, 256, 0, st>>>((const __nv_bfloat16*)logits, (const __nv_bfloat16*)teacher, LB, R, (__nv_bfloat16*)dlogits, RS, C, scale, on,
                         off, alpha, temperature);
  }
  count_launch(); TMPI_CHECK_LAUNCH("softmax_xent_kd"); ::tmpi::check_capture(st, "softmax_xent_kd");
  rowstat_mean_kernel<<<1, 256, 0, st>>>((const float*)rowstat, (float*)out3, B, 1.f);
  count_launch(); TMPI_CHECK_LAUNCH("rowstat_mean"); ::tmpi::check_capture(st, "rowstat_mean");
}

// ============================================================================ activation mask + bias gradient
// dym = act'(y) * dy (contiguous [R, C]; ReLU: dy * (y > 0));  db[c] += sum_r dym[r, c]   (db pre-zeroed by the launcher, unless it
// accumulates a gradient over several micro-batches)
// dy / y have row pitch ld (elements) so channel slices of a wider tensor work (grouped conv).
template <typename T, int ACT, bool WRITE>
__global__ void relu_bias_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ y,
                                     T* __restrict__ dym, float* __restrict__ db, float* __restrict__ db1, int c_split,
                                     long long R, int C, long long ld, int VT, int rows_per_cta, float slope) {
  constexpr bool RELU = ACT != ACT_NONE;              // y is read
  using V = VecIO<T>;
  constexpr int N = V::N;
  extern __shared__ float sm[];                       // [RL][VT*N]
  const int nvec = C >> V::LOG2N;
  const int RL = blockDim.x / VT;
  const int tv = threadIdx.x % VT, tr = threadIdx.x / VT;
  const int cv = blockIdx.y * VT + tv;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  if (tr < RL && cv < nvec) {
    const long long rend = min(R, r0 + rows_per_cta);
    for (long long r = r0 + tr; r < rend; r += 4 * RL) {
      // 4 rows per trip, all loads issued before any use (memory-level parallelism: this kernel is pure streaming)
      typename V::Raw dv[4], yv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < rend) {
          dv[u] = *reinterpret_cast<const typename V::Raw*>(dy + rr * ld + cv * N);
          if (RELU) yv[u] = *reinterpret_cast<const typename V::Raw*>(y + rr * ld + cv * N);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long rr = r + (long long)u * RL;
        if (rr < rend) {
          float d[N];
          V::unpack(dv[u], d);
          if (RELU) {
            float v[N];
            V::unpack(yv[u], v);
#pragma unroll
            for (int i = 0; i < N; ++i) {
              if (ACT == ACT_RELU) { if (!(v[i] > 0.f)) d[i] = 0.f; }
              else d[i] = act_bwd<ACT>(d[i], v[i], slope);
            }
          }
          if (WRITE) *reinterpret_cast<typename V::Raw*>(dym + rr * C + cv * N) = V::pack(d);
#pragma unroll
          for (int i = 0; i < N; ++i) acc[i] += d[i];
        }
      }
    }
  }
  if (db == nullptr) return;
  if (tr < RL) {
#pragma unroll
    for (int i = 0; i < N; ++i) sm[(tr * VT + tv) * N + i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < VT * N) {
    const int v = threadIdx.x / N, i = threadIdx.x % N;
    const int c = (blockIdx.y * VT + v) * N + i;
    if (c < C) {
      float s = 0.f;
      for (int t = 0; t < RL; ++t) s += sm[(t * VT + v) * N + i];
      atomicAdd(c < c_split ? db + c : db1 + (c - c_split), s);
    }
  }
}

// db: bias gradient for channels [0, c_split), db1: for channels [c_split, C) (the two parameter sets of a 2-group block);
// pass db1 = nullptr / c_split = C for a single bias vector.
template <typename T>
static void relu_bias_bwd_t(const void* dy, const void* y, void* dym, void* db, void* db1, int c_split, long long R, int C, long long ld,
                            int act, float slope, int accumulate, cudaStream_t st) {
  constexpr int N = VecIO<T>::N;
  const int nvec = C / N;
  const int VT = nvec < 32 ? nvec : 32;
  const int RL = 256 / VT;
  // deterministic mode: one CTA per channel group sums ALL rows (fixed order) instead of row slabs + atomics
  const long long rows_per_cta_ll = deterministic_mode() ? std::max<long long>(R, 1) : (long long)RL * 8;
  if (rows_per_cta_ll >= (1LL << 31)) throw std::runtime_error("relu_bias_bwd: too many rows for the deterministic mode");
  const int rows_per_cta = (int)rows_per_cta_ll;
  dim3 grid((unsigned)((R + rows_per_cta - 1) / rows_per_cta), (unsigned)((nvec + VT - 1) / VT));
  const size_t smem = (size_t)RL * VT * N * sizeof(float);
  if (!db1 || c_split > C) c_split = C;
  if (db && !accumulate) check_cuda(cudaMemsetAsync(db, 0, (size_t)c_split * 4, st), "relu_bias_bwd memset");
  if (db && !accumulate && c_split < C) check_cuda(cudaMemsetAsync(db1, 0, (size_t)(C - c_split) * 4, st), "relu_bias_bwd memset");
  const bool write = dym != nullptr;
  auto DY = (const T*)dy; auto Y = (const T*)y; auto DM = (T*)dym; auto DB = (float*)db; auto DB1 = (float*)db1;
#define RBB(A, WR) relu_bias_bwd_kernel<T, A, WR><<<grid, 256, smem, st>>>(DY, Y, DM, DB, DB1, c_split, R, C, ld, VT, rows_per_cta, slope)
  if ((act == ACT_LEAKY || act == ACT_SIGMOID) && !write) throw std::runtime_error("relu_bias_bwd: this activation mask needs the dym output");
  if (act == ACT_RELU && write) RBB(ACT_RELU, true);
  else if (act == ACT_RELU) RBB(ACT_RELU, false);
  else if (act == ACT_LEAKY) RBB(ACT_LEAKY, true);
  else if (act == ACT_SIGMOID) RBB(ACT_SIGMOID, true);
  else if (act != ACT_NONE) throw std::runtime_error("relu_bias_bwd: unknown activation");
  else if (write) RBB(ACT_NONE, true);
  else RBB(ACT_NONE, false);
#undef RBB
  count_launch(); TMPI_CHECK_LAUNCH("relu_bias_bwd"); ::tmpi::check_capture(st, "relu_bias_bwd");
}
void relu_bias_bwd(const void* dy, const void* y, void* dym, void* db, void* db1, int c_split, long long R, int C, long long ld, int act,
                   float slope, int accumulate, int f32, cudaStream_t st) {
  need_vec(C, f32, "relu_bias_bwd");
  if (f32) relu_bias_bwd_t<float>(dy, y, dym, db, db1, c_split, R, C, ld, act, slope, accumulate, st);
  else relu_bias_bwd_t<__nv_bfloat16>(dy, y, dym, db, db1, c_split, R, C, ld, act, slope, accumulate, st);
}

// y[r, c] = act(acc[r, c] (fp32) + bias[c]), stored as T — finishing pass of a split-K forward GEMM (small-batch FC layers: the
// parallelism has to come from splitting K, and split-K accumulates in fp32 with reductions, so bias / ReLU / cast run here).
// The fp32 output may alias acc (in place).  ACT_FLAG: ReLU when `relu` is set; ACT_LEAKY / ACT_SIGMOID: compile-time variants.
template <typename T, int ACT>
__global__ void bias_act_kernel(const float* __restrict__ acc, const float* __restrict__ bias, T* __restrict__ y, int R, int C, int relu,
                                float slope) {
  constexpr int N = VecIO<T>::N;
  const int nvec = C >> VecIO<T>::LOG2N;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;            // host guarantees R * nvec < 2^32
  if (idx >= (unsigned)R * (unsigned)nvec) return;
  const unsigned r = idx / (unsigned)nvec; const int cv = (int)(idx - r * (unsigned)nvec);
  float v[N];
#pragma unroll
  for (int j = 0; j < N; j += 4) VecIO<float>::ld(acc + (size_t)r * C + cv * N + j, v + j);
  if (bias) {
#pragma unroll
    for (int j = 0; j < N; j += 4) {
      const float4 b = *reinterpret_cast<const float4*>(bias + cv * N + j);
      v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
    }
  }
  if (ACT == ACT_FLAG) {
    if (relu) {
#pragma unroll
      for (int i = 0; i < N; ++i) v[i] = fmaxf(v[i], 0.f);
    }
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = act_fwd<ACT>(v[i], slope);
  }
  VecIO<T>::st(y + (size_t)r * C + cv * N, v);
}
template <typename T>
static void bias_act_t(const float* acc, const float* bias, void* y, int R, int C, int act, float slope, long long total, cudaStream_t st) {
  const int g = grid_for(total, 256);
  if (act == ACT_NONE || act == ACT_RELU) bias_act_kernel<T, ACT_FLAG><<<g, 256, 0, st>>>(acc, bias, (T*)y, R, C, act, slope);
  else if (act == ACT_LEAKY) bias_act_kernel<T, ACT_LEAKY><<<g, 256, 0, st>>>(acc, bias, (T*)y, R, C, act, slope);
  else if (act == ACT_SIGMOID) bias_act_kernel<T, ACT_SIGMOID><<<g, 256, 0, st>>>(acc, bias, (T*)y, R, C, act, slope);
  else throw std::runtime_error("bias_act: unknown activation");
}
void bias_act(const void* acc, const void* bias, void* y, int R, int C, int act, float slope, int f32, cudaStream_t st) {
  need_vec(C, f32, "bias_act");
  const long long total = (long long)R * (f32 ? C / 4 : C / 8);
  if (total >= (1LL << 32)) throw std::runtime_error("bias_act: tensor too large for 32-bit indexing");
  auto A = (const float*)acc; auto B = (const float*)bias;
  if (f32) bias_act_t<float>(A, B, y, R, C, act, slope, total, st);
  else bias_act_t<__nv_bfloat16>(A, B, y, R, C, act, slope, total, st);
  count_launch(); TMPI_CHECK_LAUNCH("bias_act"); ::tmpi::check_capture(st, "bias_act");
}

// Fused backward of  conv(+bias+ReLU) -> max-pool : one pass over the conv output instead of three.
//   dym[n,h,w,c] = (sum over pooling windows whose argmax is (h,w) of dyp) * (y[n,h,w,c] > 0)     (bf16, contiguous)
//   db[c]       += sum_{n,h,w} dym                                                                 (pre-zeroed by the launcher)
// Channels < c_split accumulate into db0, the rest into db1 (the two parameter sets of a 2-group AlexNet block).
// Replaces maxpool_bwd (write dx) + relu_bias_bwd (read dx, read y, write dym): 2 reads + 2 writes of the big tensor -> 1 + 1.
// One CTA per input row (n, h): the candidate output rows are CTA-uniform, each thread owns one channel vector (so its bias
// partial sums stay in registers) and sweeps w.
template <int MAXW, bool FUSE>
__global__ void __launch_bounds__(256) maxpool_relu_bias_bwd_kernel(const __nv_bfloat16* __restrict__ dyp, const uint8_t* __restrict__ arg,
                                             const __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ dym,
                                             float* __restrict__ db0, float* __restrict__ db1, int c_split, PoolGeom g, int VT) {
  extern __shared__ float sm[];                       // [RL][VT*8]
  const int nvec = g.C >> 3;
  const int RL = blockDim.x / VT;
  const int tv = threadIdx.x % VT, tw = threadIdx.x / VT;
  const int cv = blockIdx.y * VT + tv;
  const int h = blockIdx.x % g.H, n = blockIdx.x / g.H;
  int ho_lo = (h + g.p - g.k + g.s) / g.s; if (h + g.p - g.k + 1 <= 0) ho_lo = 0;
  const int ho_hi = min(g.Ho - 1, (h + g.p) / g.s);
  const long long irow = ((long long)n * g.H + h) * g.W * g.C;
  const long long obase = (long long)n * g.Ho * g.Wo * g.C;
  float tot[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) tot[i] = 0.f;
  if (tw < RL && cv < nvec) {
    for (int w = tw; w < g.W; w += RL) {
      int wo_lo = (w + g.p - g.k + g.s) / g.s; if (w + g.p - g.k + 1 <= 0) wo_lo = 0;
      const int wo_hi = min(g.Wo - 1, (w + g.p) / g.s);
      // phase 1: all candidate windows (at most MAXW x MAXW = ceil(k/s)^2) and the activation in flight at once
      uint2 av[MAXW * MAXW];
      bf16x8 dv[MAXW * MAXW];
      uint32_t me[MAXW * MAXW];
      bool ok[MAXW * MAXW];
#pragma unroll
      for (int a = 0; a < MAXW; ++a) {
#pragma unroll
        for (int b = 0; b < MAXW; ++b) {
          const int ho = ho_lo + a, wo = wo_lo + b;
          const int t = a * MAXW + b;
          ok[t] = (ho <= ho_hi && wo <= wo_hi);
          me[t] = (uint32_t)((h + g.p - ho * g.s) * g.k + (w + g.p - wo * g.s));
          if (ok[t]) {
            const long long o = obase + (unsigned)((ho * g.Wo + wo) * g.C + cv * 8);
            av[t] = *reinterpret_cast<const uint2*>(arg + o);
            dv[t] = *reinterpret_cast<const bf16x8*>(dyp + o);
          }
        }
      }
      const long long xi = irow + (unsigned)(w * g.C + cv * 8);
      bf16x8 yv;
      if (FUSE) yv = *reinterpret_cast<const bf16x8*>(y + xi);
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
      for (int t = 0; t < MAXW * MAXW; ++t) {
        if (ok[t]) {
          // argmax match for 4 channels per instruction (__vcmpeq4 on the packed argmax bytes), byte mask widened to the
          // bf16 lanes with PRMT, gradient kept packed until the add
          const uint32_t me4 = me[t] * 0x01010101u;
          const uint32_t eq_lo = __vcmpeq4(av[t].x, me4), eq_hi = __vcmpeq4(av[t].y, me4);
          const uint32_t* dw = reinterpret_cast<const uint32_t*>(&dv[t]);
          const uint32_t w0 = dw[0] & __byte_perm(eq_lo, 0, 0x1100), w1 = dw[1] & __byte_perm(eq_lo, 0, 0x3322);
          const uint32_t w2 = dw[2] & __byte_perm(eq_hi, 0, 0x1100), w3 = dw[3] & __byte_perm(eq_hi, 0, 0x3322);
          acc[0] += __uint_as_float(w0 << 16); acc[1] += __uint_as_float(w0 & 0xFFFF0000u);
          acc[2] += __uint_as_float(w1 << 16); acc[3] += __uint_as_float(w1 & 0xFFFF0000u);
          acc[4] += __uint_as_float(w2 << 16); acc[5] += __uint_as_float(w2 & 0xFFFF0000u);
          acc[6] += __uint_as_float(w3 << 16); acc[7] += __uint_as_float(w3 & 0xFFFF0000u);
        }
      }
      bf16x8 pk = pack8(acc);
      if (FUSE) {
        // ReLU mask on the packed result: a bf16 is > 0 exactly when its bits, read as int16, are > 0
        uint32_t* pw = reinterpret_cast<uint32_t*>(&pk);
        const uint32_t* yw = reinterpret_cast<const uint32_t*>(&yv);
#pragma unroll
        for (int i = 0; i < 4; ++i) pw[i] &= __vcmpgts2(yw[i], 0u);
      }
      *reinterpret_cast<bf16x8*>(dym + xi) = pk;
      if (FUSE) {
        unpack8(pk, acc);                               // db sums what wgrad / dgrad will actually see (bf16-rounded)
#pragma unroll
        for (int i = 0; i < 8; ++i) tot[i] += acc[i];
      }
    }
  }
  if (!FUSE) return;                                    // plain max-pool backward: no mask, no bias gradient
  if (tw < RL) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sm[(tw * VT + tv) * 8 + i] = tot[i];
  }
  __syncthreads();
  if (threadIdx.x < VT * 8) {
    const int v = threadIdx.x / 8, i = threadIdx.x % 8;
    const int c = (blockIdx.y * VT + v) * 8 + i;
    if (c < g.C) {
      float sacc = 0.f;
      for (int t = 0; t < RL; ++t) sacc += sm[(t * VT + v) * 8 + i];
      atomicAdd(c < c_split ? db0 + c : db1 + (c - c_split), sacc);
    }
  }
}

void maxpool_relu_bias_bwd(const void* dyp, const void* arg, const void* y, void* dym, void* db0, void* db1, int c_split, int N, int H,
                           int W, int C, int Ho, int Wo, int k, int s, int p, int accumulate, cudaStream_t st) {
  if (C % 8) throw std::runtime_error("maxpool_relu_bias_bwd: C must be a multiple of 8");
  if ((long long)H * W * C >= (1LL << 31)) throw std::runtime_error("maxpool_relu_bias_bwd: image too large for 32-bit in-image offsets");
  PoolGeom g{N, H, W, C, Ho, Wo, k, s, p};
  const int nvec = C / 8;
  const int VT = nvec < 32 ? nvec : 32;
  const int RL = 256 / VT;
  dim3 grid((unsigned)N * H, (unsigned)((nvec + VT - 1) / VT));
  const size_t smem = (size_t)RL * VT * 8 * sizeof(float);
  if (c_split > C) c_split = C;
  if (!accumulate) check_cuda(cudaMemsetAsync(db0, 0, (size_t)c_split * 4, st), "maxpool_relu_bias_bwd memset");
  if (!accumulate && c_split < C) check_cuda(cudaMemsetAsync(db1, 0, (size_t)(C - c_split) * 4, st), "maxpool_relu_bias_bwd memset");
  const int maxw = (k + s - 1) / s;
  auto DYP = (const __nv_bfloat16*)dyp; auto A = (const uint8_t*)arg; auto Y = (const __nv_bfloat16*)y; auto DM = (__nv_bfloat16*)dym;
  if (maxw == 1) maxpool_relu_bias_bwd_kernel<1, true><<<grid, 256, smem, st>>>(DYP, A, Y, DM, (float*)db0, (float*)db1, c_split, g, VT);
  else if (maxw == 2) maxpool_relu_bias_bwd_kernel<2, true><<<grid, 256, smem, st>>>(DYP, A, Y, DM, (float*)db0, (float*)db1, c_split, g, VT);
  else if (maxw == 3) maxpool_relu_bias_bwd_kernel<3, true><<<grid, 256, smem, st>>>(DYP, A, Y, DM, (float*)db0, (float*)db1, c_split, g, VT);
  else throw std::runtime_error("maxpool_relu_bias_bwd: pooling windows overlapping more than 3x3 outputs are not supported");
  count_launch(); TMPI_CHECK_LAUNCH("maxpool_relu_bias_bwd"); ::tmpi::check_capture(st, "maxpool_relu_bias_bwd");
}

// ============================================================================ im2col / col2im (NHWC)
struct ConvGeom { int N, H, W, Ctot, c_off, Cg, KH, KW, Ho, Wo, s, p; long long ldcol; int K; };

// col[m, (kh*KW+kw)*Cg + c] = x[n, ho*s-p+kh, wo*s-p+kw, c_off+c]   (zero outside the image)
template <typename T>
__global__ void __launch_bounds__(256) im2col_vec_kernel(const T* __restrict__ x, T* __restrict__ col, ConvGeom g) {
  // one CTA per IM2COL_ROWS consecutive output pixels; (n, ho, wo) is decoded once per row, the threads sweep the
  // row's KH*KW*(Cg/N) 16-byte vectors with 32-bit index math only.
  constexpr int IM2COL_ROWS = 8;
  constexpr int N = VecIO<T>::N;
  const int cvn = g.Cg >> VecIO<T>::LOG2N;
  const int per_m = g.KH * g.KW * cvn;
  const long long M = (long long)g.N * g.Ho * g.Wo;
  const long long m_base = (long long)blockIdx.x * IM2COL_ROWS;
  for (int rr = 0; rr < IM2COL_ROWS; ++rr) {
    const long long m = m_base + rr;
    if (m >= M) return;
    const int wo = (int)(m % g.Wo); const long long t = m / g.Wo;
    const int ho = (int)(t % g.Ho); const int n = (int)(t / g.Ho);
    const int h0 = ho * g.s - g.p, w0 = wo * g.s - g.p;
    const T* xin = x + (long long)n * g.H * g.W * g.Ctot + g.c_off;
    T* dst = col + m * g.ldcol;
    for (int v = threadIdx.x; v < per_m; v += blockDim.x) {
      const int kk = v / cvn, cv = v - kk * cvn;
      const int kh = kk / g.KW, kw = kk - kh * g.KW;
      const int h = h0 + kh, w = w0 + kw;
      typename VecIO<T>::Raw val;
      if (h >= 0 && h < g.H && w >= 0 && w < g.W)
        val = *reinterpret_cast<const typename VecIO<T>::Raw*>(xin + ((long long)h * g.W + w) * g.Ctot + cv * N);
      else {
        const float zero[N] = {};
        val = VecIO<T>::pack(zero);
      }
      *reinterpret_cast<typename VecIO<T>::Raw*>(dst + kk * g.Cg + cv * N) = val;
    }
  }
}

// generic (any Cg): one thread per (m, kh*KW+kw); the extra index KH*KW zero-fills the K..ldcol padding
template <typename T>
__global__ void im2col_scalar_kernel(const T* __restrict__ x, T* __restrict__ col, ConvGeom g) {
  const int per_m = g.KH * g.KW + 1;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long M = (long long)g.N * g.Ho * g.Wo;
  if (idx >= M * per_m) return;
  const long long m = idx / per_m; const int kk = (int)(idx % per_m);
  T* dst = col + m * g.ldcol;
  if (kk == g.KH * g.KW) { for (int c = g.K; c < g.ldcol; ++c) dst[c] = from_f<T>(0.f); return; }
  const int kh = kk / g.KW, kw = kk % g.KW;
  const int wo = (int)(m % g.Wo); long long t = m / g.Wo;
  const int ho = (int)(t % g.Ho); const int n = (int)(t / g.Ho);
  const int h = ho * g.s - g.p + kh, w = wo * g.s - g.p + kw;
  const bool ok = (h >= 0 && h < g.H && w >= 0 && w < g.W);
  const T* src = x + (((long long)n * g.H + h) * g.W + w) * g.Ctot + g.c_off;
  dst += (long long)kk * g.Cg;
  for (int c = 0; c < g.Cg; ++c) dst[c] = ok ? src[c] : from_f<T>(0.f);
}

// small-C path (conv1: C = 3): one CTA per (image, output row).  The KH input rows the output row needs are staged in
// shared memory with coalesced loads; the CTA then emits its Wo consecutive col rows (one contiguous Wo*ldcol span)
// as 16-byte vectors — each col row is KH runs of KW*Cg contiguous input elements.
template <typename T>
__global__ void __launch_bounds__(256) im2col_rows_kernel(const T* __restrict__ x, T* __restrict__ col, ConvGeom g) {
  constexpr int N = VecIO<T>::N;
  extern __shared__ __align__(16) unsigned char im2col_smem[];
  T* rows = reinterpret_cast<T*>(im2col_smem);             // [KH][W*Cg]
  const int n = blockIdx.x / g.Ho, ho = blockIdx.x % g.Ho;
  const int rowlen = g.W * g.Cg;
  const bool dense = (g.Cg == g.Ctot);                     // all channels used: an input row is one contiguous span
  for (int kh = 0; kh < g.KH; ++kh) {
    const int h = ho * g.s - g.p + kh;
    T* dst = rows + kh * rowlen;
    if (h < 0 || h >= g.H) {
      for (int e = threadIdx.x; e < rowlen; e += blockDim.x) dst[e] = from_f<T>(0.f);
    } else if (dense) {
      const T* src = x + ((long long)n * g.H + h) * g.W * g.Ctot;
      for (int e = threadIdx.x; e < rowlen; e += blockDim.x) dst[e] = src[e];
    } else {
      const T* src = x + ((long long)n * g.H + h) * g.W * g.Ctot + g.c_off;
      for (int e = threadIdx.x; e < rowlen; e += blockDim.x) { const int w = e / g.Cg; dst[e] = src[(long long)w * g.Ctot + (e - w * g.Cg)]; }
    }
  }
  __syncthreads();
  const int run = g.KW * g.Cg;                             // contiguous elements per (kh)
  const int vec_per_row = (int)(g.ldcol >> VecIO<T>::LOG2N);
  T* out = col + ((long long)n * g.Ho + ho) * g.Wo * g.ldcol;
  for (int i = threadIdx.x; i < g.Wo * vec_per_row; i += blockDim.x) {
    const int wo = i / vec_per_row, e0 = (i - wo * vec_per_row) * N;
    const int xbase = (wo * g.s - g.p) * g.Cg;              // may be negative with padding
    int kh = e0 / run, r = e0 - kh * run;
    __align__(16) T v[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
      T t = from_f<T>(0.f);
      if (e0 + j < g.K) {
        const int xi = xbase + r;
        if (xi >= 0 && xi < rowlen) t = rows[kh * rowlen + xi];
      }
      v[j] = t;
      if (++r == run) { r = 0; ++kh; }
    }
    *reinterpret_cast<uint4*>(out + (long long)wo * g.ldcol + e0) = *reinterpret_cast<const uint4*>(v);
  }
}

// dx[n,h,w,c_off+c] = sum over (kh,kw) with (h+p-kh)%s==0, (w+p-kw)%s==0 of dcol[m(n,ho,wo), (kh*KW+kw)*Cg + c]
// BIAS / ACT: the transposed-convolution forward, y = act(col2im(x · W) + b) with a per-channel fp32 bias, applied before the
// single store; channels >= c_real (zero padding of a layer narrower than 16 bytes) are stored as 0.
// <T, ACT_NONE, false> is the plain gather of the convolution's input gradient.
template <typename T, int ACT, bool BIAS>
__global__ void col2im_vec_kernel(const T* __restrict__ dcol, T* __restrict__ dx, ConvGeom g, const float* __restrict__ bias, float slope,
                                  int c_real) {
  constexpr int N = VecIO<T>::N;
  const unsigned cvn = (unsigned)(g.Cg >> VecIO<T>::LOG2N);
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;           // host guarantees total < 2^32
  const unsigned total = (unsigned)g.N * g.H * g.W * cvn;
  if (idx >= total) return;
  const int cv = (int)(idx % cvn); unsigned t = idx / cvn;
  const int w = (int)(t % g.W); t /= g.W;
  const int h = (int)(t % g.H); const int n = (int)(t / g.H);
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.f;
  for (int kh = 0; kh < g.KH; ++kh) {
    const int th = h + g.p - kh;
    if (th < 0 || th % g.s) continue;
    const int ho = th / g.s;
    if (ho >= g.Ho) continue;
    for (int kw = 0; kw < g.KW; ++kw) {
      const int tw = w + g.p - kw;
      if (tw < 0 || tw % g.s) continue;
      const int wo = tw / g.s;
      if (wo >= g.Wo) continue;
      const long long m = ((long long)n * g.Ho + ho) * g.Wo + wo;
      float v[N];
      VecIO<T>::ld(dcol + m * g.ldcol + (long long)(kh * g.KW + kw) * g.Cg + cv * N, v);
#pragma unroll
      for (int i = 0; i < N; ++i) acc[i] += v[i];
    }
  }
  if (BIAS) {
#pragma unroll
    for (int i = 0; i < N; ++i) acc[i] += __ldg(bias + cv * N + i);
  }
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = act_fwd<ACT>(acc[i], slope);
  if (BIAS || ACT != ACT_NONE) {
#pragma unroll
    for (int i = 0; i < N; ++i) if (cv * N + i >= c_real) acc[i] = 0.f;
  }
  VecIO<T>::st(dx + (((long long)n * g.H + h) * g.W + w) * g.Ctot + g.c_off + cv * N, acc);
}

template <typename T>
static void im2col_t(const void* x, void* col, const ConvGeom& g, cudaStream_t st) {
  constexpr int N = VecIO<T>::N;
  const long long M = (long long)g.N * g.Ho * g.Wo;
  // the vector kernel writes the K columns only: it needs rows without padding
  if (g.Cg % N == 0 && g.c_off % N == 0 && g.Ctot % N == 0 && g.ldcol == g.K) {
    im2col_vec_kernel<T><<<grid_for(M, 8), 256, 0, st>>>((const T*)x, (T*)col, g);
  } else if (g.ldcol % N == 0 && (size_t)g.KH * g.W * g.Cg * sizeof(T) <= 48 * 1024) {
    im2col_rows_kernel<T><<<g.N * g.Ho, 256, (size_t)g.KH * g.W * g.Cg * sizeof(T), st>>>((const T*)x, (T*)col, g);
  } else {
    const long long total = M * (g.KH * g.KW + 1);
    im2col_scalar_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)col, g);
  }
}

void im2col(const void* x, void* col, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho, int Wo, int s, int p,
            long long ldcol, int f32, cudaStream_t st) {
  ConvGeom g{N, H, W, Ctot, c_off, Cg, KH, KW, Ho, Wo, s, p, ldcol, KH * KW * Cg};
  if (f32) im2col_t<float>(x, col, g, st);
  else im2col_t<__nv_bfloat16>(x, col, g, st);
  count_launch(); TMPI_CHECK_LAUNCH("im2col"); ::tmpi::check_capture(st, "im2col");
}

void col2im(const void* dcol, void* dx, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho, int Wo, int s, int p,
            long long ldcol, int f32, cudaStream_t st) {
  const int V = f32 ? 4 : 8;
  if (Cg % V || c_off % V || Ctot % V || ldcol % V)
    throw std::runtime_error(f32 ? "col2im: channel counts must be multiples of 4" : "col2im: channel counts must be multiples of 8");
  ConvGeom g{N, H, W, Ctot, c_off, Cg, KH, KW, Ho, Wo, s, p, ldcol, KH * KW * Cg};
  long long total = (long long)N * H * W * (Cg / V);
  if (total >= (1LL << 32)) throw std::runtime_error("col2im: tensor too large for 32-bit indexing");
  if (f32) col2im_vec_kernel<float, ACT_NONE, false><<<grid_for(total, 256), 256, 0, st>>>((const float*)dcol, (float*)dx, g, nullptr, 0.f, 0);
  else col2im_vec_kernel<__nv_bfloat16, ACT_NONE, false><<<grid_for(total, 256), 256, 0, st>>>((const __nv_bfloat16*)dcol, (__nv_bfloat16*)dx, g,
                                                                                               nullptr, 0.f, 0);
  count_launch(); TMPI_CHECK_LAUNCH("col2im"); ::tmpi::check_capture(st, "col2im");
}

template <typename T>
static void col2im_bias_act_t(const void* dcol, void* y, const ConvGeom& g, const float* bias, int act, float slope, int c_real,
                              long long total, cudaStream_t st) {
  const int gr = grid_for(total, 256);
  auto D = (const T*)dcol; auto Y = (T*)y;
#define C2I(A) (bias ? col2im_vec_kernel<T, A, true><<<gr, 256, 0, st>>>(D, Y, g, bias, slope, c_real) \
                     : col2im_vec_kernel<T, A, false><<<gr, 256, 0, st>>>(D, Y, g, bias, slope, c_real))
  if (act == ACT_NONE) C2I(ACT_NONE);
  else if (act == ACT_RELU) C2I(ACT_RELU);
  else if (act == ACT_LEAKY) C2I(ACT_LEAKY);
  else if (act == ACT_SIGMOID) C2I(ACT_SIGMOID);
  else throw std::runtime_error("col2im_bias_act: unknown activation");
#undef C2I
}
void col2im_bias_act(const void* dcol, void* y, const float* bias, int N, int H, int W, int C, int KH, int KW, int Hi, int Wi, int s, int p,
                     long long ldcol, int act, float slope, int c_real, int f32, cudaStream_t st) {
  const int V = f32 ? 4 : 8;
  if (C % V || ldcol % V) throw std::runtime_error(f32 ? "col2im_bias_act: channel counts must be multiples of 4"
                                                       : "col2im_bias_act: channel counts must be multiples of 8");
  ConvGeom g{N, H, W, C, 0, C, KH, KW, Hi, Wi, s, p, ldcol, KH * KW * C};
  const long long total = (long long)N * H * W * (C / V);
  if (total >= (1LL << 32)) throw std::runtime_error("col2im_bias_act: tensor too large for 32-bit indexing");
  if (act == ACT_NONE && !bias && c_real < C) throw std::runtime_error("col2im_bias_act: padded channels need a bias or an activation");
  if (f32) col2im_bias_act_t<float>(dcol, y, g, bias, act, slope, c_real, total, st);
  else col2im_bias_act_t<__nv_bfloat16>(dcol, y, g, bias, act, slope, c_real, total, st);
  count_launch(); TMPI_CHECK_LAUNCH("col2im_bias_act"); ::tmpi::check_capture(st, "col2im_bias_act");
}

// ============================================================================ small utility kernels
// rows x cols (pitch src_ld) → rows x dst_ld with zero padding (K-padding of conv1 weights for TMA pitch rules)
template <typename T>
__global__ void pad_rows_kernel(const T* __restrict__ src, T* __restrict__ dst, long long rows, int cols, long long src_ld, long long dst_ld) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * dst_ld) return;
  const long long r = idx / dst_ld; const int c = (int)(idx % dst_ld);
  dst[idx] = c < cols ? src[r * src_ld + c] : from_f<T>(0.f);
}
void pad_rows(const void* src, void* dst, long long rows, int cols, long long src_ld, long long dst_ld, int f32, cudaStream_t st) {
  if (f32) pad_rows_kernel<float><<<grid_for(rows * dst_ld, 256), 256, 0, st>>>((const float*)src, (float*)dst, rows, cols, src_ld, dst_ld);
  else pad_rows_kernel<__nv_bfloat16><<<grid_for(rows * dst_ld, 256), 256, 0, st>>>((const __nv_bfloat16*)src, (__nv_bfloat16*)dst, rows, cols,
                                                                                      src_ld, dst_ld);
  count_launch(); TMPI_CHECK_LAUNCH("pad_rows"); ::tmpi::check_capture(st, "pad_rows");
}

// ============================================================================ space-to-depth for strided few-channel convs
// A KHxKW / stride-S convolution on C (< 8) channels is the ceil(KH/S) x ceil(KW/S) / stride-1 convolution of the
// space-to-depth image x'[n, i, j, (dy*S+dx)*C + c] = x[n, S*i+dy, S*j+dx, c] with the re-indexed (zero padded) filter.
// That turns AlexNet's conv1 (11x11/4 on RGB, which TMA cannot gather: 6-byte pixels) into a 3x3 conv on 48 channels
// that runs on the implicit-GEMM wgmma path.
// One CTA per output row (n, i): for a fixed dy the S*C output channels of pixel j are S*C CONTIGUOUS input elements of image
// row S*i+dy starting at j*S*C — a strided copy of short runs; threads sweep the row's output elements (coalesced stores).
template <int SCT>
__global__ void __launch_bounds__(256) space_to_depth_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H,
                                                             int W, int C, int S, int Hs, int Ws, int Cp, int P) {
  // blockDim = (Cp, 256 / Cp): threadIdx.x = output channel cp, threadIdx.y strides over the pixels j of output row (n, i).
  // SCT > 0: S*C is a compile-time constant, so cp / SC and cp % SC are a multiply-shift (the generic version was
  // issue-bound on runtime divisions: 74 instructions per 2-byte element).
  // P = zero padding of the ORIGINAL convolution, folded in here: output (i, j, (dy, dx, c)) reads x[S*i + dy - P, S*j + dx - P, c].
  const int i = blockIdx.x % Hs, n = blockIdx.x / Hs;
  const int SC = SCT > 0 ? SCT : S * C;
  const int WC = W * C;
  const int cp = threadIdx.x;
  const int dy = cp / SC, e = cp - dy * SC;
  const int h = i * S + dy - P;
  const bool chan_ok = cp < S * SC && h >= 0 && h < H;
  __nv_bfloat16* orow = y + ((long long)n * Hs + i) * Ws * Cp + cp;
  const __nv_bfloat16* irow = x + ((long long)n * H + (chan_ok ? h : 0)) * WC;
  const __nv_bfloat16 zero = f_to_bf16(0.f);
  const int shift = e - P * C;
  for (int j = threadIdx.y; j < Ws; j += blockDim.y) {
    const int col = j * SC + shift;                      // element offset inside the image row
    orow[(unsigned)(j * Cp)] = (chan_ok && col >= 0 && col < WC) ? irow[col] : zero;
  }
}
// fp32: one thread per output element (the row kernel above is limited to 256 packed channels)
__global__ void space_to_depth_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int H, int W, int C, int S, int Hs, int Ws,
                                          int Cp, int P) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * Hs * Ws * Cp;
  if (idx >= total) return;
  const int cp = (int)(idx % Cp); long long t = idx / Cp;
  const int j = (int)(t % Ws); t /= Ws;
  const int i = (int)(t % Hs); const int n = (int)(t / Hs);
  float v = 0.f;
  if (cp < S * S * C) {
    const int c = cp % C, d = cp / C, dy = d / S, dx = d % S;
    const int h = i * S + dy - P, w = j * S + dx - P;
    if (h >= 0 && h < H && w >= 0 && w < W) v = x[(((long long)n * H + h) * W + w) * C + c];
  }
  y[idx] = v;
}

void space_to_depth(const void* x, void* y, int N, int H, int W, int C, int S, int Hs, int Ws, int Cp, int P, int f32, cudaStream_t st) {
  if (f32) {
    space_to_depth_f32_kernel<<<grid_for((long long)N * Hs * Ws * Cp, 256), 256, 0, st>>>((const float*)x, (float*)y, N, H, W, C, S, Hs, Ws, Cp, P);
    count_launch(); TMPI_CHECK_LAUNCH("space_to_depth"); ::tmpi::check_capture(st, "space_to_depth");
    return;
  }
  if (Cp > 256) throw std::runtime_error("space_to_depth: more than 256 packed channels");
  const dim3 blk((unsigned)Cp, (unsigned)std::max(1, 256 / Cp));
  auto X = (const __nv_bfloat16*)x; auto Y = (__nv_bfloat16*)y;
  if (S * C == 12) space_to_depth_kernel<12><<<(unsigned)N * Hs, blk, 0, st>>>(X, Y, N, H, W, C, S, Hs, Ws, Cp, P);
  else space_to_depth_kernel<0><<<(unsigned)N * Hs, blk, 0, st>>>(X, Y, N, H, W, C, S, Hs, Ws, Cp, P);
  count_launch(); TMPI_CHECK_LAUNCH("space_to_depth"); ::tmpi::check_capture(st, "space_to_depth");
}

// w [O][KH][KW][C]  <->  ws [O][KHs][KWs][Cp]   with  ws[o, a, b, (dy*S+dx)*C + c] = w[o, S*a+dy, S*b+dx, c]  (0 outside the filter)
// dir 0: pack the filter of storage type T (w -> ws);  dir 1: unpack the fp32 gradient (gs -> g);  dir 2: unpack and add (g += ...)
template <typename T>
__global__ void s2d_filter_kernel(const void* __restrict__ src, void* __restrict__ dst, int O, int KH, int KW, int C, int S, int KHs, int KWs,
                                  int Cp, int dir) {
  if (dir == 0) {
    const int total = O * KHs * KWs * Cp;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
      const int cp = i % Cp; int t = i / Cp;
      const int b = t % KWs; t /= KWs;
      const int a = t % KHs; const int o = t / KHs;
      T v = from_f<T>(0.f);
      if (cp < S * S * C) {
        const int c = cp % C, d = cp / C, dy = d / S, dx = d % S;
        const int kh = a * S + dy, kw = b * S + dx;
        if (kh < KH && kw < KW) v = reinterpret_cast<const T*>(src)[(((long long)o * KH + kh) * KW + kw) * C + c];
      }
      reinterpret_cast<T*>(dst)[i] = v;
    }
  } else {
    const int total = O * KH * KW * C;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
      const int c = i % C; int t = i / C;
      const int kw = t % KW; t /= KW;
      const int kh = t % KH; const int o = t / KH;
      const int a = kh / S, dy = kh % S, b = kw / S, dx = kw % S;
      const float v = reinterpret_cast<const float*>(src)[(((long long)o * KHs + a) * KWs + b) * Cp + (dy * S + dx) * C + c];
      if (dir == 2) reinterpret_cast<float*>(dst)[i] += v;
      else reinterpret_cast<float*>(dst)[i] = v;
    }
  }
}
void s2d_filter(const void* src, void* dst, int O, int KH, int KW, int C, int S, int KHs, int KWs, int Cp, int dir, int f32, cudaStream_t st) {
  const int total = dir == 0 ? O * KHs * KWs * Cp : O * KH * KW * C;
  const int grid = std::min(grid_for(total, 256), sm_count() * 8);
  if (f32) s2d_filter_kernel<float><<<grid, 256, 0, st>>>(src, dst, O, KH, KW, C, S, KHs, KWs, Cp, dir);
  else s2d_filter_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(src, dst, O, KH, KW, C, S, KHs, KWs, Cp, dir);
  count_launch(); TMPI_CHECK_LAUNCH("s2d_filter"); ::tmpi::check_capture(st, "s2d_filter");
}

// ============================================================================ loader: normalise + crop + mirror → NHWC bf16/fp32
// One output pixel: (src[c] − mean)·scale·cscale[c] for c < C, 0 for C ≤ c < Cout.  Shared by crop_mirror_norm_kernel and
// multi_crop_norm_kernel, so a view of the latter is bit-equal to the former run with the view's offsets.
template <typename Tin, typename Tout>
__device__ __forceinline__ void norm_pixel(const Tin* __restrict__ src, const float* __restrict__ mp, int mean_mode, float scale,
                                           const float* __restrict__ cscale, Tout* __restrict__ o, int C, int Cout) {
  if (C == 3 && Cout == 3) {
    const float m0 = mean_mode == 0 ? mp[0] : mp[0], m1 = mean_mode == 0 ? mp[0] : mp[1], m2 = mean_mode == 0 ? mp[0] : mp[2];
    // per-channel 1/std on top of the scalar scale (ref proc_load_mpi.py:99: (arr - img_mean) / 255. / img_std)
    const float s0 = cscale ? scale * cscale[0] : scale, s1 = cscale ? scale * cscale[1] : scale, s2 = cscale ? scale * cscale[2] : scale;
    const float v0 = ((float)src[0] - m0) * s0, v1 = ((float)src[1] - m1) * s1, v2 = ((float)src[2] - m2) * s2;
    o[0] = (Tout)v0; o[1] = (Tout)v1; o[2] = (Tout)v2;
    return;
  }
  for (int c = 0; c < Cout; ++c) {
    float v = 0.f;
    if (c < C) {
      const float m = mean_mode == 0 ? mp[0] : mp[c];
      v = ((float)src[c] - m) * (cscale ? scale * cscale[c] : scale);
    }
    o[c] = (Tout)v;
  }
}

// One CTA per output row (n, oy): crop offsets / flip flag are CTA-uniform, threads sweep the row's (ox, c) elements with 32-bit
// math (coalesced stores; loads are contiguous runs of the source row, reversed when mirrored).
// grid = (N * ch, ceil(cw / 128)): the output row (n, oy) comes from blockIdx.x, the pixel from blockIdx.y / threadIdx.x — no
// per-thread divisions (the one-thread-per-pixel version with 64-bit div/mod was issue-bound: 230 instructions per pixel).
// kZeroFill: the offsets may put (sy, sx) outside the image (the zero-padded random crop of cifar_augment); such a pixel is 0 in
// every output channel, i.e. the mean pixel of the normalised image.  Without it the offsets must keep the crop inside the image.
template <typename Tin, typename Tout, bool kZeroFill = false>
__global__ void __launch_bounds__(128) crop_mirror_norm_kernel(const Tin* __restrict__ x, const float* __restrict__ mean, int mean_mode,
                                        float scale, const float* __restrict__ cscale, Tout* __restrict__ out, const int* __restrict__ offs,
                                        const uint8_t* __restrict__ flips, int N, int H, int W, int C, int ch, int cw, int Cout) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int oy = blockIdx.x % ch, n = blockIdx.x / ch;
  const int sy = offs[2 * n] + oy;
  const int sx = offs[2 * n + 1] + (flips[n] ? (cw - 1 - ox) : ox);
  if constexpr (kZeroFill) {
    if ((unsigned)sy >= (unsigned)H || (unsigned)sx >= (unsigned)W) {
      Tout* z = out + ((long long)blockIdx.x * cw + ox) * Cout;
      for (int c = 0; c < Cout; ++c) z[c] = (Tout)0.f;
      return;
    }
  }
  const unsigned pix = (unsigned)(sy * W + sx) * (unsigned)C;          // inside one image (host checks H*W*C < 2^31)
  norm_pixel(x + (long long)n * H * W * C + pix, mean_mode == 2 ? mean + pix : mean, mean_mode, scale, cscale,
             out + ((long long)blockIdx.x * cw + ox) * Cout, C, Cout);
}

void crop_mirror_norm(const void* x, int in_kind /*0 u8, 1 bf16, 2 f32*/, const void* mean, int mean_mode, float scale, const void* cscale, void* out,
                      int out_bf16, const void* offs, const void* flips, int N, int H, int W, int C, int ch, int cw, int Cout, int zero_fill,
                      cudaStream_t st) {
  if ((long long)H * W * C >= (1LL << 31) || (long long)N * ch >= (1LL << 31)) throw std::runtime_error("crop_mirror_norm: image too large");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  auto M = (const float*)mean; auto O = (const int*)offs; auto F = (const uint8_t*)flips;
#define CMN(TI, TO) (zero_fill ? crop_mirror_norm_kernel<TI, TO, true> : crop_mirror_norm_kernel<TI, TO, false>)<<<g, 128, 0, st>>>( \
      (const TI*)x, M, mean_mode, scale, (const float*)cscale, (TO*)out, O, F, N, H, W, C, ch, cw, Cout)
  if (in_kind == 0) { if (out_bf16) CMN(uint8_t, __nv_bfloat16); else CMN(uint8_t, float); }
  else if (in_kind == 1) { if (out_bf16) CMN(__nv_bfloat16, __nv_bfloat16); else CMN(__nv_bfloat16, float); }
  else { if (out_bf16) CMN(float, __nv_bfloat16); else CMN(float, float); }
#undef CMN
  count_launch(); TMPI_CHECK_LAUNCH("crop_mirror_norm"); ::tmpi::check_capture(st, "crop_mirror_norm");
}

// ============================================================================ loader: every test-time view in one launch
// V fixed views (y0, x0, mirror) of the uint8 NHWC batch into the view-major output [V, N, ch, cw, C].  The table travels by value
// in the kernel's parameters, so there is no per-image offset array and no copy to the device; __grid_constant__ lets the CTA-uniform
// view index read it in place (a by-value array indexed at run time is otherwise copied to local memory by every thread, which made
// the kernel several times slower per view than crop_mirror_norm_kernel).  The grid of crop_mirror_norm_kernel with the view in
// blockIdx.z: output row (v·N + n)·ch + oy, no per-thread division by N; each pixel goes through norm_pixel.
template <typename Tout>
__global__ void __launch_bounds__(128) multi_crop_norm_kernel(const uint8_t* __restrict__ x, const float* __restrict__ mean, int mean_mode,
                                                              float scale, const float* __restrict__ cscale, Tout* __restrict__ out,
                                                              const __grid_constant__ ViewTable views, int N, int H, int W, int C,
                                                              int ch, int cw) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int oy = blockIdx.x % ch, n = blockIdx.x / ch, v = blockIdx.z;
  const int sy = views.y0[v] + oy;
  const int sx = views.x0[v] + (views.mirror[v] ? (cw - 1 - ox) : ox);
  const unsigned pix = (unsigned)(sy * W + sx) * (unsigned)C;
  norm_pixel(x + (long long)n * H * W * C + pix, mean_mode == 2 ? mean + pix : mean, mean_mode, scale, cscale,
             out + (((long long)v * N * ch + blockIdx.x) * cw + ox) * C, C, C);
}

void multi_crop_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                     const ViewTable& views, int V, int N, int H, int W, int C, int ch, int cw, cudaStream_t st) {
  if (V < 1 || V > kMaxViews) throw std::runtime_error("multi_crop_norm: 1 to 10 views");
  if ((long long)H * W * C >= (1LL << 31) || (long long)V * N * ch >= (1LL << 31)) throw std::runtime_error("multi_crop_norm: image too large");
  for (int v = 0; v < V; ++v)
    if (views.y0[v] < 0 || views.x0[v] < 0 || views.y0[v] + ch > H || views.x0[v] + cw > W)
      throw std::runtime_error("multi_crop_norm: a view is not inside the image");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128), (unsigned)V);
  auto X = (const uint8_t*)x; auto M = (const float*)mean; auto CS = (const float*)cscale;
  if (out_bf16) multi_crop_norm_kernel<__nv_bfloat16><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (__nv_bfloat16*)out, views, N, H, W, C, ch, cw);
  else multi_crop_norm_kernel<float><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (float*)out, views, N, H, W, C, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("multi_crop_norm"); ::tmpi::check_capture(st, "multi_crop_norm");
}

// ============================================================================ loader: random-resized crop → NHWC bf16/fp32
// Output pixel (oy, ox) of image n is the bilinear resample of the normalised box (y0, x0, h, w) = boxes[n] to ch × cw, as
// F.interpolate(mode='bilinear', align_corners=False, antialias=False), mirrored after the resize.  Each of the four taps is
// normalised with its own mean (the per-pixel mean makes normalise-then-resize the definition).  Per axis of box length L:
// s = max((o + ½)·L/out − ½, 0), i0 = ⌊s⌋, i1 = i0 + (i0 < L − 1), λ = s − i0, in fp32 as ATen's bilinear kernel computes it: an
// IEEE division L/out and one fused multiply-add (explicit _rn intrinsics, so --use_fast_math changes neither; the unfused form
// moves λ by an ulp of s, about 1.5e-5 at s ≈ 250).
// Same grid as crop_mirror_norm_kernel: one CTA per output row (n, oy), so the box, the flip, both source rows and the y weight are
// CTA-uniform; threads sweep ox with one multiply per coordinate, and adjacent ox gather the same or adjacent texels (L1 hits).
__device__ __forceinline__ void rrc_axis(int o, float ratio, int L, int& i0, int& i1, float& lam) {
  const float s = fmaxf(__fmaf_rn(ratio, (float)o + 0.5f, -0.5f), 0.f);
  i0 = min((int)s, L - 1);
  i1 = i0 + (i0 < L - 1 ? 1 : 0);
  lam = fminf(fmaxf(s - (float)i0, 0.f), 1.f);
}

// JITTER (colour jitter + lighting, C == 3): image n's 96-byte record rec[n] = (M, K, ℓ, 0) and its crop mean mu[n] (float4, null when
// K ≡ 0) map the bilinear resample v̂ of the raw box to M·v̂ + K·μ + ℓ, which is then normalised with the same resample m̂ of the mean:
// out = (M·v̂ + t − m̂)·s_c, t = K·μ + ℓ formed once per thread from CTA-uniform loads.  A box of the output's size (λ = 0) gives
// v̂ = x and m̂ = m exactly, so the identity record reproduces crop_mirror_norm_kernel bit for bit.
template <typename Tout, bool JITTER = false>
__global__ void __launch_bounds__(128) resized_crop_mirror_norm_kernel(const uint8_t* __restrict__ x, const float* __restrict__ mean,
                                        int mean_mode, float scale, const float* __restrict__ cscale, Tout* __restrict__ out,
                                        const int4* __restrict__ boxes, const uint8_t* __restrict__ flips, int H, int W, int C, int ch,
                                        int cw, const float4* __restrict__ rec = nullptr, const float4* __restrict__ mu = nullptr) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int oy = blockIdx.x % ch, n = blockIdx.x / ch;
  const int4 b = boxes[n];                                               // (y0, x0, h, w), inside the image (host-drawn)
  int iy0, iy1, ix0, ix1;
  float ly, lx;
  rrc_axis(oy, __fdiv_rn((float)b.z, (float)ch), b.z, iy0, iy1, ly);
  rrc_axis(flips[n] ? cw - 1 - ox : ox, __fdiv_rn((float)b.w, (float)cw), b.w, ix0, ix1, lx);
  // texel offsets inside one image (host checks H*W*C < 2^31)
  const unsigned r0 = (unsigned)((b.x + iy0) * W + b.y) * (unsigned)C, r1 = (unsigned)((b.x + iy1) * W + b.y) * (unsigned)C;
  const unsigned c0 = (unsigned)ix0 * (unsigned)C, c1 = (unsigned)ix1 * (unsigned)C;
  const unsigned t00 = r0 + c0, t01 = r0 + c1, t10 = r1 + c0, t11 = r1 + c1;
  const uint8_t* src = x + (long long)n * H * W * C;
  const float wy0 = 1.f - ly, wx0 = 1.f - lx;
  Tout* o = out + ((long long)blockIdx.x * cw + ox) * C;
  if constexpr (std::is_same_v<Tout, uint8_t>) {
    // raw mode (auto_augment's uint8 crop): u = round-half-to-even of the bilinear resample v̂ of the raw box, no normalisation
    for (int c = 0; c < C; ++c) {
      const float v = wy0 * (wx0 * (float)src[t00 + c] + lx * (float)src[t01 + c]) + ly * (wx0 * (float)src[t10 + c] + lx * (float)src[t11 + c]);
      o[c] = (uint8_t)__float2int_rn(v);
    }
    return;
  }
  if constexpr (JITTER) {
    const float4* r = rec + 6 * n;
    const float4 r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3], r4 = r[4], r5 = r[5];
    // floats 0-8 M row-major (m00 m01 m02 m10 | m11 m12 m20 m21 | m22), 9-17 K the same way (k00 at r2.y), 18-20 ℓ (r4.z, r4.w, r5.x)
    float t0 = r4.z, t1 = r4.w, t2 = r5.x;
    if (mu) {
      const float4 u = mu[n];
      t0 = __fmaf_rn(r2.y, u.x, __fmaf_rn(r2.z, u.y, __fmaf_rn(r2.w, u.z, t0)));
      t1 = __fmaf_rn(r3.x, u.x, __fmaf_rn(r3.y, u.y, __fmaf_rn(r3.z, u.z, t1)));
      t2 = __fmaf_rn(r3.w, u.x, __fmaf_rn(r4.x, u.y, __fmaf_rn(r4.y, u.z, t2)));
    }
    auto bilerp = [&](const uint8_t* p, int c) {
      return wy0 * (wx0 * (float)p[t00 + c] + lx * (float)p[t01 + c]) + ly * (wx0 * (float)p[t10 + c] + lx * (float)p[t11 + c]);
    };
    auto mhat = [&](int c) {
      if (mean_mode != 2) return mean_mode == 0 ? mean[0] : mean[c];
      return wy0 * (wx0 * mean[t00 + c] + lx * mean[t01 + c]) + ly * (wx0 * mean[t10 + c] + lx * mean[t11 + c]);
    };
    const float v0 = bilerp(src, 0), v1 = bilerp(src, 1), v2 = bilerp(src, 2);
    const float a0 = __fmaf_rn(r0.x, v0, __fmaf_rn(r0.y, v1, __fmaf_rn(r0.z, v2, t0)));
    const float a1 = __fmaf_rn(r0.w, v0, __fmaf_rn(r1.x, v1, __fmaf_rn(r1.y, v2, t1)));
    const float a2 = __fmaf_rn(r1.z, v0, __fmaf_rn(r1.w, v1, __fmaf_rn(r2.x, v2, t2)));
    const float s0 = cscale ? scale * cscale[0] : scale, s1 = cscale ? scale * cscale[1] : scale, s2 = cscale ? scale * cscale[2] : scale;
    o[0] = (Tout)((a0 - mhat(0)) * s0); o[1] = (Tout)((a1 - mhat(1)) * s1); o[2] = (Tout)((a2 - mhat(2)) * s2);
    return;
  }
  auto tap = [&](unsigned t, int c, float s) {
    const float m = mean_mode == 0 ? mean[0] : (mean_mode == 1 ? mean[c] : mean[t + c]);
    return ((float)src[t + c] - m) * s;
  };
  auto blend = [&](int c, float s) {
    return wy0 * (wx0 * tap(t00, c, s) + lx * tap(t01, c, s)) + ly * (wx0 * tap(t10, c, s) + lx * tap(t11, c, s));
  };
  if (C == 3) {
    const float s0 = cscale ? scale * cscale[0] : scale, s1 = cscale ? scale * cscale[1] : scale, s2 = cscale ? scale * cscale[2] : scale;
    const float v0 = blend(0, s0), v1 = blend(1, s1), v2 = blend(2, s2);
    o[0] = (Tout)v0; o[1] = (Tout)v1; o[2] = (Tout)v2;
    return;
  }
  for (int c = 0; c < C; ++c) o[c] = (Tout)blend(c, cscale ? scale * cscale[c] : scale);
}

void resized_crop_mirror_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                              const void* boxes, const void* flips, int N, int H, int W, int C, int ch, int cw, cudaStream_t st) {
  if ((long long)H * W * C >= (1LL << 31) || (long long)N * ch >= (1LL << 31)) throw std::runtime_error("resized_crop_mirror_norm: image too large");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  auto X = (const uint8_t*)x; auto M = (const float*)mean; auto CS = (const float*)cscale;
  auto B = (const int4*)boxes; auto F = (const uint8_t*)flips;
  if (out_bf16) resized_crop_mirror_norm_kernel<__nv_bfloat16><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (__nv_bfloat16*)out, B, F, H, W, C, ch, cw);
  else resized_crop_mirror_norm_kernel<float><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (float*)out, B, F, H, W, C, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("resized_crop_mirror_norm"); ::tmpi::check_capture(st, "resized_crop_mirror_norm");
}

void color_crop_mirror_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                            const void* boxes, const void* flips, const void* rec, const void* mu, int N, int H, int W, int ch, int cw,
                            cudaStream_t st) {
  if ((long long)H * W * 3 >= (1LL << 31) || (long long)N * ch >= (1LL << 31)) throw std::runtime_error("color_crop_mirror_norm: image too large");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  auto X = (const uint8_t*)x; auto M = (const float*)mean; auto CS = (const float*)cscale;
  auto B = (const int4*)boxes; auto F = (const uint8_t*)flips; auto R = (const float4*)rec; auto U = (const float4*)mu;
  if (out_bf16) resized_crop_mirror_norm_kernel<__nv_bfloat16, true><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (__nv_bfloat16*)out, B, F, H, W, 3, ch, cw, R, U);
  else resized_crop_mirror_norm_kernel<float, true><<<g, 128, 0, st>>>(X, M, mean_mode, scale, CS, (float*)out, B, F, H, W, 3, ch, cw, R, U);
  count_launch(); TMPI_CHECK_LAUNCH("color_crop_mirror_norm"); ::tmpi::check_capture(st, "color_crop_mirror_norm");
}

// ============================================================================ loader: mean RGB of each output crop (colour jitter's μ)
// mu[n] = (Σ v̂) / (ch·cw) over the ch × cw output pixels of box n, v̂ the bilinear value of the raw uint8 box from the same rrc_axis
// taps and the same arithmetic as the resize (the mirror does not change a sum).  One CTA per image, one warp per output row
// (rows warp, warp + 16, ...), lanes stride the row; per-thread sums in a fixed order, then a shuffle tree and a tree over the 16
// warps: no atomics, the same bits on every run.  A box of the output's size sums integers below 2^24 (256² · 255), exact in fp32.
constexpr int CROP_MEAN_THREADS = 512;

__global__ void __launch_bounds__(CROP_MEAN_THREADS) crop_mean_kernel(const uint8_t* __restrict__ x, const int4* __restrict__ boxes,
                                                                      float4* __restrict__ mu, int H, int W, int ch, int cw) {
  const int n = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int4 b = boxes[n];
  const uint8_t* src = x + (long long)n * H * W * 3;
  const float ry = __fdiv_rn((float)b.z, (float)ch), rx = __fdiv_rn((float)b.w, (float)cw);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (int oy = warp; oy < ch; oy += CROP_MEAN_THREADS / 32) {
    int iy0, iy1;
    float ly;
    rrc_axis(oy, ry, b.z, iy0, iy1, ly);
    const unsigned r0 = (unsigned)((b.x + iy0) * W + b.y) * 3u, r1 = (unsigned)((b.x + iy1) * W + b.y) * 3u;
    const float wy0 = 1.f - ly;
    for (int ox = lane; ox < cw; ox += 32) {
      int ix0, ix1;
      float lx;
      rrc_axis(ox, rx, b.w, ix0, ix1, lx);
      const unsigned t00 = r0 + 3u * ix0, t01 = r0 + 3u * ix1, t10 = r1 + 3u * ix0, t11 = r1 + 3u * ix1;
      const float wx0 = 1.f - lx;
      auto bilerp = [&](int c) {
        return wy0 * (wx0 * (float)src[t00 + c] + lx * (float)src[t01 + c]) + ly * (wx0 * (float)src[t10 + c] + lx * (float)src[t11 + c]);
      };
      s0 += bilerp(0); s1 += bilerp(1); s2 += bilerp(2);
    }
  }
  for (int d = 16; d > 0; d >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, d); s1 += __shfl_xor_sync(0xffffffffu, s1, d); s2 += __shfl_xor_sync(0xffffffffu, s2, d);
  }
  __shared__ float part[3][CROP_MEAN_THREADS / 32];
  if (lane == 0) { part[0][warp] = s0; part[1][warp] = s1; part[2][warp] = s2; }
  __syncthreads();
  if (warp == 0) {
    const bool live = lane < CROP_MEAN_THREADS / 32;
    s0 = live ? part[0][lane] : 0.f; s1 = live ? part[1][lane] : 0.f; s2 = live ? part[2][lane] : 0.f;
    for (int d = 8; d > 0; d >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, d); s1 += __shfl_xor_sync(0xffffffffu, s1, d); s2 += __shfl_xor_sync(0xffffffffu, s2, d);
    }
    if (lane == 0) {
      const float p = (float)(ch * cw);
      mu[n] = make_float4(__fdiv_rn(s0, p), __fdiv_rn(s1, p), __fdiv_rn(s2, p), 0.f);
    }
  }
}

void crop_mean(const void* x, const void* boxes, void* mu, int N, int H, int W, int ch, int cw, cudaStream_t st) {
  if ((long long)H * W * 3 >= (1LL << 31) || (long long)ch * cw >= (1LL << 24)) throw std::runtime_error("crop_mean: image too large");
  crop_mean_kernel<<<N, CROP_MEAN_THREADS, 0, st>>>((const uint8_t*)x, (const int4*)boxes, (float4*)mu, H, W, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("crop_mean"); ::tmpi::check_capture(st, "crop_mean");
}

// ============================================================================ loader: TrivialAugmentWide / RandAugment / AutoAugment / AugMix
// torchvision.transforms.v2's uint8 ops, one op slot at a time, on the [N, ch, cw, 3] uint8 crop u.  rec[n] = 12 floats per slot: op id,
// scalar (factor, Solarize threshold or Posterize bits), 1 − factor (blends), bilinear (0 / 1; the launch argument selects the path),
// the fp32 inverse affine matrix (6), 0, 0.  AA_NONE is an AugMix chain step past the chain's depth: nothing is written.
// aa_lut_kernel builds image n's per-channel 256-entry LUT for the point ops (Brightness, Contrast, Posterize, Solarize, AutoContrast,
// Equalize) from the ping buffer, with the image-wide statistics they need; aa_apply_kernel maps ping → pong; aa_normalize_kernel
// writes (u' − m̂)·s_c.  The fp32 expressions are torchvision's: a separate multiply and a fused add for the blends (ATen's vectorised
// a + α·b), truncating casts after a clamp to [0, 255], an fma chain and a floor for the grey level.
enum AaOp { AA_IDENTITY, AA_SHEARX, AA_SHEARY, AA_TRANSX, AA_TRANSY, AA_ROTATE, AA_BRIGHTNESS, AA_COLOR, AA_CONTRAST, AA_SHARPNESS,
            AA_POSTERIZE, AA_SOLARIZE, AA_AUTOCONTRAST, AA_EQUALIZE, AA_INVERT, AA_NONE };
constexpr int AA_REC = 12;
constexpr int AA_LUT_THREADS = 512;

__device__ __forceinline__ uint8_t aa_clamp_trunc(float v) { return (uint8_t)(int)fminf(fmaxf(v, 0.f), 255.f); }
__device__ __forceinline__ float aa_gray(float r, float g, float b) {
  return floorf(__fmaf_rn(b, 0.114f, __fmaf_rn(g, 0.587f, __fmul_rn(r, 0.2989f))));
}

// One CTA per image; images whose op in this slot is not a point op return at once.  Reductions in shared memory (integer sums,
// min / max, a shared-memory histogram): no global atomics, the same bits on every run.
__global__ void __launch_bounds__(AA_LUT_THREADS) aa_lut_kernel(const uint8_t* __restrict__ u, const float* __restrict__ rec,
                                                                 uint8_t* __restrict__ lut, int slot, int slots, int P) {
  const int n = blockIdx.x, tid = threadIdx.x;
  const float* r = rec + ((long long)n * slots + slot) * AA_REC;
  const int op = (int)r[0];
  if (!(op == AA_BRIGHTNESS || op == AA_CONTRAST || op == AA_POSTERIZE || op == AA_SOLARIZE || op == AA_AUTOCONTRAST || op == AA_EQUALIZE ||
        op == AA_INVERT)) return;
  const float f = r[1], d = r[2];
  const uint8_t* src = u + (long long)n * P * 3;
  uint8_t* L = lut + (long long)n * 768;
  __shared__ int hist[3][256];
  __shared__ int red[3][AA_LUT_THREADS / 32];
  __shared__ float mean_s;
  if (op == AA_CONTRAST) {
    int sum = 0;                                            // floored grey levels: an exact integer sum (< 2^24 for 256² images)
    for (int p = tid; p < P; p += AA_LUT_THREADS) sum += (int)aa_gray(src[3 * p], src[3 * p + 1], src[3 * p + 2]);
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((tid & 31) == 0) red[0][tid >> 5] = sum;
    __syncthreads();
    if (tid == 0) {
      long long t = 0;
      for (int w = 0; w < AA_LUT_THREADS / 32; ++w) t += red[0][w];
      mean_s = __fdiv_rn((float)t, (float)P);
    }
    __syncthreads();
    const float mterm = mean_s;
    for (int i = tid; i < 768; i += AA_LUT_THREADS) L[i] = aa_clamp_trunc(__fmaf_rn(mterm, d, __fmul_rn((float)(i & 255), f)));
  } else if (op == AA_AUTOCONTRAST) {
    int mn0 = 255, mn1 = 255, mn2 = 255, mx0 = 0, mx1 = 0, mx2 = 0;
    for (int p = tid; p < P; p += AA_LUT_THREADS) {
      const int a = src[3 * p], b = src[3 * p + 1], c = src[3 * p + 2];
      mn0 = min(mn0, a); mn1 = min(mn1, b); mn2 = min(mn2, c); mx0 = max(mx0, a); mx1 = max(mx1, b); mx2 = max(mx2, c);
    }
    for (int o = 16; o > 0; o >>= 1) {
      mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
      mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
      mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
    }
    if ((tid & 31) == 0) { red[0][tid >> 5] = mn0 | (mx0 << 16); red[1][tid >> 5] = mn1 | (mx1 << 16); red[2][tid >> 5] = mn2 | (mx2 << 16); }
    __syncthreads();
    for (int i = tid; i < 768; i += AA_LUT_THREADS) {
      const int c = i >> 8;
      int mn = 255, mx = 0;
      for (int w = 0; w < AA_LUT_THREADS / 32; ++w) { mn = min(mn, red[c][w] & 0xffff); mx = max(mx, red[c][w] >> 16); }
      float lo = (float)mn, inv = __fmul_rn((float)(mx - mn), 1.0f / 255.0f);
      if (mx == mn) { lo = 0.f; inv = 1.f; }
      L[i] = aa_clamp_trunc(__fdiv_rn(__fsub_rn((float)(i & 255), lo), inv));
    }
  } else if (op == AA_EQUALIZE) {
    for (int i = tid; i < 768; i += AA_LUT_THREADS) (&hist[0][0])[i] = 0;
    __syncthreads();
    for (int p = tid; p < P; p += AA_LUT_THREADS) {
      atomicAdd(&hist[0][src[3 * p]], 1); atomicAdd(&hist[1][src[3 * p + 1]], 1); atomicAdd(&hist[2][src[3 * p + 2]], 1);
    }
    __syncthreads();
    if (tid < 3) {                                          // PIL's LUT, as torchvision computes it (step == 0: the identity)
      const int c = tid;
      int last = 255;
      while (last > 0 && hist[c][last] == 0) --last;
      const int step = (P - hist[c][last]) / 255;
      uint8_t* Lc = L + c * 256;
      if (step == 0) {
        for (int k = 0; k < 256; ++k) Lc[k] = (uint8_t)k;
      } else {
        int cum = 0;
        Lc[0] = 0;
        for (int k = 1; k < 256; ++k) { cum += hist[c][k - 1]; Lc[k] = (uint8_t)min((cum + step / 2) / step, 255); }
      }
    }
  } else {
    for (int i = tid; i < 768; i += AA_LUT_THREADS) {
      const int v = i & 255;
      uint8_t o;
      if (op == AA_BRIGHTNESS) o = aa_clamp_trunc(__fmul_rn((float)v, f));
      else if (op == AA_POSTERIZE) { const int bits = (int)f; o = bits >= 8 ? (uint8_t)v : (uint8_t)(v & (((1 << bits) - 1) << (8 - bits))); }
      else if (op == AA_INVERT) o = (uint8_t)(255 - v);
      else o = (float)v >= f ? (uint8_t)(255 - v) : (uint8_t)v;      // Solarize
      L[i] = o;
    }
  }
}

// One CTA per output row (n, oy), like the crop kernels, so the op is CTA-uniform; reads ping, writes pong (never in place: the
// geometric ops and Sharpness read neighbours).  kBilinear selects the geometric ops' resampling: nearest, or torchvision's
// _apply_grid_transform with fill None, evaluated as ATen's CPU kernels evaluate it: the grid of _affine_grid (the rescaled matrix,
// then bx·t0 fused into by·t1, then + t2, as the CPU bmm rounds it), grid_sample's unnormalize (g + 1)·(size/2) − ½, the four taps
// ((nw·v + ne·v) + sw·v) + se·v with separate roundings (a tap outside the image is 0), then round half to even.
template <bool kBilinear>
__global__ void __launch_bounds__(128) aa_apply_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const float* __restrict__ rec,
                                                       const uint8_t* __restrict__ lut, int slot, int slots, int ch, int cw) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int oy = blockIdx.x % ch, n = blockIdx.x / ch;
  const float* r = rec + ((long long)n * slots + slot) * AA_REC;
  const int op = (int)r[0];
  if (op == AA_NONE) return;
  const uint8_t* img = in + (long long)n * ch * cw * 3;
  const uint8_t* px = img + ((long long)oy * cw + ox) * 3;
  uint8_t* o = out + ((long long)blockIdx.x * cw + ox) * 3;
  if (kBilinear && op >= AA_SHEARX && op <= AA_ROTATE) {
    const float bx = (float)ox - 0.5f * (float)(cw - 1), by = (float)oy - 0.5f * (float)(ch - 1);
    const float hw = 0.5f * (float)cw, hh = 0.5f * (float)ch;
    const float gx = __fadd_rn(__fmaf_rn(by, __fdiv_rn(r[5], hw), __fmul_rn(bx, __fdiv_rn(r[4], hw))), __fdiv_rn(r[6], hw));
    const float gy = __fadd_rn(__fmaf_rn(by, __fdiv_rn(r[8], hh), __fmul_rn(bx, __fdiv_rn(r[7], hh))), __fdiv_rn(r[9], hh));
    const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), hw), 0.5f), iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), hh), 0.5f);
    const float xw = floorf(ix), yn = floorf(iy);
    const float w = __fsub_rn(ix, xw), e = __fsub_rn(1.f, w), nn = __fsub_rn(iy, yn), s = __fsub_rn(1.f, nn);
    const float wt[4] = {__fmul_rn(s, e), __fmul_rn(s, w), __fmul_rn(nn, e), __fmul_rn(nn, w)};   // nw, ne, sw, se
    const int x0 = (int)xw, y0 = (int)yn;
    const uint8_t* q[4];
    for (int t = 0; t < 4; ++t) {
      const int x = x0 + (t & 1), y = y0 + (t >> 1);
      q[t] = (x >= 0 && x < cw && y >= 0 && y < ch) ? img + ((long long)y * cw + x) * 3 : nullptr;
    }
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
      for (int t = 0; t < 4; ++t) v = t == 0 ? __fmul_rn(q[0] ? (float)q[0][c] : 0.f, wt[0]) : __fadd_rn(v, __fmul_rn(q[t] ? (float)q[t][c] : 0.f, wt[t]));
      o[c] = (uint8_t)(int)rintf(v);
    }
  } else if (op >= AA_SHEARX && op <= AA_ROTATE) {
    // nearest source of torchvision's affine grid: (m0·xb + m1·yb + m2) + (cw − 1)/2 about the centred output coordinates
    const float xb = (float)ox - 0.5f * (float)(cw - 1), yb = (float)oy - 0.5f * (float)(ch - 1);
    const float sx = __fmaf_rn(r[4], xb, __fmaf_rn(r[5], yb, r[6])) + 0.5f * (float)(cw - 1);
    const float sy = __fmaf_rn(r[7], xb, __fmaf_rn(r[8], yb, r[9])) + 0.5f * (float)(ch - 1);
    const float fx = rintf(sx), fy = rintf(sy);
    if (fx >= 0.f && fx <= (float)(cw - 1) && fy >= 0.f && fy <= (float)(ch - 1)) {
      const uint8_t* q = img + ((long long)fy * cw + (int)fx) * 3;
      o[0] = q[0]; o[1] = q[1]; o[2] = q[2];
    } else {
      o[0] = 0; o[1] = 0; o[2] = 0;
    }
  } else if (op == AA_COLOR) {
    const float f = r[1], d = r[2];
    const float g = aa_gray(px[0], px[1], px[2]);
    for (int c = 0; c < 3; ++c) o[c] = aa_clamp_trunc(__fmaf_rn(g, d, __fmul_rn((float)px[c], f)));
  } else if (op == AA_SHARPNESS) {
    if (oy == 0 || ox == 0 || oy == ch - 1 || ox == cw - 1) { o[0] = px[0]; o[1] = px[1]; o[2] = px[2]; return; }
    const float d = r[2];
    const long long rs = (long long)cw * 3;
    for (int c = 0; c < 3; ++c) {
      const uint8_t* q = px + c;
      const int S = q[-rs - 3] + q[-rs] + q[-rs + 3] + q[-3] + 5 * q[0] + q[3] + q[rs - 3] + q[rs] + q[rs + 3];
      const int blur = (2 * S + 13) / 26;                   // round(S / 13): S / 13 is never within 1/26 of a half
      const float x = (float)q[0];
      o[c] = aa_clamp_trunc(__fmaf_rn((float)blur - x, d, x));
    }
  } else if (op == AA_IDENTITY) {
    o[0] = px[0]; o[1] = px[1]; o[2] = px[2];
  } else {
    const uint8_t* L = lut + (long long)n * 768;
    o[0] = L[px[0]]; o[1] = L[256 + px[1]]; o[2] = L[512 + px[2]];
  }
}

// out = (u' − m̂)·s_c, m̂ the bilinear resample of the mean over image n's (mirrored) box with the crop kernels' taps: geometry moves
// content, not m̂, so a fill pixel becomes −m̂·s_c (torchvision's fill 0, then Normalize).
template <typename Tout>
__global__ void __launch_bounds__(128) aa_normalize_kernel(const uint8_t* __restrict__ u, const float* __restrict__ mean, int mean_mode,
                                                           float scale, const float* __restrict__ cscale, Tout* __restrict__ out,
                                                           const int4* __restrict__ boxes, const uint8_t* __restrict__ flips, int W,
                                                           int ch, int cw) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int oy = blockIdx.x % ch, n = blockIdx.x / ch;
  const long long e = ((long long)blockIdx.x * cw + ox) * 3;
  float m[3];
  if (mean_mode != 2) {
    for (int c = 0; c < 3; ++c) m[c] = mean_mode == 0 ? mean[0] : mean[c];
  } else {
    const int4 b = boxes[n];
    int iy0, iy1, ix0, ix1;
    float ly, lx;
    rrc_axis(oy, __fdiv_rn((float)b.z, (float)ch), b.z, iy0, iy1, ly);
    rrc_axis(flips[n] ? cw - 1 - ox : ox, __fdiv_rn((float)b.w, (float)cw), b.w, ix0, ix1, lx);
    const unsigned r0 = (unsigned)((b.x + iy0) * W + b.y) * 3u, r1 = (unsigned)((b.x + iy1) * W + b.y) * 3u;
    const unsigned t00 = r0 + 3u * ix0, t01 = r0 + 3u * ix1, t10 = r1 + 3u * ix0, t11 = r1 + 3u * ix1;
    const float wy0 = 1.f - ly, wx0 = 1.f - lx;
    for (int c = 0; c < 3; ++c)
      m[c] = wy0 * (wx0 * mean[t00 + c] + lx * mean[t01 + c]) + ly * (wx0 * mean[t10 + c] + lx * mean[t11 + c]);
  }
  for (int c = 0; c < 3; ++c) out[e + c] = (Tout)(((float)u[e + c] - m[c]) * (cscale ? scale * cscale[c] : scale));
}

void aa_crop_u8(const void* x, void* u, const void* boxes, const void* flips, int N, int H, int W, int ch, int cw, cudaStream_t st) {
  if ((long long)H * W * 3 >= (1LL << 31) || (long long)N * ch >= (1LL << 31)) throw std::runtime_error("aa_crop_u8: image too large");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  resized_crop_mirror_norm_kernel<uint8_t><<<g, 128, 0, st>>>((const uint8_t*)x, nullptr, 0, 1.f, nullptr, (uint8_t*)u, (const int4*)boxes,
                                                               (const uint8_t*)flips, H, W, 3, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("aa_crop_u8"); ::tmpi::check_capture(st, "aa_crop_u8");
}

void aa_lut(const void* u, const void* rec, void* lut, int slot, int slots, int N, int ch, int cw, cudaStream_t st) {
  if ((long long)ch * cw * 255 >= (1LL << 31)) throw std::runtime_error("aa_lut: image too large");
  aa_lut_kernel<<<N, AA_LUT_THREADS, 0, st>>>((const uint8_t*)u, (const float*)rec, (uint8_t*)lut, slot, slots, ch * cw);
  count_launch(); TMPI_CHECK_LAUNCH("aa_lut"); ::tmpi::check_capture(st, "aa_lut");
}

void aa_apply(const void* in, void* out, const void* rec, const void* lut, int slot, int slots, int N, int ch, int cw, int bilinear,
              cudaStream_t st) {
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  auto I = (const uint8_t*)in; auto O = (uint8_t*)out; auto R = (const float*)rec; auto Lt = (const uint8_t*)lut;
  if (bilinear) aa_apply_kernel<true><<<g, 128, 0, st>>>(I, O, R, Lt, slot, slots, ch, cw);
  else aa_apply_kernel<false><<<g, 128, 0, st>>>(I, O, R, Lt, slot, slots, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("aa_apply"); ::tmpi::check_capture(st, "aa_apply");
}

// AugMix's mix, in place on the crop u: per element acc = m₀·u, then for each chain acc = acc + w_i·c_i (separate fp32 roundings, as
// torchvision's mix.add_(w * aug)), then a truncating cast to uint8.  chains = [width][2][N, ch, cw, 3]: step s of chain i wrote
// buffer s & 1, so image n's chain i ends in buffer (depth − 1) & 1, its depth read from its records (AA_NONE steps trail the chain).
// Elementwise, so in place is safe.
__global__ void __launch_bounds__(128) aa_mix_kernel(uint8_t* __restrict__ u, const uint8_t* __restrict__ chains, const float* __restrict__ rec,
                                                     const float* __restrict__ weights, int width, int N, int ch, int cw) {
  const int ox = blockIdx.y * blockDim.x + threadIdx.x;
  if (ox >= cw) return;
  const int n = blockIdx.x / ch;
  const long long e = ((long long)blockIdx.x * cw + ox) * 3, img = (long long)N * ch * cw * 3;
  const float* wn = weights + (long long)n * (1 + width);
  float acc[3];
  for (int c = 0; c < 3; ++c) acc[c] = __fmul_rn(wn[0], (float)u[e + c]);
  for (int i = 0; i < width; ++i) {
    const float* r = rec + ((long long)n * 3 * width + 3 * i) * AA_REC;
    const int depth = 1 + ((int)r[AA_REC] != AA_NONE) + ((int)r[2 * AA_REC] != AA_NONE);
    const uint8_t* q = chains + (2 * i + ((depth - 1) & 1)) * img + e;
    const float wi = wn[1 + i];
    for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(wi, (float)q[c]));
  }
  for (int c = 0; c < 3; ++c) u[e + c] = (uint8_t)(int)acc[c];
}

void aa_mix(void* u, const void* chains, const void* rec, const void* weights, int width, int N, int ch, int cw, cudaStream_t st) {
  if ((long long)N * ch * cw * 3 * 2 * width >= (1LL << 40) || (long long)N * ch >= (1LL << 31)) throw std::runtime_error("aa_mix: batch too large");
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  aa_mix_kernel<<<g, 128, 0, st>>>((uint8_t*)u, (const uint8_t*)chains, (const float*)rec, (const float*)weights, width, N, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("aa_mix"); ::tmpi::check_capture(st, "aa_mix");
}

void aa_normalize(const void* u, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16, const void* boxes,
                  const void* flips, int N, int W, int ch, int cw, cudaStream_t st) {
  const dim3 g((unsigned)(N * ch), (unsigned)((cw + 127) / 128));
  auto U = (const uint8_t*)u; auto M = (const float*)mean; auto CS = (const float*)cscale; auto B = (const int4*)boxes; auto F = (const uint8_t*)flips;
  if (out_bf16) aa_normalize_kernel<__nv_bfloat16><<<g, 128, 0, st>>>(U, M, mean_mode, scale, CS, (__nv_bfloat16*)out, B, F, W, ch, cw);
  else aa_normalize_kernel<float><<<g, 128, 0, st>>>(U, M, mean_mode, scale, CS, (float*)out, B, F, W, ch, cw);
  count_launch(); TMPI_CHECK_LAUNCH("aa_normalize"); ::tmpi::check_capture(st, "aa_normalize");
}

// ============================================================================ loader: random erasing of the normalised output
// torchvision's RandomErasing(value=0) on the loader's output slot, in place: every element of image n's box (i, j, h, w) = boxes[n]
// (output coordinates, after the mirror; h = w = 0 erases nothing) is set to 0.  Both output dtypes store 0 as all-zero bits, so the
// kernel writes zero words of the element's width.  Grid (N, ERASE_ROW_CTAS): CTA (n, r) zeroes rows i + r, i + r + ERASE_ROW_CTAS, ...
// of box n, its threads striding the w·C contiguous elements of each row; no other element is read or written.
constexpr int ERASE_ROW_CTAS = 16;

template <typename T>
__global__ void __launch_bounds__(256) erase_boxes_kernel(T* __restrict__ out, const int4* __restrict__ boxes, int ch, int cw, int C) {
  const int n = blockIdx.x;
  const int4 b = boxes[n];                                               // (i, j, h, w), inside the output (host-drawn)
  const int len = b.w * C;
  for (int y = b.x + blockIdx.y; y < b.x + b.z; y += ERASE_ROW_CTAS) {
    T* row = out + (((long long)n * ch + y) * cw + b.y) * C;
    for (int e = threadIdx.x; e < len; e += blockDim.x) row[e] = T(0);
  }
}

void erase_boxes(void* out, int out_bf16, const void* boxes, int N, int ch, int cw, int C, cudaStream_t st) {
  const dim3 g((unsigned)N, ERASE_ROW_CTAS);
  if (out_bf16) erase_boxes_kernel<unsigned short><<<g, 256, 0, st>>>((unsigned short*)out, (const int4*)boxes, ch, cw, C);
  else erase_boxes_kernel<unsigned int><<<g, 256, 0, st>>>((unsigned int*)out, (const int4*)boxes, ch, cw, C);
  count_launch(); TMPI_CHECK_LAUNCH("erase_boxes"); ::tmpi::check_capture(st, "erase_boxes");
}

}  // namespace tmpi
