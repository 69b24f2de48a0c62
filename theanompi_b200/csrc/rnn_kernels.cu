// LSTM cell, embedding gather / scatter and masked mean pooling for the IMDB LSTM (ref theanompi/models/lstm.py:117-253 — the Theano
// tutorial LSTM: preact = x_t·W + h_{t-1}·U + b, gates sliced i | f | o | c̃, masked state carry, mean pooling over time).
// The matrix products run on the wgmma GEMM (ops/rnn.py); these kernels are the fused elementwise parts, forward and backward.
// Activations T = bf16 or fp32 (tf32 mode); the cell state and all accumulations are fp32.
#include "common.cuh"
#include "api.h"

namespace tmpi {

static inline int grid_r(long long n, int block) { return (int)((n + block - 1) / block); }
template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + __expf(-x)); }

// gx, gh: [B, 4H] pre-activation halves (input projection incl. bias, recurrent projection);  act: post-activation gates
template <typename T>
__global__ void lstm_cell_fwd_kernel(const T* __restrict__ gx, const T* __restrict__ gh, const float* __restrict__ c_prev,
                                     const T* __restrict__ h_prev, const float* __restrict__ mask, T* __restrict__ act,
                                     float* __restrict__ c_out, T* __restrict__ h_out, int B, int H) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H, j = idx - b * H;
  const long long g0 = (long long)b * 4 * H + j;
  const float i = sigm(ldf(gx + g0) + ldf(gh + g0));
  const float f = sigm(ldf(gx + g0 + H) + ldf(gh + g0 + H));
  const float o = sigm(ldf(gx + g0 + 2 * H) + ldf(gh + g0 + 2 * H));
  const float g = tanhf(ldf(gx + g0 + 3 * H) + ldf(gh + g0 + 3 * H));
  const float cp = c_prev[idx], hp = ldf(h_prev + idx), m = mask[b];
  const float ct = f * cp + i * g;
  const float ht = o * tanhf(ct);
  c_out[idx] = m * ct + (1.f - m) * cp;
  stf(h_out + idx, m * ht + (1.f - m) * hp);
  stf(act + g0, i); stf(act + g0 + H, f); stf(act + g0 + 2 * H, o); stf(act + g0 + 3 * H, g);
}

// dh_out: gradient reaching h_t from the layers above; dh_rec: gradient from step t+1 through the recurrent projection (may be null);
// dc_next: gradient wrt c_t from step t+1.  Writes the pre-activation gate gradient dG [B, 4H], dc_prev and the part of dh that
// by-passes the cell through the mask (dh_pass).
template <typename T>
__global__ void lstm_cell_bwd_kernel(const T* __restrict__ dh_out, const T* __restrict__ dh_rec, const float* __restrict__ dh_pass_in,
                                     const float* __restrict__ dc_next, const T* __restrict__ act, const float* __restrict__ c,
                                     const float* __restrict__ c_prev, const float* __restrict__ mask, T* __restrict__ dG,
                                     float* __restrict__ dc_prev, float* __restrict__ dh_pass, int B, int H) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H, j = idx - b * H;
  const long long g0 = (long long)b * 4 * H + j;
  const float m = mask[b];
  float dh = ldf(dh_out + idx);
  if (dh_rec) dh += ldf(dh_rec + idx);
  if (dh_pass_in) dh += dh_pass_in[idx];
  const float dcn = dc_next ? dc_next[idx] : 0.f;
  const float i = ldf(act + g0), f = ldf(act + g0 + H), o = ldf(act + g0 + 2 * H), g = ldf(act + g0 + 3 * H);
  const float tc = tanhf(c[idx]);                  // masked rows: multiplied by m = 0 below
  const float dht = m * dh;
  const float dct = m * dcn + dht * o * (1.f - tc * tc);
  dc_prev[idx] = dct * f + (1.f - m) * dcn;
  dh_pass[idx] = (1.f - m) * dh;
  stf(dG + g0, dct * g * i * (1.f - i));
  stf(dG + g0 + H, dct * c_prev[idx] * f * (1.f - f));
  stf(dG + g0 + 2 * H, dht * tc * o * (1.f - o));
  stf(dG + g0 + 3 * H, dct * i * (1.f - g * g));
}

// out[n, :] = W[ids[n], :]   (W: T = the compute copy of the embedding table)
template <typename T>
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const T* __restrict__ W, T* __restrict__ out, long long n, int D) {
  const long long row = blockIdx.x;
  if (row >= n) return;
  const T* src = W + ids[row] * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) out[row * D + d] = src[d];
}
template <typename T>
__global__ void embedding_bwd_kernel(const long long* __restrict__ ids, const T* __restrict__ dout, float* __restrict__ dW, long long n, int D) {
  const long long row = blockIdx.x;
  if (row >= n) return;
  float* dst = dW + ids[row] * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) atomicAdd(dst + d, ldf(dout + row * D + d));
}

// Deterministic mode: dW[v, :] = ((dout[r0] + dout[r1]) + dout[r2]) + ... over the rows r0 < r1 < ... with ids[r] = v, in
// ascending row order and without atomics.  CTA k owns the ids [k·EMB_DET_IDS, (k + 1)·EMB_DET_IDS): it walks all rows in chunks
// of EMB_DET_CHUNK, compacts the chunk's rows that hit its ids into an ordered list (block-wide scan) and then each thread adds
// its columns of those rows in list order.  A thread keeps the running sum of the current id in a register and writes it back
// when the id changes, so the padding id's long run costs one fp32 add per row.
constexpr int EMB_DET_IDS = 64, EMB_DET_THREADS = 256, EMB_DET_PER_THREAD = 4, EMB_DET_CHUNK = EMB_DET_THREADS * EMB_DET_PER_THREAD;
template <typename T>
__global__ void __launch_bounds__(EMB_DET_THREADS) embedding_bwd_det_kernel(const long long* __restrict__ ids, const T* __restrict__ dout,
                                                                            float* __restrict__ dW, int n, int D, long long V) {
  __shared__ int hit_row[EMB_DET_CHUNK], hit_id[EMB_DET_CHUNK], warp_tot[EMB_DET_THREADS / 32];
  const long long v0 = (long long)blockIdx.x * EMB_DET_IDS;
  const int nv = (int)min((long long)EMB_DET_IDS, V - v0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += EMB_DET_CHUNK) {
    int loc[EMB_DET_PER_THREAD], cnt = 0;
#pragma unroll
    for (int j = 0; j < EMB_DET_PER_THREAD; ++j) {
      const int r = base + threadIdx.x * EMB_DET_PER_THREAD + j;
      const long long v = r < n ? ids[r] - v0 : -1;
      loc[j] = (v >= 0 && v < nv) ? (int)v : -1;
      cnt += loc[j] >= 0;
    }
    int incl = cnt;                                   // block-wide exclusive scan of the per-thread hit counts
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += x; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int pos = incl - cnt, total = 0;
    for (int w = 0; w < EMB_DET_THREADS / 32; ++w) { if (w < warp) pos += warp_tot[w]; total += warp_tot[w]; }
#pragma unroll
    for (int j = 0; j < EMB_DET_PER_THREAD; ++j)
      if (loc[j] >= 0) { hit_row[pos] = base + threadIdx.x * EMB_DET_PER_THREAD + j; hit_id[pos] = loc[j]; ++pos; }
    __syncthreads();
    for (int d = threadIdx.x; d < D; d += EMB_DET_THREADS) {
      int cur = -1;
      float acc = 0.f;
      for (int k = 0; k < total; ++k) {
        const int v = hit_id[k];
        const float x = ldf(dout + (long long)hit_row[k] * D + d);
        if (v != cur) {
          if (cur >= 0) dW[(v0 + cur) * D + d] = acc;
          cur = v;
          acc = dW[(v0 + v) * D + d];
        }
        acc += x;
      }
      if (cur >= 0) dW[(v0 + cur) * D + d] = acc;
    }
    __syncthreads();                                  // hit_row / hit_id / warp_tot are rewritten by the next chunk
  }
}

// pooled[b, :] = sum_t h[t, b, :] * mask[t, b] / max(1, sum_t mask[t, b])     (h: [T, B, H])
template <typename T>
__global__ void masked_mean_fwd_kernel(const T* __restrict__ h, const float* __restrict__ mask, T* __restrict__ out, int Tn, int B, int H) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H;
  float acc = 0.f, cnt = 0.f;
  for (int t = 0; t < Tn; ++t) { const float m = mask[t * B + b]; acc += m * ldf(h + (long long)t * B * H + idx); cnt += m; }
  stf(out + idx, acc / fmaxf(cnt, 1.f));
}
template <typename T>
__global__ void masked_mean_bwd_kernel(const T* __restrict__ dout, const float* __restrict__ mask, T* __restrict__ dh, int Tn, int B, int H) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Tn * B * H) return;
  const int bh = (int)(idx % ((long long)B * H));
  const int t = (int)(idx / ((long long)B * H));
  const int b = bh / H;
  float cnt = 0.f;
  for (int s = 0; s < Tn; ++s) cnt += mask[s * B + b];
  stf(dh + idx, ldf(dout + bh) * mask[t * B + b] / fmaxf(cnt, 1.f));
}

#define TMPI_RNN_DISPATCH(CALL_F32, CALL_BF16) do { if (f32) { CALL_F32; } else { CALL_BF16; } } while (0)

void lstm_cell_fwd(const void* gx, const void* gh, const void* c_prev, const void* h_prev, const void* mask, void* act, void* c_out, void* h_out,
                   int B, int H, int f32, cudaStream_t st) {
  const int g = grid_r((long long)B * H, 256);
  TMPI_RNN_DISPATCH(
      (lstm_cell_fwd_kernel<float><<<g, 256, 0, st>>>((const float*)gx, (const float*)gh, (const float*)c_prev, (const float*)h_prev, (const float*)mask,
                                                      (float*)act, (float*)c_out, (float*)h_out, B, H)),
      (lstm_cell_fwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((const __nv_bfloat16*)gx, (const __nv_bfloat16*)gh, (const float*)c_prev,
                                                              (const __nv_bfloat16*)h_prev, (const float*)mask, (__nv_bfloat16*)act, (float*)c_out,
                                                              (__nv_bfloat16*)h_out, B, H)));
  count_launch(); TMPI_CHECK_LAUNCH("lstm_cell_fwd"); ::tmpi::check_capture(st, "lstm_cell_fwd");
}
void lstm_cell_bwd(const void* dh_out, const void* dh_rec, const void* dh_pass_in, const void* dc_next, const void* act, const void* c,
                   const void* c_prev, const void* mask, void* dG, void* dc_prev, void* dh_pass, int B, int H, int f32, cudaStream_t st) {
  const int g = grid_r((long long)B * H, 256);
  TMPI_RNN_DISPATCH(
      (lstm_cell_bwd_kernel<float><<<g, 256, 0, st>>>((const float*)dh_out, (const float*)dh_rec, (const float*)dh_pass_in, (const float*)dc_next,
                                                      (const float*)act, (const float*)c, (const float*)c_prev, (const float*)mask, (float*)dG,
                                                      (float*)dc_prev, (float*)dh_pass, B, H)),
      (lstm_cell_bwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((const __nv_bfloat16*)dh_out, (const __nv_bfloat16*)dh_rec, (const float*)dh_pass_in,
                                                              (const float*)dc_next, (const __nv_bfloat16*)act, (const float*)c, (const float*)c_prev,
                                                              (const float*)mask, (__nv_bfloat16*)dG, (float*)dc_prev, (float*)dh_pass, B, H)));
  count_launch(); TMPI_CHECK_LAUNCH("lstm_cell_bwd"); ::tmpi::check_capture(st, "lstm_cell_bwd");
}
void embedding_fwd(const void* ids, const void* W, void* out, long long n, int D, int f32, cudaStream_t st) {
  if (n <= 0) return;
  TMPI_RNN_DISPATCH((embedding_fwd_kernel<float><<<(unsigned)n, 128, 0, st>>>((const long long*)ids, (const float*)W, (float*)out, n, D)),
                    (embedding_fwd_kernel<__nv_bfloat16><<<(unsigned)n, 128, 0, st>>>((const long long*)ids, (const __nv_bfloat16*)W, (__nv_bfloat16*)out, n, D)));
  count_launch(); TMPI_CHECK_LAUNCH("embedding_fwd"); ::tmpi::check_capture(st, "embedding_fwd");
}
void embedding_bwd(const void* ids, const void* dout, void* dW, long long n, int D, long long V, int f32, cudaStream_t st) {
  check_cuda(cudaMemsetAsync(dW, 0, (size_t)V * D * 4, st), "embedding_bwd memset");
  if (n <= 0) return;
  if (deterministic_mode()) {                       // fixed ascending-row order per id, no float atomics
    if (n > 0x7fffffffLL) throw std::runtime_error("embedding_bwd: too many rows for the deterministic mode");
    const unsigned g = (unsigned)((V + EMB_DET_IDS - 1) / EMB_DET_IDS);
    TMPI_RNN_DISPATCH(
        (embedding_bwd_det_kernel<float><<<g, EMB_DET_THREADS, 0, st>>>((const long long*)ids, (const float*)dout, (float*)dW, (int)n, D, V)),
        (embedding_bwd_det_kernel<__nv_bfloat16><<<g, EMB_DET_THREADS, 0, st>>>((const long long*)ids, (const __nv_bfloat16*)dout, (float*)dW,
                                                                                (int)n, D, V)));
    count_launch(); TMPI_CHECK_LAUNCH("embedding_bwd"); ::tmpi::check_capture(st, "embedding_bwd");
    return;
  }
  TMPI_RNN_DISPATCH((embedding_bwd_kernel<float><<<(unsigned)n, 128, 0, st>>>((const long long*)ids, (const float*)dout, (float*)dW, n, D)),
                    (embedding_bwd_kernel<__nv_bfloat16><<<(unsigned)n, 128, 0, st>>>((const long long*)ids, (const __nv_bfloat16*)dout, (float*)dW, n, D)));
  count_launch(); TMPI_CHECK_LAUNCH("embedding_bwd"); ::tmpi::check_capture(st, "embedding_bwd");
}
void masked_mean_fwd(const void* h, const void* mask, void* out, int Tn, int B, int H, int f32, cudaStream_t st) {
  const int g = grid_r((long long)B * H, 256);
  TMPI_RNN_DISPATCH((masked_mean_fwd_kernel<float><<<g, 256, 0, st>>>((const float*)h, (const float*)mask, (float*)out, Tn, B, H)),
                    (masked_mean_fwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((const __nv_bfloat16*)h, (const float*)mask, (__nv_bfloat16*)out, Tn, B, H)));
  count_launch(); TMPI_CHECK_LAUNCH("masked_mean_fwd"); ::tmpi::check_capture(st, "masked_mean_fwd");
}
void masked_mean_bwd(const void* dout, const void* mask, void* dh, int Tn, int B, int H, int f32, cudaStream_t st) {
  const int g = grid_r((long long)Tn * B * H, 256);
  TMPI_RNN_DISPATCH((masked_mean_bwd_kernel<float><<<g, 256, 0, st>>>((const float*)dout, (const float*)mask, (float*)dh, Tn, B, H)),
                    (masked_mean_bwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((const __nv_bfloat16*)dout, (const float*)mask, (__nv_bfloat16*)dh, Tn, B, H)));
  count_launch(); TMPI_CHECK_LAUNCH("masked_mean_bwd"); ::tmpi::check_capture(st, "masked_mean_bwd");
}

}  // namespace tmpi
