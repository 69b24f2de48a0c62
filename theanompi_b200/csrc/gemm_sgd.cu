// The wgmma GEMM with the momentum-SGD epilogue (gemm_wgmma<SgdEpilogue<T>, BN, 1>, see gemm_wgmma.cuh).  A translation unit
// of its own: instantiated next to the plain kernels, the tf32 SGD kernels change the code the compiler emits for the plain
// tf32 instantiations of the same tile shape.
#include "gemm_wgmma.cuh"

namespace tmpi {

// FC weight gradient G[M,N] = A^T B (A: [K, M] pitch lda, B: [K, N] pitch ldb, both MN-major) consumed by the momentum-SGD
// epilogue instead of being stored.  The tiles (BN = 128, or 64 when N <= 64) and the single K split are the ones gemm() picks
// for this un-split fp32 output, so the update sees the same G bits as sgd_flat would read.
namespace wgmma {
template <typename T>
static void gemm_sgd_host(const void* A, const void* B, int M, int N, int K, long long lda, long long ldb, const Params::Sgd& s,
                          cudaStream_t st) {
  using E = Elem<T>;
  constexpr int BK = E::BK, ESZ = E::ESZ;
  if (M <= 0 || N <= 0 || K <= 0) return;
  if ((s.ldw % 4) != 0 || (reinterpret_cast<uintptr_t>(s.W) & 15) != 0 || (reinterpret_cast<uintptr_t>(s.U) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(s.H) & 7) != 0 || s.lr_ptr == nullptr)
    throw std::runtime_error("gemm_sgd: W / U need 16-byte aligned rows (ldw % 4 == 0), H 8-byte aligned rows, and an lr pointer");
  const int BN = N <= 64 ? 64 : 128;
  Params p;
  p.C = nullptr; p.bias = nullptr; p.alpha = 1.f; p.M = M; p.N = N; p.K = K; p.ldc = s.ldw; p.a_mn = 1; p.b_mn = 1;
  p.out_bf16 = 0; p.bias_mode = 0; p.relu = 0; p.atomic_out = 0;
  p.mt = (M + BM - 1) / BM; p.nt = (N + BN - 1) / BN; p.splits = 1;
  p.num_kb = (K + BK - 1) / BK; p.kb_per_split = p.num_kb; p.conv_mode = 0;
  p.group_m = (p.mt > 12 && p.nt > 12) ? 12 : 0;
  p.cHo = p.cWo = p.cS = p.cP = p.cKH = p.cKW = p.cCg = p.c_chunks = 0;
  p.sgd = s;
  CUtensorMap ta = make_tmap(A, (uint64_t)M, (uint64_t)K, (uint64_t)lda * ESZ, (uint32_t)BK, ESZ, 1);
  CUtensorMap tb = make_tmap(B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * ESZ, (uint32_t)BK, ESZ, 1);
  if (BN == 128) launch<SgdEpilogue<T>, 128, 1>(ta, tb, p, 1, st);
  else launch<SgdEpilogue<T>, 64, 1>(ta, tb, p, 1, st);
}
}  // namespace wgmma

void gemm_sgd(const void* A, const void* B, void* W, void* U, void* H, const void* lr_ptr, float lr_mult, float wd, float mu, int nesterov,
              float inv_k, int M, int N, int K, long long lda, long long ldb, long long ldw, int f32, cudaStream_t st) {
  wgmma::Params::Sgd s;
  s.W = static_cast<float*>(W); s.U = static_cast<float*>(U); s.H = static_cast<__nv_bfloat16*>(H);
  s.lr_ptr = static_cast<const float*>(lr_ptr); s.lr_mult = lr_mult; s.wd = wd; s.mu = mu; s.inv_k = inv_k; s.nesterov = nesterov;
  s.ldw = ldw;
  if (f32) wgmma::gemm_sgd_host<float>(A, B, M, N, K, lda, ldb, s, st);
  else wgmma::gemm_sgd_host<__nv_bfloat16>(A, B, M, N, K, lda, ldb, s, st);
}

}  // namespace tmpi
