// Host side of the wgmma GEMM / implicit-GEMM convolution (the kernel: gemm_wgmma.cuh).  The SGD-epilogue instantiations
// live in gemm_sgd.cu, so adding them leaves the code of the instantiations here unchanged.
#include "gemm_wgmma.cuh"
#include <vector>

namespace tmpi {
std::atomic<unsigned long long> g_launch_count{0};

namespace wgmma {

int g_dbg = 0;

// Split-K factor for a persistent grid of `sms` CTAs walking equal-length tiles round-robin: minimise
// waves x (k-blocks per slice + per-tile overhead).  A plain ceil(sms / tiles) overshoots the machine by a few tiles
// and pays a whole second wave for them (conv2 wgrad: 13 tiles x 11 slices = 143 > 132).
static int choose_splits(int tiles, int num_kb, int sms) {
  // TMPI_DETERMINISTIC=1: never split K — split-K slices combine with fp32 red.global.add in arrival order, so weight gradients
  // differ in the last bits from run to run; without it every output element is produced by ONE CTA in a fixed k order
  if (deterministic_mode()) return 1;
  if (tiles >= sms || num_kb < 8) return 1;
  const int kTileOverheadKb = 4;                    // pipeline fill + accumulator hand-off, in k-block units
  int best = 1;
  long long best_cost = -1;
  const int max_s = std::min(num_kb / 4, 4 * sms);
  for (int s = 1; s <= max_s; ++s) {
    const int kb_per = (num_kb + s - 1) / s;
    const int s_eff = (num_kb + kb_per - 1) / kb_per;
    const long long waves = ((long long)tiles * s_eff + sms - 1) / sms;
    const long long cost = waves * (kb_per + kTileOverheadKb) * 64 + s_eff;     // tie-break: fewer slices (less atomic traffic)
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = s_eff; }
  }
  return best;
}

// 256-row tiles (MT = 2) when the output is not split-K and the wave arithmetic favours them: a tall tile shares the B tile
// and the per-k-block barrier traffic between two sub-tiles, so it is taken as costing 1.7x a 128-row tile; it wins unless
// halving the tile count wastes most of a wave.
static bool use_tall_tiles(long long M, int nt, int eligible, int sms) {
  if (!eligible || M < 2 * BM) return false;
  const long long t1 = ((M + BM - 1) / BM) * nt, t2 = ((M + 2 * BM - 1) / (2 * BM)) * nt;
  const long long w1 = (t1 + sms - 1) / sms, w2 = (t2 + sms - 1) / sms;
  return w2 * 17 <= w1 * 10;
}

// Tile of an implicit-GEMM convolution: the layout-legal (BN, MT) with the least estimated time.  A persistent launch takes
// waves x (time of one tile); a tile costs (its k-blocks + kTileOverheadKb for pipeline fill and epilogue) x (the columns of
// wgmma work it issues per k-block, MT x BN, zero-filled columns past N included, + a fixed per-k-block cost of barrier waits
// and wgmma.wait_group worth kKblockCols columns).  256-row tiles are candidates only where use_tall_tiles accepts them;
// split-K (wgrad) is planned per candidate exactly as the launcher will run it.
//   kind 0 fprop: K-major weights, BN 64 / 96 / 128 / 192;  kind 1 dgrad: MN-major weights, BN a whole number of 64-wide
//   bf16 atoms;  kind 2 wgrad: fp32 split-K output, 128-row tiles of BN / ATOM (tap, channel-chunk) boxes.
//   N: output columns (wgrad: boxes x ATOM, the columns the kernel issues).  BN = 192 tiles are 128 rows only: 2 x 96
//   accumulators per thread would not fit next to the rest of the consumer's registers.
struct ConvTile { int bn, mt, splits; };
static ConvTile choose_conv_tile(int kind, long long M, int N, int groups, int num_kb, int tall_ok, int sms) {
  static const int kCand[7][2] = {{128, 2}, {128, 1}, {192, 1}, {96, 2}, {96, 1}, {64, 2}, {64, 1}};   // ties: first wins
  const int kTileOverheadKb = 4, kKblockCols = 64;
  // 3-box wgrad tiles only for deep reductions: on an H100 they paid off for AlexNet-128b's conv1 / conv2 wgrads (6050 /
  // 1458 pixel blocks) but cost GoogLeNet-32b about 1.5 % of its step with the shallow (25-400 block) wgrads of its inception
  // layers, which the cost model above does not see
  const int kWideWgradMinKb = 1024;
  ConvTile best{0, 0, 1};
  long long best_cost = -1;
  for (const auto& c : kCand) {
    const int bn = c[0], mt = c[1];
    if (bn == 96 && kind != 0) continue;
    if (kind == 2 && (bn == 64 || mt == 2)) continue;
    if (kind == 2 && bn == 192 && num_kb < kWideWgradMinKb) continue;
    const int nt = (N + bn - 1) / bn;
    if (mt == 2 && !use_tall_tiles(M, nt * groups, tall_ok, sms)) continue;
    const long long tiles = ((M + mt * BM - 1) / (mt * BM)) * nt * groups;
    int splits = kind == 2 ? choose_splits((int)tiles, num_kb, sms) : 1;
    const int kb_per = (num_kb + splits - 1) / splits;
    splits = (num_kb + kb_per - 1) / kb_per;
    const long long waves = (tiles * splits + sms - 1) / sms;
    const long long cost = waves * (kb_per + kTileOverheadKb) * (mt * bn + kKblockCols);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = {bn, mt, splits}; }
  }
  return best;
}

}  // namespace wgmma

void gemm_set_debug(int flags) { wgmma::g_dbg = flags; }

// ---- reduce-scatter epilogue registry (see api.h)
namespace wgmma {
struct RsRange { const char* lo; const char* hi; long long blo, per; };
static int g_rs_world = 0, g_rs_rank = 0;
static float* g_rs_peer[kMaxRanks] = {};
static const char* g_rs_local = nullptr;
static std::vector<RsRange> g_rs_ranges;
static std::mutex g_rs_mu;
// fills the rs_* fields of p when C lies in a registered tensor; returns true if the epilogue will reduce-scatter
static bool rs_lookup(const void* C, Params& p) {
  std::lock_guard<std::mutex> lk(g_rs_mu);
  if (g_rs_world < 2) return false;
  const char* c = reinterpret_cast<const char*>(C);
  for (const RsRange& r : g_rs_ranges) {
    if (c >= r.lo && c < r.hi) {
      p.rs_world = g_rs_world; p.rs_rank = g_rs_rank;
      p.rs_blo = (unsigned)r.blo; p.rs_per = (unsigned)std::max<long long>(1, r.per);
      p.rs_e0 = (long long)((c - g_rs_local) / 4);
      for (int q = 0; q < kMaxRanks; ++q) p.rs_g[q] = q < g_rs_world ? g_rs_peer[q] : nullptr;
      return true;
    }
  }
  return false;
}
}  // namespace wgmma

void gemm_rs_configure(int world, const void* const* peer_g, const void* local_g) {
  std::lock_guard<std::mutex> lk(wgmma::g_rs_mu);
  if (world > kMaxRanks) throw std::runtime_error("gemm_rs_configure: too many ranks");
  wgmma::g_rs_world = world;
  wgmma::g_rs_local = reinterpret_cast<const char*>(local_g);
  wgmma::g_rs_rank = 0;
  for (int q = 0; q < world; ++q) {
    wgmma::g_rs_peer[q] = reinterpret_cast<float*>(const_cast<void*>(peer_g[q]));
    if (peer_g[q] == local_g) wgmma::g_rs_rank = q;
  }
  wgmma::g_rs_ranges.clear();
}
void gemm_rs_add_range(const void* c_lo, const void* c_hi, long long blo, long long per) {
  std::lock_guard<std::mutex> lk(wgmma::g_rs_mu);
  wgmma::g_rs_ranges.push_back({reinterpret_cast<const char*>(c_lo), reinterpret_cast<const char*>(c_hi), blo, per});
}
void gemm_rs_clear() {
  std::lock_guard<std::mutex> lk(wgmma::g_rs_mu);
  wgmma::g_rs_world = 0; wgmma::g_rs_ranges.clear();
}

// host-side planning helpers, exported so the wave arithmetic can be unit-tested without a GPU
int gemm_plan_splits(int tiles, int num_kb, int sms) { return wgmma::choose_splits(tiles, num_kb, sms); }
int gemm_plan_tall(long long M, int nt, int out_bf16, int sms) { return wgmma::use_tall_tiles(M, nt, out_bf16, sms) ? 1 : 0; }
std::tuple<int, int, int> gemm_plan_conv(int kind, long long M, int N, int groups, int num_kb, int tall_ok, int sms) {
  const wgmma::ConvTile t = wgmma::choose_conv_tile(kind, M, N, groups, num_kb, tall_ok, sms);
  return {t.bn, t.mt, t.splits};
}

// C[M,N] (ldc) = alpha * op(A) op(B) + bias, optional ReLU.
//   a_mn == 0: A is [M, K] with row pitch lda (elements);  a_mn == 1: A is [K, M] with row pitch lda.
//   b_mn == 0: B is [N, K] with row pitch ldb;             b_mn == 1: B is [K, N] with row pitch ldb.
//   bn_hint: 0 = auto, else 32/64/128.  splitk: 0 = auto, 1 = none, >1 = forced (fp32 output only, no bias/relu).
//   accumulate = 1: C += op(A) op(B) (fp32 output only, no bias/relu): every tile reaches C through the epilogue's fp32 reductions
//   and the split-K clear is skipped (gradient accumulation into the arena's G).
//   T = __nv_bfloat16: bf16 operands (wgmma bf16), bf16 or fp32 output.  T = float: fp32 operands (wgmma tf32), fp32 output.
namespace wgmma {
template <typename T>
static void gemm_host(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long lda, long long ldb,
                      long long ldc, int a_mn, int b_mn, int out_bf16, int bias_mode, int relu, float alpha, int bn_hint, int splitk,
                      int accumulate, cudaStream_t st) {
  using E = Elem<T>;
  constexpr int BK = E::BK, ATOM = E::ATOM, ESZ = E::ESZ;
  if (M <= 0 || N <= 0 || K <= 0) return;
  const int sms = sm_count();
  const int mt = (M + BM - 1) / BM;
  const bool fused_epi = bias_mode != 0 || relu;
  const bool can_split = (!out_bf16) && !fused_epi;
  if (accumulate && !can_split) throw std::runtime_error("gemm: accumulate needs an fp32 output without bias / ReLU");
  int BN = bn_hint;
  if (BN == 0) {
    BN = 128;
    // Narrow tiles only buy parallelism when split-K cannot (fused bias/ReLU or bf16 output): with split-K available the
    // wide tile is always better — every extra n-tile re-reads the whole A operand through L2.
    if (!(can_split && splitk != 1)) {
      if (mt * ((N + 127) / 128) < sms && N >= 64) BN = 64;
      if (BN == 64 && mt * ((N + 63) / 64) < sms && !b_mn && N >= 32) BN = 32;
    } else if (N <= 64) {
      BN = 64;
    }
  }
  if (b_mn && BN < 64) BN = 64;
  const int nt = (N + BN - 1) / BN;
  const int num_kb = (K + BK - 1) / BK;
  int splits = 1;
  if (splitk > 1 && can_split) splits = splitk;
  else if (splitk == 0 && can_split) splits = choose_splits(mt * nt, num_kb, sms);
  int kb_per = (num_kb + splits - 1) / splits;
  splits = (num_kb + kb_per - 1) / kb_per;          // every slice owns >= 1 k-block

  Params p;
  p.C = C; p.bias = bias; p.alpha = alpha; p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.a_mn = a_mn; p.b_mn = b_mn;
  p.out_bf16 = out_bf16; p.bias_mode = bias ? bias_mode : 0; p.relu = relu; p.kb_per_split = kb_per; p.atomic_out = splits > 1 || accumulate;
  // tall tiles: bf16 path — bf16 outputs (fprop / dgrad); tf32 path — un-split outputs of K-major operands
  const int tall_ok = ESZ == 2 ? out_bf16 : (!a_mn && !b_mn);
  const bool tall = splits == 1 && BN >= 64 && use_tall_tiles(M, nt, tall_ok, sms);
  p.mt = tall ? (M + 2 * BM - 1) / (2 * BM) : mt; p.nt = nt; p.splits = splits; p.num_kb = num_kb; p.conv_mode = 0;
  p.group_m = (p.mt > 12 && nt > 12) ? (tall ? 8 : 12) : 0;
  p.cHo = p.cWo = p.cS = p.cP = p.cKH = p.cKW = p.cCg = p.c_chunks = 0;
  // wgrad outputs registered for the fused reduce-scatter: every vector is red.add-ed into its owner's G (the exchange kernel
  // clears G after consuming it, so there is no memset here — a memset would race with the peers' adds)
  const bool rs = !accumulate && (!out_bf16) && bias_mode == 0 && !relu && alpha == 1.f && (ldc % 4) == 0 && rs_lookup(C, p);
  if (rs) {
    p.atomic_out = 1;
  } else if (splits > 1 && !accumulate) {
    // split-K accumulates with fp32 atomics: clear the (possibly strided) output first
    check_cuda(cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, st), "gemm split-K memset");
  }
  CUtensorMap ta = a_mn ? make_tmap(A, (uint64_t)M, (uint64_t)K, (uint64_t)lda * ESZ, (uint32_t)BK, ESZ, 1)
                        : make_tmap(A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * ESZ, (uint32_t)BM, ESZ, 0);
  CUtensorMap tb = b_mn ? make_tmap(B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * ESZ, (uint32_t)BK, ESZ, 1)
                        : make_tmap(B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * ESZ, (uint32_t)BN, ESZ, 0);
  (void)ATOM;
  if (tall) { if (BN == 128) launch<T, 128, 2>(ta, tb, p, splits, st); else launch<T, 64, 2>(ta, tb, p, splits, st); }
  else if (BN == 128) launch<T, 128, 1>(ta, tb, p, splits, st);
  else if (BN == 64) launch<T, 64, 1>(ta, tb, p, splits, st);
  else launch<T, 32, 1>(ta, tb, p, splits, st);
}
}  // namespace wgmma

void gemm(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long lda, long long ldb,
          long long ldc, int a_mn, int b_mn, int out_bf16, int bias_mode, int relu, float alpha, int bn_hint, int splitk, int f32,
          cudaStream_t st, int accumulate) {
  if (f32) wgmma::gemm_host<float>(A, B, C, bias, M, N, K, lda, ldb, ldc, a_mn, b_mn, 0, bias_mode, relu, alpha, bn_hint, splitk, accumulate, st);
  else wgmma::gemm_host<__nv_bfloat16>(A, B, C, bias, M, N, K, lda, ldb, ldc, a_mn, b_mn, out_bf16, bias_mode, relu, alpha, bn_hint, splitk,
                                       accumulate, st);
}

// ------------------------------------------------------------------ implicit-GEMM convolution (TMA im2col)
namespace wgmma {
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                     const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeIm2col get_encode_im2col() {
  static PFN_encodeIm2col fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeIm2col)f;
    (void)cudaGetLastError();
  });
  if (!fn) throw std::runtime_error("tmpi_native: cuTensorMapEncodeIm2col unavailable");
  return fn;
}

// NHWC activation (channel slice [c_off, c_off+Cg) of a tensor with Ctot channels) as an im2col tensor map:
// box = pixels x 128 bytes of channels (64 bf16 / 32 fp32), 128 B swizzle, zero fill for padding / out-of-range pixels /
// channels >= Cg.
static CUtensorMap make_im2col_map(const void* x, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int S, int P, int pixels,
                                   int esz, int mn_major) {
  const char* base = reinterpret_cast<const char*>(x) + (size_t)c_off * esz;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((Ctot * esz) % 16) != 0) throw std::runtime_error("tmpi_native: im2col operand must be 16B aligned");
  using Key = std::tuple<const void*, int, int, int, int, int, int, int, int, int, int, int, int>;
  static std::map<Key, CUtensorMap> cache;
  static std::mutex mu;
  Key key{base, N, H, W, Ctot, Cg, KH, KW, S, P, pixels, esz, mn_major};
  const CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  CUtensorMap m;
  cuuint64_t dims[4] = {(cuuint64_t)Cg, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)Ctot * esz, (cuuint64_t)W * Ctot * esz, (cuuint64_t)H * W * Ctot * esz};
  int lower[2] = {-P, -P};
  int upper[2] = {P - (KW - 1), P - (KH - 1)};
  cuuint32_t estr[4] = {1u, (cuuint32_t)S, (cuuint32_t)S, 1u};
  CUresult r = get_encode_im2col()(&m, map_type(esz), 4, const_cast<char*>(base),
                                   dims, strides, lower, upper, (cuuint32_t)(128 / esz), (cuuint32_t)pixels, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("tmpi_native: cuTensorMapEncodeIm2col failed, code " + std::to_string((int)r));
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  return m;
}

// weights [O][KH*KW][Cg] (contiguous) as a 3-D tiled map, box {box_c ch, 1 tap, box_o out-channels}
static CUtensorMap make_weight_map(const void* w, int O, int taps, int Cg, int box_o, int box_c, int esz, int mn_major) {
  if ((reinterpret_cast<uintptr_t>(w) & 15) != 0 || ((Cg * esz) % 16) != 0) throw std::runtime_error("tmpi_native: conv weights must be 16B aligned, C * esz % 16 == 0");
  using Key = std::tuple<const void*, int, int, int, int, int, int, int>;
  static std::map<Key, CUtensorMap> cache;
  static std::mutex mu;
  Key key{w, O, taps, Cg, box_o, box_c, esz, mn_major};
  const CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  CUtensorMap m;
  cuuint64_t dims[3] = {(cuuint64_t)Cg, (cuuint64_t)taps, (cuuint64_t)O};
  cuuint64_t strides[2] = {(cuuint64_t)Cg * esz, (cuuint64_t)taps * Cg * esz};
  cuuint32_t box[3] = {(cuuint32_t)box_c, 1u, (cuuint32_t)box_o};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = get_encode()(&m, map_type(esz), 3, const_cast<void*>(w), dims, strides,
                            box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("tmpi_native: cuTensorMapEncodeTiled(3D weights) failed, code " + std::to_string((int)r));
  if (cache.size() > 4096) cache.clear();
  cache[key] = m;
  return m;
}

// y[N*Ho*Wo, O] (ld = ldc) = relu(conv(x[.., c_off:c_off+Cg], w[O][KH][KW][Cg]) + bias)   — no col matrix in memory
// dgrad = 1: the same kernel computes the input gradient — x is dy, (Cg, O) are (#dy channels, #dx channels) and w is the
// FORWARD filter [Cg][KH][KW][O], read mirrored and transposed by the TMA loads (stride-1 convolutions only).
// ngroups = 2: both groups of a grouped convolution in ONE persistent launch (group g reads channel slice c_off[g] of x,
// filter w[g], writes y[g] / adds bias[g]) — their tiles fill the machine together instead of two under-filled waves.
template <typename T>
static void conv_fprop_groups(int ngroups, const void* x, const int* c_off, const void* const* w, void* const* y, const float* const* bias,
                              int N, int H, int W, int Ctot, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldc,
                              int relu, int out_bf16, int dgrad, cudaStream_t st) {
  using E = Elem<T>;
  constexpr int BK = E::BK, ATOM = E::ATOM, ESZ = E::ESZ;
  const long long M = (long long)N * Ho * Wo;
  if (M <= 0 || O <= 0) return;
  if (M >= (1LL << 31)) throw std::runtime_error("conv_fprop: too many output pixels");
  if (ESZ == 4) out_bf16 = 0;
  const int c_chunks = (Cg + BK - 1) / BK, num_kb = KH * KW * c_chunks;
  // tall tiles: bf16 outputs; on the tf32 path K-major operands only (dgrad's weights are MN-major)
  const ConvTile tile = choose_conv_tile(dgrad ? 1 : 0, M, O, ngroups, num_kb, ESZ == 2 ? out_bf16 : !dgrad, sm_count());
  const int BN = tile.bn;
  const bool tall = tile.mt == 2;
  Params p;
  p.C = y[0]; p.bias = bias[0]; p.alpha = 1.f; p.M = (int)M; p.N = O; p.K = KH * KW * Cg; p.ldc = ldc; p.a_mn = 0; p.b_mn = dgrad ? 1 : 0;
  p.groups = ngroups; p.C1 = ngroups > 1 ? y[1] : nullptr; p.bias1 = ngroups > 1 ? bias[1] : nullptr;
  p.out_bf16 = out_bf16; p.bias_mode = bias[0] ? 1 : 0; p.relu = relu; p.atomic_out = 0;
  if (ngroups > 1 && ((bias[0] == nullptr) != (bias[1] == nullptr))) throw std::runtime_error("conv_fprop: both groups need a bias or none");
  if (dgrad && (S != 1 || ((O * ESZ) % 16) != 0)) throw std::runtime_error("conv dgrad through the fprop kernel needs stride 1 and 16-byte channel rows");
  p.nt = (O + BN - 1) / BN; p.splits = 1;
  p.mt = tall ? (int)((M + 2 * BM - 1) / (2 * BM)) : (int)((M + BM - 1) / BM);
  p.group_m = 0;
  p.conv_mode = 1; p.cHo = Ho; p.cWo = Wo; p.cS = S; p.cP = P; p.cKH = KH; p.cKW = KW; p.cCg = Cg; p.c_chunks = c_chunks;
  p.num_kb = num_kb; p.kb_per_split = p.num_kb;
  CUtensorMap ta[2], tb[2];
  for (int g = 0; g < ngroups; ++g) {
    ta[g] = make_im2col_map(x, N, H, W, Ctot, c_off[g], Cg, KH, KW, S, P, BM, ESZ, 0);                     // K-major (channels = K)
    tb[g] = dgrad ? make_weight_map(w[g], Cg, KH * KW, O, BK, ATOM, ESZ, 1) : make_weight_map(w[g], O, KH * KW, Cg, BN, BK, ESZ, 0);
  }
  const CUtensorMap* a1 = ngroups > 1 ? &ta[1] : nullptr;
  const CUtensorMap* b1 = ngroups > 1 ? &tb[1] : nullptr;
  if (tall) {
    if (BN == 128) launch<T, 128, 2>(ta[0], tb[0], p, 1, st, a1, b1);
    else if (BN == 96) launch<T, 96, 2>(ta[0], tb[0], p, 1, st, a1, b1);
    else launch<T, 64, 2>(ta[0], tb[0], p, 1, st, a1, b1);
  } else if (BN == 192) launch<T, 192, 1>(ta[0], tb[0], p, 1, st, a1, b1);
  else if (BN == 128) launch<T, 128, 1>(ta[0], tb[0], p, 1, st, a1, b1);
  else if (BN == 96) launch<T, 96, 1>(ta[0], tb[0], p, 1, st, a1, b1);
  else launch<T, 64, 1>(ta[0], tb[0], p, 1, st, a1, b1);
}

// dw[O][KH*KW][Cg] (fp32, contiguous) = sum over pixels dy[pix, o] * im2col(x)[pix, (tap, c)]   (dy: [M, O], row pitch ldy)
// ngroups = 2: both groups in one launch (dy[g] = the group's channel slice of the output gradient, x slice c_off[g], dw[g]).
// accumulate = 1: dw += ... through the epilogue's fp32 reductions, without the split-K clear.
template <typename T>
static void conv_wgrad_groups(int ngroups, const void* const* dy, const void* x, void* const* dw, const int* c_off, int N, int H, int W,
                              int Ctot, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldy, int accumulate,
                              cudaStream_t st) {
  using E = Elem<T>;
  constexpr int BK = E::BK, ATOM = E::ATOM, ESZ = E::ESZ;
  const long long M = (long long)N * Ho * Wo;
  if (M <= 0 || O <= 0) return;
  if (M >= (1LL << 31)) throw std::runtime_error("conv_wgrad: too many output pixels");
  const int c_chunks = (Cg + ATOM - 1) / ATOM, num_kb = (int)((M + BK - 1) / BK);
  // BN / ATOM (tap, channel-chunk) boxes per n-tile: wider tiles re-read dy fewer times
  const ConvTile tile = choose_conv_tile(2, O, KH * KW * c_chunks * ATOM, ngroups, num_kb, 0, sm_count());
  const int BN = tile.bn;
  Params p;
  p.C = dw[0]; p.bias = nullptr; p.alpha = 1.f; p.M = O; p.N = KH * KW * Cg; p.K = (int)M; p.ldc = (long long)KH * KW * Cg; p.a_mn = 1; p.b_mn = 1;
  p.groups = ngroups; p.C1 = ngroups > 1 ? dw[1] : nullptr; p.bias1 = nullptr;
  p.out_bf16 = 0; p.bias_mode = 0; p.relu = 0;
  p.group_m = 0;
  p.conv_mode = 2; p.cHo = Ho; p.cWo = Wo; p.cS = S; p.cP = P; p.cKH = KH; p.cKW = KW; p.cCg = Cg; p.c_chunks = c_chunks;
  p.mt = (O + BM - 1) / BM; p.nt = (KH * KW * p.c_chunks + BN / ATOM - 1) / (BN / ATOM);
  p.num_kb = num_kb;
  const int splits = tile.splits;
  p.kb_per_split = (p.num_kb + splits - 1) / splits;
  p.splits = splits; p.atomic_out = splits > 1 || accumulate;
  CUtensorMap ta[2], tb[2];
  for (int g = 0; g < ngroups; ++g) {
    if (splits > 1 && !accumulate) check_cuda(cudaMemsetAsync(dw[g], 0, (size_t)O * KH * KW * Cg * 4, st), "conv_wgrad memset");
    ta[g] = make_tmap(dy[g], (uint64_t)O, (uint64_t)M, (uint64_t)ldy * ESZ, (uint32_t)BK, ESZ, 1);          // both operands MN-major
    tb[g] = make_im2col_map(x, N, H, W, Ctot, c_off[g], Cg, KH, KW, S, P, BK, ESZ, 1);
  }
  const CUtensorMap* a1 = ngroups > 1 ? &ta[1] : nullptr;
  const CUtensorMap* b1 = ngroups > 1 ? &tb[1] : nullptr;
  if (BN == 192) launch<T, 192, 1>(ta[0], tb[0], p, splits, st, a1, b1);
  else launch<T, 128, 1>(ta[0], tb[0], p, splits, st, a1, b1);
}
}  // namespace wgmma

// the output has the activation dtype: bf16, or fp32 on the tf32 path
void conv_fprop(const void* x, const void* w, void* y, const float* bias, int N, int H, int W, int Ctot, int c_off, int Cg, int KH,
                int KW, int Ho, int Wo, int S, int P, int O, long long ldc, int relu, int dgrad, int f32, cudaStream_t st) {
  const void* ws[1] = {w}; void* ys[1] = {y}; const float* bs[1] = {bias};
  if (f32) wgmma::conv_fprop_groups<float>(1, x, &c_off, ws, ys, bs, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldc, relu, 0, dgrad, st);
  else wgmma::conv_fprop_groups<__nv_bfloat16>(1, x, &c_off, ws, ys, bs, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldc, relu, 1, dgrad, st);
}

void conv_fprop2(const void* x, const void* w0, const void* w1, void* y0, void* y1, const float* bias0, const float* bias1, int N, int H,
                 int W, int Ctot, int c_off0, int c_off1, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldc,
                 int relu, int dgrad, int f32, cudaStream_t st) {
  const int co[2] = {c_off0, c_off1}; const void* ws[2] = {w0, w1}; void* ys[2] = {y0, y1}; const float* bs[2] = {bias0, bias1};
  if (f32) wgmma::conv_fprop_groups<float>(2, x, co, ws, ys, bs, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldc, relu, 0, dgrad, st);
  else wgmma::conv_fprop_groups<__nv_bfloat16>(2, x, co, ws, ys, bs, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldc, relu, 1, dgrad, st);
}

void conv_wgrad(const void* dy, const void* x, void* dw, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho,
                int Wo, int S, int P, int O, long long ldy, int accumulate, int f32, cudaStream_t st) {
  const void* dys[1] = {dy}; void* dws[1] = {dw};
  if (f32) wgmma::conv_wgrad_groups<float>(1, dys, x, dws, &c_off, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldy, accumulate, st);
  else wgmma::conv_wgrad_groups<__nv_bfloat16>(1, dys, x, dws, &c_off, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldy, accumulate, st);
}

void conv_wgrad2(const void* dy0, const void* dy1, const void* x, void* dw0, void* dw1, int N, int H, int W, int Ctot, int c_off0,
                 int c_off1, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldy, int accumulate, int f32,
                 cudaStream_t st) {
  const void* dys[2] = {dy0, dy1}; void* dws[2] = {dw0, dw1}; const int co[2] = {c_off0, c_off1};
  if (f32) wgmma::conv_wgrad_groups<float>(2, dys, x, dws, co, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldy, accumulate, st);
  else wgmma::conv_wgrad_groups<__nv_bfloat16>(2, dys, x, dws, co, N, H, W, Ctot, Cg, KH, KW, Ho, Wo, S, P, O, ldy, accumulate, st);
}

}  // namespace tmpi
