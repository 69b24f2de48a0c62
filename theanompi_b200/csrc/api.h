// Host-visible API of the sm_90a extension (implemented in the .cu / .cpp files of this directory).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <tuple>
#include "common.cuh"

namespace tmpi {

constexpr int kMaxRanks = 8;
constexpr int kMaxCommBlocks = 1024;     // signal-pad rows

struct CommCtx {
  void* arena[kMaxRanks];                // base of rank p's arena as mapped in THIS process
  uint32_t* sig[kMaxRanks];              // signal pad of rank p: uint32 [kMaxCommBlocks][kMaxRanks]
  uint32_t* epoch;                       // local: per-block barrier epoch counters [kMaxCommBlocks]
  void* mc_arena;                        // multicast mapping of the arena (NVLS) or nullptr
  int rank, world;
  long long spin_limit;                  // clock64 cycles a flag barrier may spin before it traps (TMPI_BARRIER_TIMEOUT_S)
};

struct FusedArgs {
  CommCtx ctx;
  long long w_off, g_off, u_off, h_off, wire_off;   // byte offsets of the regions inside the arena (h_off < 0: no shadow)
  const uint8_t* block_group;
  GroupTable tab;
  const float* lr_ptr;                               // device scalar (CUDA-graph friendly)
  float mu;
  int nesterov;
  float inv_k;
  long long lo, hi;                                  // element range, multiples of kArenaBlock
  int wire16;                                        // gradients travel as bf16 (cast into the wire region first)
  int pre_reduced;                                   // the range's gradients were already reduce-scattered into their owner's G by the
                                                     // wgrad GEMM epilogues (gemm_rs_*): skip the gather, zero G after use
  int push_master = 1;                               // two-shot: 1 = push the updated fp32 master slice AND the bf16 shadow to every peer;
                                                     // 0 = owner keeps the master of WEIGHT blocks (group 0): peers receive only their bf16
                                                     // compute shadow — a third of the all-gather bytes; bias blocks (read in fp32 by the
                                                     // forward pass) are always pushed; push_master_slices() re-synchronises W on demand
};

struct ReduceArgs {
  CommCtx ctx;
  long long src_off, dst_off, h_off;     // h_off >= 0: also refresh the bf16 shadow from the result (weight averaging)
  const uint8_t* block_group;
  GroupTable tab;
  float scale;
  long long lo, hi;
  int skip_local_groups;                 // leave non-exchanged blocks untouched
};

// ---- gemm_wgmma.cu
void gemm_set_debug(int flags);
// Reduce-scatter fused into the wgrad GEMM epilogue: register the peer views of the gradient region and the tensors whose
// fp32 GEMM output (C pointer inside [c_lo, c_hi)) must be red.add-ed into the OWNER rank's G instead of stored locally.
// Ownership = the two-shot exchange kernel's partition of the bucket [blo, blo + world * per) in 1024-element blocks.
void gemm_rs_configure(int world, const void* const* peer_g /*[world]*/, const void* local_g);
void gemm_rs_add_range(const void* c_lo, const void* c_hi, long long blo, long long per);
void gemm_rs_clear();
int gemm_plan_splits(int tiles, int num_kb, int sms);          // split-K factor the launcher would pick
int gemm_plan_tall(long long M, int nt, int out_bf16, int sms);   // 1 = 256-row CTA tiles   // bottleneck probe knobs of the wgmma GEMM (see Params::dbg)
// (BN, MT, split-K slices) an implicit-GEMM convolution launch would use.  kind 0 fprop, 1 dgrad, 2 wgrad; fprop / dgrad:
// M = output pixels, N = output channels, num_kb = taps x channel chunks; wgrad: M = output channels, N = (tap, channel-chunk)
// boxes x box width, num_kb = pixel blocks.  tall_ok: the output may use 256-row tiles (bf16 output, or K-major tf32).
std::tuple<int, int, int> gemm_plan_conv(int kind, long long M, int N, int groups, int num_kb, int tall_ok, int sms);
// f32 = 1: fp32 operands through wgmma tf32 (fp32 output), else bf16 operands.  accumulate = 1: C += the product (fp32 output
// without bias / ReLU; gradient accumulation): the epilogue reduces every tile into C and the split-K clear is skipped
void gemm(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, long long lda, long long ldb, long long ldc,
          int a_mn, int b_mn, int out_bf16, int bias_mode, int relu, float alpha, int bn_hint, int splitk, int f32, cudaStream_t st,
          int accumulate = 0);
// FC weight gradient A^T B (A: [K, M], B: [K, N], both MN-major) applied as a momentum-SGD step to W / U [M, N] (fp32, row pitch
// ldw) and the bf16 shadow H (may be null) in the GEMM epilogue, the same arithmetic as flat_update's SGD rule; lr is read from lr_ptr[0]
void gemm_sgd(const void* A, const void* B, void* W, void* U, void* H, const void* lr_ptr, float lr_mult, float wd, float mu, int nesterov,
              float inv_k, int M, int N, int K, long long lda, long long ldb, long long ldw, int f32, cudaStream_t st);

void conv_fprop(const void* x, const void* w, void* y, const float* bias, int N, int H, int W, int Ctot, int c_off, int Cg, int KH,
                int KW, int Ho, int Wo, int S, int P, int O, long long ldc, int relu, int dgrad, int f32, cudaStream_t st);
// accumulate = 1: dw += the weight gradient (gradient accumulation), else dw = it
void conv_wgrad(const void* dy, const void* x, void* dw, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho,
                int Wo, int S, int P, int O, long long ldy, int accumulate, int f32, cudaStream_t st);
// both groups of a 2-group convolution in one persistent launch (see gemm_wgmma.cu)
void conv_fprop2(const void* x, const void* w0, const void* w1, void* y0, void* y1, const float* bias0, const float* bias1, int N, int H,
                 int W, int Ctot, int c_off0, int c_off1, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldc,
                 int relu, int dgrad, int f32, cudaStream_t st);
void conv_wgrad2(const void* dy0, const void* dy1, const void* x, void* dw0, void* dw1, int N, int H, int W, int Ctot, int c_off0,
                 int c_off1, int Cg, int KH, int KW, int Ho, int Wo, int S, int P, int O, long long ldy, int accumulate, int f32,
                 cudaStream_t st);

// ---- nn_kernels.cu  (f32: fp32 activations, C % 4 == 0; else bf16, C % 8 == 0)
void space_to_depth(const void* x, void* y, int N, int H, int W, int C, int S, int Hs, int Ws, int Cp, int P, int f32, cudaStream_t st);
// dir 0: pack a filter for the space-to-depth conv; 1: unpack its fp32 weight gradient (store); 2: unpack and add into dst
void s2d_filter(const void* src, void* dst, int O, int KH, int KW, int C, int S, int KHs, int KWs, int Cp, int dir, int f32, cudaStream_t st);
void lrn_fwd(const void* x, void* y, long long rows, int C, int n, float k, float alpha, float beta, int f32, cudaStream_t st);
void lrn_bwd(const void* x, const void* dy, void* dx, long long rows, int C, int n, float k, float alpha, float beta, int f32, cudaStream_t st);
void pool_fwd(const void* x, void* y, void* arg, int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p, int is_max, int f32,
              cudaStream_t st);
void pool_bwd(const void* dy, const void* arg, void* dx, int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p, int is_max, int f32,
              cudaStream_t st);
void dropout_fwd(const void* x, void* y, void* mask, long long n, float p_drop, unsigned long long seed, int layer, const void* step, int f32,
                 cudaStream_t st);
void dropout_bwd(const void* dy, const void* mask, void* dx, long long n, int f32, cudaStream_t st);
void advance_step(void* step, cudaStream_t st);
// out3 = {weight · mean NLL, top-1 error, top-5 error}; dlogits = (softmax − onehot) · grad_weight / B (grad_weight = weight / n under
// n-micro-batch gradient accumulation, so the accumulated gradient is the mean over the window).  label_smoothing ε in (0, 1]: the
// target is (1 − ε)·onehot + ε / C in both the loss and dlogits (soft-target cross-entropy); ε = 0 is the plain NLL
void softmax_xent(const void* logits, const void* labels, void* dlogits, void* rowstat, void* out3, int B, int C, float weight,
                  float grad_weight, float label_smoothing, int f32, cudaStream_t st);
// Mixup / CutMix (ops/mixup.py owns the same layout on the Python side).  One MixRecord per training step, written by mix_draw on
// the device and read by mix_batch and softmax_xent_mix: sample i is paired with j = B − 1 − i and trains against
// λ·s(y_i) + (1 − λ)·s(y_j), s the (smoothed) one-hot target.
enum MixMode : int { MIX_NONE = 0, MIX_MIXUP = 1, MIX_CUTMIX = 2 };
struct MixRecord {                       // 64 bytes
  int mode;                              // MixMode
  float lam;                             // effective λ: the weight of y_i (1 when mode = MIX_NONE; CutMix: 1 − box area / (H·W))
  double lam_raw;                        // the Beta(α, α) draw (1 when mode = MIX_NONE)
  int cy, cx;                            // CutMix: box centre (0 otherwise)
  int y0, y1, x0, x1;                    // CutMix: the clipped box [y0, y1) × [x0, x1) (0 otherwise)
  int H, W;                              // image size the box refers to
  int pad[4];
};
static_assert(sizeof(MixRecord) == 64, "MixRecord layout is shared with ops/mixup.py");
struct MixParams {
  double alpha, cutmix_alpha;            // Beta(α, α) of Mixup / of CutMix; 0 disables that mode
  double switch_prob, prob;              // P(CutMix | both enabled), P(mix at all)
  unsigned long long seed;
  int rank;
  int H, W;
};
// rec[t] = the draw of step counter value *step + t, t < n (the training step launches n = 1)
void mix_draw(const MixParams& p, const void* step, void* rec, int n, cudaStream_t st);
// in place on the NHWC batch x [B, H, W, C]: Mixup x_i ← λ·x_i + (1 − λ)·x_j (fp32, rounded once), CutMix swaps the box between
// x_i and x_j; MIX_NONE leaves x untouched
void mix_batch(void* x, const void* rec, int B, int H, int W, int C, int f32, cudaStream_t st);
// softmax_xent against the mixed soft target of rec (label j from labels[B − 1 − b]); err1 / err5 count against y_i when λ ≥ ½,
// else y_j
void softmax_xent_mix(const void* logits, const void* labels, const void* rec, void* dlogits, void* rowstat, void* out3, int B, int C,
                      float weight, float grad_weight, float label_smoothing, int f32, cudaStream_t st);
// knowledge distillation: out3 = {mean L, top-1 error, top-5 error} with L = (1 − α)·CE_q(z) + α·T²·KL(softmax(t/T) ‖ softmax(z/T)) per row,
// dlogits = [(1 − α)·(softmax(z) − q) + α·T·(softmax(z/T) − softmax(t/T))] · grad_weight / B; q is the target of softmax_xent
// (label_smoothing ε) or, with a mix record rec (nullptr: none), of softmax_xent_mix.  teacher: the teacher's logits, in the same dtype
void softmax_xent_kd(const void* logits, const void* teacher, const void* labels, const void* rec, void* dlogits, void* rowstat, void* out3,
                     int B, int C, float grad_weight, float label_smoothing, float alpha, float temperature, int f32, cudaStream_t st);
// drop-path table (ops/drop_path.py owns the layout): out[l·B + n] = 0 when block l drops sample n at step counter *step, else
// keep_scale[l] = fp32(1 / (1 − p_l)); thresh[l] = ⌈p_l·2^24⌉ (uint32), key (seed, rank)
void drop_path_draw(const void* thresh, const void* keep_scale, int L, int B, unsigned long long seed, int rank, const void* step, void* out,
                    cudaStream_t st);
// cifar_augment draw (ops/cifar_augment.py owns the layout) of step counter *step, key (seed, rank): offs int32 [B, 2] (oy − pad,
// ox − pad), flips uint8 [B], boxes int32 [B, 4] Cutout (i, j, h, w) of side L in an H × W image (16-byte aligned)
void cifar_augment_draw(int B, int pad, int L, int H, int W, unsigned long long seed, int rank, const void* step, void* offs, void* flips,
                        void* boxes, cudaStream_t st);
// act: 0 none, 1 ReLU, 2 leaky ReLU (negative slope `slope`), 3 sigmoid (ACT_* in common.cuh).  accumulate = 1: db / db1 += the bias
// gradient (no clear)
void relu_bias_bwd(const void* dy, const void* y, void* dym, void* db, void* db1, int c_split, long long R, int C, long long ld, int act,
                   float slope, int accumulate, int f32, cudaStream_t st);
void bias_act(const void* acc, const void* bias, void* y, int R, int C, int act, float slope, int f32, cudaStream_t st);
// transposed-convolution forward: y[N,H,W,C] = act(col2im(dcol) + bias), dcol = x[N*Hi*Wi, Cin] · W[Cin, KH*KW*C] (row pitch ldcol);
// channels >= c_real are written as zeros
void col2im_bias_act(const void* dcol, void* y, const float* bias, int N, int H, int W, int C, int KH, int KW, int Hi, int Wi, int s, int p,
                     long long ldcol, int act, float slope, int c_real, int f32, cudaStream_t st);
void gan_loss(const void* scores, void* dscores, void* out, int B, int kind, float a, int f32, cudaStream_t st);
void uniform_noise(void* out, long long n, unsigned long long seed, int stream, const void* step, int f32, cudaStream_t st);
// bf16 only (packed-bf16 compares).  accumulate = 1: db0 / db1 += the bias gradient (no clear)
void maxpool_relu_bias_bwd(const void* dyp, const void* arg, const void* y, void* dym, void* db0, void* db1, int c_split, int N, int H,
                           int W, int C, int Ho, int Wo, int k, int s, int p, int accumulate, cudaStream_t st);
void im2col(const void* x, void* col, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho, int Wo, int s, int p,
            long long ldcol, int f32, cudaStream_t st);
void col2im(const void* dcol, void* dx, int N, int H, int W, int Ctot, int c_off, int Cg, int KH, int KW, int Ho, int Wo, int s, int p,
            long long ldcol, int f32, cudaStream_t st);
void pad_rows(const void* src, void* dst, long long rows, int cols, long long src_ld, long long dst_ld, int f32, cudaStream_t st);
// zero_fill = 1: offsets may put a source pixel outside the image, which then stores 0 in every channel (else the crop stays inside)
void crop_mirror_norm(const void* x, int in_kind, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16, const void* offs,
                      const void* flips, int N, int H, int W, int C, int ch, int cw, int Cout, int zero_fill, cudaStream_t st);
// test-time views: kMaxViews entries (y0, x0, mirror) of the ch × cw crop inside the H × W image, passed by value
constexpr int kMaxViews = 10;
struct ViewTable {
  int y0[kMaxViews], x0[kMaxViews], mirror[kMaxViews];
};
// the V views of the uint8 NHWC batch x, normalised as crop_mirror_norm, into the view-major out [V, N, ch, cw, C] (bf16 or fp32)
void multi_crop_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                     const ViewTable& views, int V, int N, int H, int W, int C, int ch, int cw, cudaStream_t st);
// view v of V: acc [B, C] fp32 = softmax(logits) (v = 0) or acc + softmax(logits); on v = V − 1 acc /= V, rowstat[b] = {−log max(p̄_y,
// FLT_MIN), top-1 error, top-5 error} and out3 = their means over the batch
void view_softmax_accum(const void* logits, const void* labels, void* acc, void* rowstat, void* out3, int B, int C, int v, int V, int f32,
                        cudaStream_t st);
// random-resized crop: uint8 NHWC x → bilinear resample of the normalised box boxes[n] = (y0, x0, h, w) (int32 [N, 4], 16-byte
// aligned, inside the H × W image) to ch × cw, mirrored after the resize where flips[n]; out bf16 (out_bf16) or fp32 NHWC
void resized_crop_mirror_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                              const void* boxes, const void* flips, int N, int H, int W, int C, int ch, int cw, cudaStream_t st);
// colour jitter + lighting on top of the resized crop (C = 3): out = (M·v̂ + K·μ + ℓ − m̂)·s_c, v̂ / m̂ the bilinear resample of the raw
// box / of the mean; rec = fp32 [N, 24] (M, K, ℓ, 0; 16-byte aligned), mu = fp32 [N, 4] from crop_mean, or null when K ≡ 0
void color_crop_mirror_norm(const void* x, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16,
                            const void* boxes, const void* flips, const void* rec, const void* mu, int N, int H, int W, int ch, int cw,
                            cudaStream_t st);
// mu[n] = mean RGB (fp32 [N, 4], last lane 0) of the ch × cw bilinear resample of the raw uint8 box n (x: [N, H, W, 3])
void crop_mean(const void* x, const void* boxes, void* mu, int N, int H, int W, int ch, int cw, cudaStream_t st);
// auto_augment (C = 3): the uint8 crop u (round-half-to-even of the bilinear resample of the raw box, mirrored; [N, ch, cw, 3]);
// the per-slot point-op LUTs (uint8 [N, 3, 256]) from the ping buffer; one op slot ping → pong; the normalisation (u' − m̂)·s_c.
// rec = fp32 [N, slots, 12], 16-byte aligned
void aa_crop_u8(const void* x, void* u, const void* boxes, const void* flips, int N, int H, int W, int ch, int cw, cudaStream_t st);
void aa_lut(const void* u, const void* rec, void* lut, int slot, int slots, int N, int ch, int cw, cudaStream_t st);
void aa_apply(const void* in, void* out, const void* rec, const void* lut, int slot, int slots, int N, int ch, int cw, int bilinear,
              cudaStream_t st);
void aa_mix(void* u, const void* chains, const void* rec, const void* weights, int width, int N, int ch, int cw, cudaStream_t st);
void aa_normalize(const void* u, const void* mean, int mean_mode, float scale, const void* cscale, void* out, int out_bf16, const void* boxes,
                  const void* flips, int N, int W, int ch, int cw, cudaStream_t st);
// random erasing in place: out (bf16 (out_bf16) or fp32 NHWC [N, ch, cw, C]) is set to 0 inside box n = (i, j, h, w) (int32 [N, 4],
// 16-byte aligned, inside the output; h = w = 0 erases nothing)
void erase_boxes(void* out, int out_bf16, const void* boxes, int N, int ch, int cw, int C, cudaStream_t st);

// ---- bn_kernels.cu: batch norm (+ residual)(+ ReLU) forward / backward, residual add  (f32: fp32 activations, else bf16)
// drop_scale (optional, null = off): one row of the step's drop-path table, a float per sample of the `batch` samples (rows
// r of sample r / (R / batch)); forward y = act(s_n·(γ·x̂ + β) + res) needs res, backward uses s_n·g for dγ, dβ and dx while
// dres = g.  act must be ACT_NONE or ACT_RELU with a row.
void bn_forward(const void* x, const void* res, void* y, const void* gamma, const void* beta, void* mean, void* rstd, void* run_mean,
                void* run_var, void* scratch, long long R, int C, float momentum, float eps, int training, int act, float slope,
                const void* drop_scale, int batch, int f32, cudaStream_t st);
// scratch: 3*C floats, 5*C with accumulate = 1 (dgamma / dbeta += this batch's gradients; dx is computed from this batch's sums, which
// go to the scratch, exactly as without accumulate)
void bn_backward(const void* x, const void* dy, const void* y, void* dx, void* dres, const void* gamma, const void* mean, const void* rstd,
                 void* dgamma, void* dbeta, void* scratch, long long R, int C, int act, float slope, int accumulate, const void* drop_scale,
                 int batch, int f32, cudaStream_t st);
void add_tensors(const void* a, const void* b, void* y, long long n, int f32, cudaStream_t st);
// y = s_n·a + b over `batch` equal samples of n / batch elements (b null: y = s_n·a), s = one row of the drop-path table
void add_scaled(const void* a, const void* b, const void* scale, void* y, long long n, int batch, int f32, cudaStream_t st);
void add4_tensors(const void* a, const void* b, const void* c, const void* d, void* y, long long n, int f32, cudaStream_t st);

// ---- rnn_kernels.cu: LSTM cell fwd / bwd, embedding gather / scatter, masked mean pooling  (f32: fp32 activations, else bf16)
void lstm_cell_fwd(const void* gx, const void* gh, const void* c_prev, const void* h_prev, const void* mask, void* act, void* c_out, void* h_out,
                   int B, int H, int f32, cudaStream_t st);
void lstm_cell_bwd(const void* dh_out, const void* dh_rec, const void* dh_pass_in, const void* dc_next, const void* act, const void* c,
                   const void* c_prev, const void* mask, void* dG, void* dc_prev, void* dh_pass, int B, int H, int f32, cudaStream_t st);
void embedding_fwd(const void* ids, const void* W, void* out, long long n, int D, int f32, cudaStream_t st);
void embedding_bwd(const void* ids, const void* dout, void* dW, long long n, int D, long long V, int f32, cudaStream_t st);
void masked_mean_fwd(const void* h, const void* mask, void* out, int Tn, int B, int H, int f32, cudaStream_t st);
void masked_mean_bwd(const void* dout, const void* mask, void* dh, int Tn, int B, int H, int f32, cudaStream_t st);

// ---- comm_kernels.cu
// One step of a local flat optimizer over the arena elements [lo, hi) (multiples of kArenaBlock): one launch, two for Adam (its
// step counter advances after the update).  lr is read from lr_ptr[0] on the device.
//   rule                   S (the rule's state; the arena's U region first)   hp (float hyperparameters)
//   FLAT_SGD               U                                                   mu, nesterov (0 / 1), inv_k
//   FLAT_ADAM              M (U), V                                            b1, b2, eps           (+ step)
//   FLAT_RMSPROP           V                                                   alpha, eps, clip
//   FLAT_ADADELTA          U, V                                                rho, eps
//   FLAT_RMSPROP_CENTERED  M (U), R, S                                         rho, mu, eps
//   FLAT_LARS              U                                                   mu, nesterov (0 / 1), inv_k   (+ block_tensor, tensor_scale)
//   FLAT_LAMB              M (U), V (read only: lamb_trust advanced them)      b1, b2, eps           (+ step, block_tensor, tensor_scale)
// clip (the first five rules): the ClipRecord grad_clip_norm wrote for this step.  The step then uses s·g; when the norm is not finite
// it changes nothing, Adam's counter included.
enum FlatRuleId : int { FLAT_SGD = 0, FLAT_ADAM, FLAT_RMSPROP, FLAT_ADADELTA, FLAT_RMSPROP_CENTERED, FLAT_LARS, FLAT_LAMB };
// device record of one gradient-norm clipping step (16 bytes)
struct ClipRecord {
  float norm;                            // ‖g‖ over the real elements, before clipping
  float scale;                           // s = min(1, max_norm / (norm + 1e-6)); 0 when the step is skipped
  int finite;                            // 0: the norm is NaN or Inf and the step is skipped
  int pad;
};
struct FlatUpdateArgs {
  int rule;
  void* W;
  const void* G;
  void* S[3];
  void* H;                               // bf16 shadow of W, or null
  const void* block_group;
  GroupTable tab;
  const void* lr_ptr;
  void* step;                            // Adam, LAMB: device step counter (uint64; LAMB: not advanced by a filter-1 pass), else null
  const float* hp;
  int n_hp;
  long long lo, hi;
  int filter;                            // SGD, LARS, LAMB: 0 all groups, 1 only non-exchanged groups, 2 only exchanged groups
  const void* block_tensor;              // LARS, LAMB: tensor index of every arena block (int32), else null
  const void* tensor_scale;              // LARS, LAMB: trust ratio of every tensor (fp32, from lars_trust / lamb_trust), else null
  const void* clip;                      // gradient-norm clipping: the step's ClipRecord, else null
};
void flat_update(const FlatUpdateArgs& a, cudaStream_t st);
// Global gradient-norm clipping over the whole arena, two launches: per-block Σg² over the real elements of G into partial ([n_blocks]
// fp32), then one CTA sums them in fp64 in a fixed order and writes *rec; when the norm is not finite it adds 1 to *skipped (uint64).
// G is not changed: the clip pointer of the flat_update pass that follows applies s.
struct GradClipArgs {
  const void* G;
  const void* block_tensor;
  const void* tensor_span;
  long long n_blocks;
  float max_norm;
  void* partial;
  void* rec;
  void* skipped;
};
void grad_clip_norm(const GradClipArgs& a, cudaStream_t st);
// LARS trust ratios over the whole arena, two launches: per-block sums of squares of W and G into partial ([n_blocks, 2] fp32),
// then one CTA per tensor: norms[t] = {‖W‖, ‖G‖·inv_k} ([n_tensors, 2] fp32) and trust[t] = eta·‖W‖ / (‖g‖ + wd·‖W‖) for the
// weight group (group 0) when both norms are positive, else 1.  tensor_span: [n_tensors, 2] int64 {element offset, size}.
struct LarsTrustArgs {
  const void* W;
  const void* G;
  const void* block_tensor;
  const void* tensor_span;
  const void* block_group;
  GroupTable tab;
  float inv_k, eta;
  long long n_blocks;
  int n_tensors;
  void* partial;
  void* norms;
  void* trust;
};
void lars_trust(const LarsTrustArgs& a, cudaStream_t st);
// LAMB passes 1 and 2 over the blocks whose group `filter` keeps (as in flat_update), two launches: with g = G·inv_k and t = *step + 1,
// advance M (the arena's U) and V in place and write the per-block sums of squares of W and of the update direction
// r = (M·c1) / (sqrt(V·c2) + eps) + wd·W into partial; then norms[t] = {‖W‖, ‖r‖} and trust[t] = ‖W‖ / ‖r‖ for the weight group
// when both norms are positive, else 1.  Neither W, G nor the counter changes: the FLAT_LAMB flat_update pass follows.
struct LambTrustArgs {
  const void* W;
  const void* G;
  void* M;
  void* V;
  const void* step;
  float b1, b2, eps, inv_k;
  int filter;
  const void* block_tensor;
  const void* tensor_span;
  const void* block_group;
  GroupTable tab;
  long long n_blocks;
  int n_tensors;
  void* partial;
  void* norms;
  void* trust;
};
void lamb_trust(const LambTrustArgs& a, cudaStream_t st);
// Per-update learning-rate schedule, one single-thread launch: with u = *counter (uint64), write lr(u) to *lr (fp32, the arena's
// hyper[0]) and u + 1 to *counter.  Warm-up for u < warmup: peak·(start + (1 − start)·u / warmup); after it, with
// q = clamp((u − warmup) / (total − warmup), 0, 1): constant peak, cosine final + (peak − final)·½(1 + cos πq), poly
// final + (peak − final)·(1 − q)^power, or multistep peak·gamma^(number of milestones ≤ u).  fp64, rounded once to fp32.
enum LrPolicy : int { LR_CONSTANT = 0, LR_COSINE, LR_POLY, LR_MULTISTEP };
constexpr int kMaxLrMilestones = 8;
struct LrScheduleParams {
  int policy;
  int n_milestones;
  long long warmup, total;
  double start, peak, final_lr, power, gamma;
  long long milestones[kMaxLrMilestones];
};
void lr_schedule(const LrScheduleParams& p, void* counter, void* lr, cudaStream_t st);
void fused_allreduce_sgd(const FusedArgs& a, int algo, int max_blocks, cudaStream_t st);
// every rank pushes the fp32 master weights of the slice it owns in the two-shot partition of [lo, hi) to all peers
void push_master_slices(const FusedArgs& a, int max_blocks, cudaStream_t st);
void allreduce_flat(const ReduceArgs& a, int algo, int max_blocks, cudaStream_t st);
void device_barrier(const CommCtx& c, cudaStream_t st);
void easgd_elastic(void* w, void* h, void* center, float alpha, long long n, int max_blocks, int lockfree, cudaStream_t st);
// device-side ticket lock in rank `owner`'s signal pad (EASGD: the center); local_state = >= 1 uint32 of local device memory
void ticket_acquire(const CommCtx& c, int owner, void* local_state, cudaStream_t st);
void ticket_release(const CommCtx& c, int owner, void* local_state, cudaStream_t st);
void copy_flat(void* dst, void* dst_h, const void* src, long long n, int max_blocks, const void* gate, cudaStream_t st);
// Model EMA (utils/opt.py: ModelEma).  state: uint64 {u, n_averaged, mode} in device memory.  ema_advance (one thread): u += 1; when
// u % every == 0 the mode is EMA_COPY (n_averaged = 1) if n_averaged == 0 or u <= warmup, else EMA_AVERAGE (n_averaged += 1);
// otherwise EMA_SKIP.  ema_update: per the mode, nothing, E ← W, or E ← fp32(d)·E + fp32(1 − d)·W (each product and the sum rounded
// once) over the n arena elements and every segment (dst = the E part, src = a batch-norm statistics tensor).  ema_swap: W ↔ E,
// H ← bf16-RN(new W) when H is not null, and dst ↔ src of every segment.
enum EmaMode : int { EMA_SKIP = 0, EMA_COPY = 1, EMA_AVERAGE = 2 };
struct EmaSegment {
  float* dst;
  float* src;
  long long n;
};
struct EmaArgs {
  void* W;
  void* E;
  void* H;                               // ema_swap: bf16 shadow of W, or null
  long long n;                           // arena elements (a multiple of kArenaBlock)
  const void* segs;                      // EmaSegment[n_segs] in device memory
  int n_segs;
  const void* state;                     // ema_update: the state words
  float decay, one_minus_decay;
};
void ema_advance(void* state, long long every, long long warmup, cudaStream_t st);
void ema_update(const EmaArgs& a, cudaStream_t st);
void ema_swap(const EmaArgs& a, cudaStream_t st);
// Sharpness-aware minimization (utils/opt.py: Sam), over the n_blocks arena blocks.  sam_norm, two launches: per-block Σg² (SAM) or
// Σ(w·g)² (adaptive, ASAM) over the real elements into partial ([n_blocks] fp32), then one CTA sums them in fp64 in a fixed order and
// writes the ClipRecord *rec: n = ‖g‖ or ‖|w|⊙g‖ rounded to fp32, s = fp32(1 / (n + 1e-12)) · rho, finite.  sam_perturb, one launch:
// P ← W; if finite, W ← W + e on the real elements with e = g·s or ((w·w)·g)·s, H ← bf16(W).  sam_restore, one launch: W ← P,
// H ← bf16(P).  H may be null (no bf16 shadow).
struct SamArgs {
  void* W;
  const void* G;
  void* P;
  void* H;
  const void* block_tensor;
  const void* tensor_span;
  long long n_blocks;
  float rho;
  int adaptive;
  void* partial;
  void* rec;
};
void sam_norm(const SamArgs& a, cudaStream_t st);
void sam_perturb(const SamArgs& a, cudaStream_t st);
void sam_restore(const SamArgs& a, cudaStream_t st);
// device-side gossip (GOSGD): state = 64 uint32 of local device memory, [0] holds the push-sum weight (float)
void gosgd_push(const CommCtx& c, void* state, int dest, long long w_off, long long snap_off, long long n, int max_blocks, cudaStream_t st);
void gosgd_poll_merge(const CommCtx& c, void* state, long long w_off, long long h_off, long long snap_off, long long n, int max_blocks,
                      cudaStream_t st);
void gosgd_merge(void* w, void* h, const void* b, float a_self, float a_src, long long n, int max_blocks, cudaStream_t st);
void cast_flat(const void* src, void* dst, long long n, int kind, cudaStream_t st);
void sum_chunks(const void* src, void* dst, long long chunk, int nchunks, int is_half, cudaStream_t st);
void vecadd(void* cur, const void* tmp, long long n, int is_half, cudaStream_t st);

}  // namespace tmpi
