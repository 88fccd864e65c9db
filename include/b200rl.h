/* b200rl — C-ABI of the H100 (sm_90a) kernels behind SheepRL's Dreamer-V3 / PPO / SAC update paths.
 *
 * The reference (Eclectic-Sheep/sheeprl) is pure Python and has NO native interface for this path
 * (SURVEY.md §0 F1, §2.2); these entry points are what a reference-side binding (ctypes / a
 * torch.utils.cpp_extension shim, see INTEGRATION.md) calls from `sheeprl.algos.<algo>.train()`.
 * Each declaration cites the reference code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer owned by the caller (borrowed);
 *     nothing is allocated or freed by the library but its split-K and deterministic-mode partials pools (grown
 *     outside stream capture only); no host synchronisation; all work is enqueued on
 *     `stream` (pass the caller's current stream) — hence CUDA-graph capturable;
 *   - fp32, row-major; `ld*` = row stride in elements of a 2-D view whose inner stride is 1;
 *   - return 0 on success; non-zero => b200rl_last_error() (thread-local message);
 *   - built for sm_90a only (b200rl_device_check refuses other devices). There is no CPU fallback.
 */
#ifndef B200RL_H_
#define B200RL_H_

#include <cuda_runtime_api.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* b200rl_last_error(void);
int b200rl_abi_version(void);
const char* b200rl_build_arch(void);
int b200rl_device_check(void);

/* ---- dense layers ------------------------------------------------------------------------------
 * nn.Linear forward/backward everywhere in sheeprl/models/models.py:16-119 (MLP), agent.py:281-341
 * (RecurrentModel), agent.py:1021-1051 (representation / transition).  C[M,N] = op(A) op(B) (+bias) (+C).
 * A is [M,K] (lda) or [K,M] if transA; B is [K,N] (ldb) or [N,K] if transB (nn.Linear weight layout).  K = 0 gives
 * C = bias (or 0), or C += bias when accumulating.  The FFMA routes (every tile config, split-K, the rank-K kernel, K = 0)
 * are checked against a float64 reference (tests/test_gpu_simt_precision.py). */
int b200rl_gemm_f32(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda, int ldb,
                    int ldc, int transA, int transB, int accumulate, cudaStream_t stream);
/* Tensor-core path used by b200rl_gemm_f32 for large NT products (transA = 0, transB = 1, 16-byte aligned
 * operands): 3xTF32 split-precision on wgmma.mma_async with TMA-fed 128B-swizzled tiles and register accumulators
 * (gemm_tc.cu).  Same contract as b200rl_gemm_f32; `_supported` tells whether a shape is eligible. */
/* Precision of every tensor-core product (GEMM, conv forward / input gradient / weight gradient), process-wide like
 * torch.set_float32_matmul_precision (the reference sets it from configs/config.yaml:18, default "high"):
 * 3 = three TF32 products per k-step on x = hi + lo (fp32-accurate, default; the 1e-4 parity tests run this),
 * 1 = one TF32 product ("high": the numerics of the reference's own GPU runs, ~3x the throughput).
 * Every tensor-core route (GEMM layouts, split-K, gemm_ln, conv down / up, both weight-gradient routes) is checked in
 * both precisions against a float64 reference (tests/test_gpu_tc_precision.py). */
int b200rl_set_matmul_precision(int tf32_passes);
int b200rl_get_matmul_precision(void);
/* Deterministic mode, process-wide like torch.use_deterministic_algorithms (0 = off, the default; 1 = on).  When on,
 * every reduction that otherwise adds float partials with atomics (sumsq, col_sum, the LayerNorm parameter gradients,
 * the SIMT and batched split-K products, the convolution weight gradients) writes one partial per CTA or warp to a slot
 * and adds the slots in a fixed order: the same inputs give bit-identical outputs on the same GPU type.  The slots live
 * in a library-owned pool, per device, that grows outside stream capture (run a step eagerly before capturing it); no
 * launch reads what the pool held before. */
int b200rl_set_deterministic(int on);
int b200rl_get_deterministic(void);
/* fills the current device's deterministic-mode pool with `byte` (0xFF: NaN in every float and double slot), so a
 * test can show that no deterministic launch reads a slot it has not written; no-op before the pool exists */
int b200rl_deterministic_pool_fill(int byte, cudaStream_t stream);
int b200rl_gemm_tc_supported(const float* A, const float* B, int M, int N, int K, int lda, int ldb, int transA,
                             int transB);
int b200rl_gemm_tc(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda, int ldb,
                   int ldc, int transA, int transB, int accumulate, cudaStream_t stream);
/* Weight operands split once, before the products that read them: X = hi + lo exactly, hi = X with the 13 low mantissa
 * bits cleared (what the TF32 datapath keeps), lo = X - hi.  b200rl_tf32_split: elementwise over n floats.
 * b200rl_tf32_split_t: W [rows][cols] (ldw) -> hi^T, lo^T [cols][ldt], columns [rows, ldt) zeroed (ldt a multiple of 4 so
 * that TMA can address the rows). */
int b200rl_tf32_split(const float* X, float* Xhi, float* Xlo, long long n, cudaStream_t stream);
int b200rl_tf32_split_t(const float* W, float* Thi, float* Tlo, int rows, int cols, long long ldw, long long ldt,
                        cudaStream_t stream);
/* C = A B^T (+bias) (+C) with B [N][K] given as its TF32 planes (row stride ldb each): the kernel loads them straight into
 * its operand stages instead of splitting B per tile.  Bit-identical to b200rl_gemm_tc(transA = 0, transB = 1) on
 * B = Bhi + Blo. */
int b200rl_gemm_tc_presplit_supported(const float* A, const float* Bhi, const float* Blo, int M, int N, int K, int lda,
                                      int ldb);
int b200rl_gemm_tc_presplit(const float* A, const float* Bhi, const float* Blo, float* C, const float* bias, int M, int N,
                            int K, int lda, int ldb, int ldc, int accumulate, cudaStream_t stream);
/* Dense block Linear(bias=False) -> LayerNorm(eps) -> activation in two launches (sheeprl/utils/model.py:34-88 miniblock,
 * as built by MLP at sheeprl/models/models.py:23-119): the wgmma product leaves split-K partial tiles, one kernel sums
 * them in split order, normalises the row in registers and applies the activation.  `pre` (optional) keeps W.x for the
 * backward.  mode 1 (N = 3R): the tail is LayerNormGRUCell's gate instead (sheeprl/models/models.py:396-403): h_out (and
 * h_out2, optional second copy, e.g. the next step's [h | x] input) = u * tanh(r * c) + (1 - u) * h_prev; `out` (optional)
 * keeps LN(W.x).  A [M, K] (lda), W [N, K] (ldw): y = A W^T.  `_supported`: 16-byte aligned NT operands, N % 4 == 0,
 * N <= 1536 (mode 1: N % 384 == 0). */
int b200rl_gemm_ln_supported(const float* A, const float* W, int M, int N, int K, int lda, int ldw, int mode);
int b200rl_gemm_ln(const float* A, const float* W, int M, int N, int K, int lda, int ldw, const float* gamma,
                   const float* beta, float eps, int act, float* pre, long long ldpre, float* out, long long ldout,
                   int mode, const float* h_prev, long long ldh, float* h_out, long long ldho, float* h_out2,
                   long long ldho2, cudaStream_t stream);
/* The same with W given as its TF32 planes (b200rl_tf32_split); bit-identical to b200rl_gemm_ln on W = Whi + Wlo. */
int b200rl_gemm_ln_presplit_supported(const float* A, const float* Whi, const float* Wlo, int M, int N, int K, int lda,
                                      int ldw, int mode);
int b200rl_gemm_ln_presplit(const float* A, const float* Whi, const float* Wlo, int M, int N, int K, int lda, int ldw,
                            const float* gamma, const float* beta, float eps, int act, float* pre, long long ldpre,
                            float* out, long long ldout, int mode, const float* h_prev, long long ldh, float* h_out,
                            long long ldho, float* h_out2, long long ldho2, cudaStream_t stream);
/* nn.LayerNorm(eps) (+ nn.SiLU): miniblock sheeprl/utils/model.py:34-88; LayerNormChannelLast
 * sheeprl/models/models.py:507-518 (channel-last is native here).  act: 0 none, 1 SiLU, 2 tanh, 3 ReLU (the last two:
 * PPO MLPs with layer_norm=True, sheeprl/algos/ppo/agent.py:58-66,152-176).
 * `_route` is the kernel both launches pick for C channels, row strides ld0..ld2 and row bases p0..p2 (forward: X, Y,
 * ld2 = 0, p2 = NULL; backward: X, dY, dX), from the values alone: 0 the warp-per-row kernels (any C; the backward
 * refuses C > 28000), 1 the register-resident rows (C in {32, 48, 64, 96, 128, 192, 256, 384, 512, 640, 768, 1024,
 * 1536}), 2 one CTA per row (C % 4 == 0, 1536 < C <= 16384); 1 and 2 need row strides that are multiples of 4 floats
 * and 16-byte aligned p0..p2, gamma and beta. */
int b200rl_ln_act_route(int C, long long ld0, long long ld1, long long ld2, const float* p0, const float* p1,
                        const float* p2, const float* gamma, const float* beta);
int b200rl_ln_act_fwd(const float* X, const float* gamma, const float* beta, float* Y, long long M, int C,
                      long long ldx, long long ldy, float eps, int act, cudaStream_t stream);
int b200rl_ln_act_bwd(const float* X, const float* gamma, const float* beta, const float* dY, float* dX, float* dgamma,
                      float* dbeta, long long M, int C, long long ldx, long long lddy, long long lddx, float eps,
                      int act, int accumulate, cudaStream_t stream);
int b200rl_col_sum(const float* X, float* out, long long M, int C, long long ldx, int accumulate, cudaStream_t stream);

/* ---- image encoder / decoder ---------------------------------------------------------------------
 * CNNEncoder agent.py:42-97 (Conv2d k4 s2 p1), CNNDecoder agent.py:154-226 (ConvTranspose2d k4 s2 p1),
 * observation normalisation dreamer_v3.py:98.  Images are NHWC; W is [C_small, C_big, 4, 4] (the
 * reference layouts of both layer kinds).  (h, w) = SMALL image size; big image is (2h, 2w). */
int b200rl_obs_prep(const void* obs_nchw, int is_uint8, float* out_nhwc, long long NB, int C, int HW,
                    cudaStream_t stream);
int b200rl_transpose_batched(const float* X, float* Y, int NB, int a, int b, cudaStream_t stream);
/* Y[j][i] = X[i][j] for a strided [rows][cols] view (used to present K-major operands to the tensor-core GEMM:
 * W^T for input gradients, dY^T / X^T for weight gradients). */
int b200rl_transpose2d(const float* X, float* Y, int rows, int cols, long long ldx, long long ldy, cudaStream_t stream);
int b200rl_conv_down(const float* big, const float* W, float* small_, int NB, int h, int w, int Cs, int Cb,
                     cudaStream_t stream);
int b200rl_conv_up(const float* small_, const float* W, float* big, const float* bias, int NB, int h, int w, int Cs,
                   int Cb, cudaStream_t stream);
int b200rl_conv_wgrad(const float* small_, const float* big, float* dW, int NB, int h, int w, int Cs, int Cb,
                      int accumulate, cudaStream_t stream);
/* Whether b200rl_conv_down / _up / _wgrad take their thin-channel kernels (conv_thin.cu: 1..4-channel big images, the
 * RGB ends of the encoder / decoder) rather than the generic implicit GEMM.  These SIMT routes and the generic ones are
 * checked against a float64 reference (tests/test_gpu_simt_precision.py). */
int b200rl_thin_down_supported(int w, int Cs, int Cb);
int b200rl_thin_up_supported(int Cs, int Cb);
int b200rl_thin_wgrad_supported(int Cs, int Cb);
/* Tensor-core implicit-GEMM versions of conv_down / conv_up (gemm_tc.cu: 4-D TMA boxes gather the taps, no
 * im2col buffer, 3xTF32 wgmma).  `Wpacked` is a caller-owned 16*Cs*Cb-float workspace filled by
 * b200rl_conv_pack (down: [Cs][tap][Cb]; up: [parity][Cb][tap][Cs]) after every weight update.  Eligible when the
 * gathered image has a multiple of 32 channels and the small grid tiles by 128 pixels (`_supported`). */
/* Weight gradient as one tensor-core GEMM over all pixels: small^T [Cs][P] times the transposed im2col of `big`
 * [16*Cb][P] (both K-major, split-K).  `workspace`: b200rl_conv_wgrad_tc_workspace(...) floats, caller-owned.
 * `_supported`: 1 for the shapes the launch runs, P = NB*h*w pixels in [1024, 2e9], Cs >= 48, Cb >= 8; b200rl_conv_wgrad
 * runs every shape. */
int b200rl_conv_wgrad_tc_supported(int NB, int h, int w, int Cs, int Cb);
long long b200rl_conv_wgrad_tc_workspace(int NB, int h, int w, int Cs, int Cb);
int b200rl_conv_wgrad_tc(const float* small_, const float* big, float* dW, float* workspace, int NB, int h, int w,
                         int Cs, int Cb, int accumulate, cudaStream_t stream);
int b200rl_conv_tc_supported(int mode_up, int NB, int h, int w, int Cs, int Cb);
/* floats of workspace b200rl_conv_pack writes (16*Cs*Cb; 36*Cs*Cb for ConvTranspose2d layers with 32 output channels, whose
 * four output-parity classes are computed as one 128-column tile over the 9 shifted input windows) */
long long b200rl_conv_pack_floats(int mode_up, int Cs, int Cb);
int b200rl_conv_pack(const float* W, float* Wpacked, int mode_up, int Cs, int Cb, cudaStream_t stream);
int b200rl_conv_down_tc(const float* big, const float* Wpacked, float* small_, int NB, int h, int w, int Cs, int Cb,
                        cudaStream_t stream);
int b200rl_conv_up_tc(const float* small_, const float* Wpacked, float* big, const float* bias, int NB, int h, int w,
                      int Cs, int Cb, cudaStream_t stream);
/* The packed weight as its TF32 planes (two workspaces of b200rl_conv_pack_floats() floats each), and the conv forwards
 * that read them; bit-identical to b200rl_conv_pack + b200rl_conv_down_tc / _up_tc. */
int b200rl_conv_pack_split(const float* W, float* Whi, float* Wlo, int mode_up, int Cs, int Cb, cudaStream_t stream);
int b200rl_conv_down_tc_presplit(const float* big, const float* Whi, const float* Wlo, float* small_, int NB, int h, int w,
                                 int Cs, int Cb, cudaStream_t stream);
int b200rl_conv_up_tc_presplit(const float* small_, const float* Whi, const float* Wlo, float* big, const float* bias,
                               int NB, int h, int w, int Cs, int Cb, cudaStream_t stream);

/* ---- RSSM ------------------------------------------------------------------------------------------
 * LayerNormGRUCell gates models.py:399-403; is_first masking agent.py:425-430; unimix agent.py:437-449;
 * straight-through categorical sampling dreamer_v2/utils.py:44-61 (noise q ~ Exp(1): sample =
 * argmax(probs / q), noise == NULL -> mode); KL balancing + free nats loss.py:61-75. */
int b200rl_gru_gate_fwd(const float* G, const float* Hin, float* Hout, long long M, int R, long long ldg,
                        long long ldhi, long long ldho, cudaStream_t stream);
int b200rl_gru_gate_bwd(const float* G, const float* Hin, const float* dH, float* dG, float* dHin, long long M, int R,
                        long long ldg, long long ldhi, long long lddh, long long lddg, long long lddhi,
                        cudaStream_t stream);
int b200rl_mask_mix(const float* prev, const float* init_row, const float* first, float* out, long long M, int C,
                    long long ldp, long long ldo, cudaStream_t stream);
int b200rl_mask_bwd(const float* dIn, const float* first, float* dPrev, float* dInit, int M, int C, long long ldi,
                    long long ldp, cudaStream_t stream);
int b200rl_cat_sample(const float* raw, const float* noise, float* onehot, float* mix_out, long long M, int groups,
                      int classes, long long ldr, long long ldn, long long ldo, long long ldm, float unimix,
                      cudaStream_t stream);
/* Policy head + straight-through sample in one launch (Actor.mlp_heads[i] + OneHotCategoricalStraightThrough.rsample,
 * sheeprl/algos/dreamer_v3/agent.py:793-818): raw [M, A] = X W^T + bias, onehot = sample(unimix(raw), noise) with
 * b200rl_cat_sample's rule.  A <= 32, Kin <= 1024, Kin % 4 == 0, 16-byte aligned rows: `_supported` is 1 for the
 * operands the launch runs (it reads the pointer values, never through them). */
int b200rl_head_sample_supported(const float* X, const float* W, int Kin, int A, long long ldx, long long ldw);
int b200rl_head_sample(const float* X, const float* W, const float* bias, const float* noise, float* raw, float* onehot,
                       long long M, int Kin, int A, long long ldx, long long ldw, long long ldr, long long ldn,
                       long long ldo, float unimix, cudaStream_t stream);
/* MinedojoActor's masked, chained sample (sheeprl/algos/dreamer_v3/agent.py:898-932) in one launch: the three heads
 * [K0 | K1 | K2] are consecutive column blocks of each row of raw, noise and onehot.  Per row: head 0 with
 * mask_action_type; head 1 with mask_craft_smelt when head 0 drew class 15 (craft), else unmasked; head 2 with
 * mask_equip_place after 16 / 17 (equip / place), mask_destroy after 18 (destroy), else unmasked.  Masks are float
 * rows (nonzero = allowed; NULL = all allowed) applied after unimix; the draw is b200rl_cat_sample's, so with every class
 * allowed the one-hot rows are bit-identical to three b200rl_cat_sample calls.  A mask row that allows no class leaves
 * its head unmasked (the reference's distribution would have NaN logits).  Only the K0 + K1 + K2 one-hot columns of a
 * row are written.  `_supported`: every head has 1 to 2048 classes. */
int b200rl_minedojo_sample_supported(int K0, int K1, int K2);
int b200rl_minedojo_sample(const float* raw, const float* noise, float* onehot, const float* mask_action_type,
                           const float* mask_craft_smelt, const float* mask_equip_place, const float* mask_destroy,
                           long long M, int K0, int K1, int K2, long long ldr, long long ldn, long long ldo,
                           long long ld_action_type, long long ld_craft_smelt, long long ld_equip_place,
                           long long ld_destroy, float unimix, cudaStream_t stream);
int b200rl_cat_sample_bwd(const float* raw, const float* dz, const float* dmix, float* draw, long long M, int groups,
                          int classes, long long ldr, long long lddz, long long lddm, long long lddr, float unimix,
                          cudaStream_t stream);
/* KL(post || prior) summed over the groups with free nats (loss.py), its rows and the gradients w.r.t. both mixes;
 * held to a float64 reference with first-order error bounds (tests/test_gpu_loss_precision.py). */
int b200rl_kl_loss_grad(const float* post_mix, const float* prior_mix, float* d_post, float* d_prior, float* rows,
                        long long M, int groups, int classes, long long ldp, long long ldq, long long lddp,
                        long long lddq, float kl_dyn, float kl_rep, float free_nats, float regularizer, float scale,
                        cudaStream_t stream);
/* Persistent fused scan: all T steps of the POSTERIOR recurrence of RSSM.dynamic (dreamer_v3.py:131-145 ->
 * agent.py:396-435: recurrent model, representation model, unimix, straight-through sample) in ONE cooperative
 * kernel; weight slices resident in shared memory, cross-SM hand-offs as flag-carrying data exchanges instead of grid
 * barriers (rssm_scan.cu).  The prior (transition model on the finished h sequence, agent.py:433) is NOT computed here:
 * it is off the recurrence and runs as batched products over all T*B rows (tr_pre / tr_act / prior_raw / prior_mix
 * below are unused by the kernels; the fields stay so that the per-step path and this one fill the same set of saved
 * activations).  Requires B <= 16, S <= 64 categoricals of D <= 32 classes, even widths (R, Dx, Dr and S*D),
 * Dx <= 1024, R <= 1024 (at most two 4-column groups per CTA), Dr <= 4096 and the per-CTA weight slices to fit in
 * 227 KB of shared memory; the backward kernel needs more of it than the forward, so it can refuse a model the forward
 * runs.  b200rl_rssm_scan_check answers that per direction; a caller asks it once and runs the per-step ops where it
 * refuses.  The launches refuse the same models (and a short workspace) before launching anything.
 * Checked against a float64 reference (tests/test_gpu_rssm_scan.py) at widths up to R = Dx = 520 and Dx = 1024, one to
 * sixteen rows, S = 1 .. 64 and D = 1 .. 32. */
typedef struct b200rl_rssm_scan_args {
  int T, B, S, D, R, A, Dx, Dt, Dr, ld_lat, ld_wr1;
  float eps, unimix;
  const float *W_in, *lnx_g, *lnx_b, *W_g, *lng_g, *lng_b, *W_t1, *lnt_g, *lnt_b, *W_t2, *b_t2;
  const float *W_r1, *lnr_g, *lnr_b, *W_r2, *b_r2;
  const float *h0, *z0;                       /* [R] tanh(initial_recurrent_state); [S*D] one-hot initial posterior */
  const float *pe, *actions, *first, *noise;  /* [T,B,Dr] embed projection; [T,B,A] shifted; [T,B]; [T,B,S*D] Exp(1) */
  float* latent;                              /* [T*B, ld_lat]: z (S*D) | h (R) */
  float *z_in, *h_in, *a_in, *x_pre, *x_act, *g_pre, *g_ln, *tr_pre, *tr_act, *rp_pre, *rp_act;
  float *post_raw, *prior_raw, *post_mix, *prior_mix;
  void* workspace;
  long long workspace_bytes;
} b200rl_rssm_scan_args;
/* Gradient buffers of the persistent BPTT kernel (same meaning as the per-step path's buffers):
 * inputs d_latent [T*B, ld_lat] (grad wrt z|h from decoder + heads + the batched prior backward), d_post_mix (KL seed
 * grads); outputs: d_post_raw and the per-step ACTIVATION gradients d_rp_act / d_g_ln / d_x_act (the batched
 * LayerNorm-backward kernels turn them into d_rp_pre / d_g_pre / d_x_pre afterwards), and d_h0 [R].
 * d_prior_mix / d_prior_raw / d_tr_act / d_tr_pre / d_*_pre are unused by the kernel. */
typedef struct b200rl_rssm_scan_grads {
  const float *d_latent, *d_post_mix, *d_prior_mix;
  float *d_post_raw, *d_prior_raw, *d_rp_act, *d_rp_pre, *d_tr_act, *d_tr_pre, *d_g_ln, *d_g_pre, *d_x_act, *d_x_pre;
  float* d_h0;
  /* pre-activation x weight products over all T*B rows (batched, before the kernel; they let the consumer of a
   * LayerNorm gradient apply the LayerNorm-backward correction by linearity, rssm_scan.cu):
   * q_r = rp_pre W_r1[:, :R] [T*B, R];  q_g = g_pre W_g [T*B, R+Dx];  q_x = x_pre W_in[:, :S*D] [T*B, S*D] */
  const float *q_r, *q_g, *q_x;
} b200rl_rssm_scan_grads;
long long b200rl_rssm_scan_workspace_bytes(int T, int B, int S, int D, int Dx, int R, int Dr);
int b200rl_rssm_scan_fwd(const b200rl_rssm_scan_args* args, cudaStream_t stream);
/* BPTT over the same scan (autograd replay inside fabric.backward, dreamer_v3.py:191); must follow
 * b200rl_rssm_scan_fwd on the same workspace (uses its saved LayerNorm statistics and class indices). */
int b200rl_rssm_scan_bwd(const b200rl_rssm_scan_args* args, const b200rl_rssm_scan_grads* grads, cudaStream_t stream);
/* envelope of the forward (backward = 0) or backward kernel for the dims of `args`: 0 if it runs them, non-zero +
 * last_error if not.  Reads no pointer (the workspace included) and launches nothing. */
int b200rl_rssm_scan_check(const b200rl_rssm_scan_args* args, int backward);
int b200rl_rssm_scan_error(const void* workspace, cudaStream_t stream);
/* cycle counters (2 x 32 int64: CTA 0, CTA 1) accumulated per phase by the last launch on `workspace` */
int b200rl_rssm_scan_profile(const void* workspace, long long* out64, cudaStream_t stream);
/* Persistent GRU-only scan for the decoupled RSSM (DecoupledRSSM agent.py:501-593, dreamer_v3.py:115-129): the
 * posterior does not depend on h there, so x = SiLU(LN(W_in [z, a])) and its share x W_g[:, R:]^T of the gate
 * pre-activation are batched over all T*B rows by the caller; the kernels run what is left on the recurrence,
 * h_in = (1-f) h_{t-1} + f h0, g_pre += h_in W_g[:, :R]^T, LayerNorm over 3R, gate, for all T steps in one cooperative
 * launch (rssm_scan.cu; same construction and helpers as b200rl_rssm_scan_*).  Requires B <= 16, R even and <= 1024,
 * and the per-CTA W_g[:, :R] slice to fit in 227 KB of shared memory.  b200rl_gru_scan_check answers that per direction,
 * reads no pointer and launches nothing; the launches refuse the same shapes (and a short workspace) before launching.
 * b200rl_rssm_scan_error reads the error word of this workspace too. */
typedef struct b200rl_gru_scan_args {
  int T, B, R, ld_wg, ld_lat, lat_off;        /* h_t is written to latent[t*B + b, lat_off : lat_off + R] */
  float eps;
  const float *W_g, *lng_g, *lng_b;           /* [3R, ld_wg], columns [:R] are read; GRU LayerNorm weight, bias [3R] */
  const float *h0, *first;                    /* [R] tanh(initial_recurrent_state); [T*B] */
  float* g_pre;                               /* [T*B, 3R] in: x's share of the pre-activation; out: all of it */
  float *g_ln, *h_in, *latent;                /* [T*B, 3R]; [T*B, R]; [T*B, ld_lat] */
  void* workspace;
  long long workspace_bytes;
} b200rl_gru_scan_args;
/* d_latent [T*B, ld_lat] (its h columns are read); q_g = g_pre W_g[:, :R] [T*B, R] over all rows (lets the consumer of
 * the LayerNorm gradient apply the LayerNorm-backward correction by linearity); outputs d_g_ln [T*B, 3R], the gradient
 * of the LayerNorm's output (the batched LayerNorm-backward kernel turns it into d_g_pre afterwards), and d_h0 [R]. */
typedef struct b200rl_gru_scan_grads {
  const float *d_latent, *q_g;
  float *d_g_ln, *d_h0;
} b200rl_gru_scan_grads;
long long b200rl_gru_scan_workspace_bytes(int T, int B, int R);
int b200rl_gru_scan_fwd(const b200rl_gru_scan_args* args, cudaStream_t stream);
/* must follow b200rl_gru_scan_fwd on the same workspace (uses its saved LayerNorm statistics) */
int b200rl_gru_scan_bwd(const b200rl_gru_scan_args* args, const b200rl_gru_scan_grads* grads, cudaStream_t stream);
int b200rl_gru_scan_check(const b200rl_gru_scan_args* args, int backward);

/* ---- losses (value + seed gradient) -----------------------------------------------------------------
 * distribution.py:212-276 (MSE, two-hot on symlog), Bernoulli continue head loss.py:77, lambda returns
 * dreamer_v3/utils.py:66-77 + dreamer_v3.py:244-260, Moments dreamer_v3/utils.py:40-63, discrete policy
 * loss dreamer_v3.py:272-297.  Each is held to a float64 reference with per-element first-order error bounds, and
 * moments_update to torch.quantile's order statistics, NaN included (tests/test_gpu_loss_precision.py). */
int b200rl_mse_loss_grad(const float* pred, const float* target, float* loss_row, float* grad, long long M, int P,
                         float scale, cudaStream_t stream);
int b200rl_twohot_loss_grad(const float* logits, const float* x, const float* weight, float* loss_row, float* dlogits,
                            long long M, int nbins, long long ldl, long long ldd, float low, float high, float scale,
                            int accumulate, cudaStream_t stream);
int b200rl_bce_loss_grad(const float* logit, const float* target, float* loss_row, float* dlogit, long long M,
                         float loss_scale, float scale, cudaStream_t stream);
int b200rl_twohot_mean(const float* logits, float* out, long long M, int nbins, long long ldl, float low, float high,
                       cudaStream_t stream);
int b200rl_lambda_returns(const float* rew, const float* val, const float* cont_logit, const float* true_cont,
                          float* lam, float* discount, int H, int N, float gamma, float lmbda, cudaStream_t stream);
int b200rl_moments_update(const float* x, long long n, float* state_low_high, float* out_offset_invscale, float decay,
                          float max_, float p_low, float p_high, cudaStream_t stream);
int b200rl_actor_loss_grad(const float* raw, const float* actions, const float* lam, const float* val,
                           const float* discount, const float* moments, float* rows, float* draw, long long M,
                           const int* head_dims_host, int n_heads, float unimix, float ent_coef, float scale,
                           cudaStream_t stream);
int b200rl_sum_rows(const float* X, float* out, long long M, int C, long long ldx, float scale, cudaStream_t stream);
int b200rl_weighted_mean(const float* x, const float* w, float* out, long long n, float scale, cudaStream_t stream);

/* ---- optimiser -----------------------------------------------------------------------------------------
 * clip_grad_norm_ + torch.optim.Adam.step fused (dreamer_v3.py:191-200,298-304,318-327); target-critic
 * EMA dreamer_v3.py:674-680; Exp(1) noise for categorical sampling (torch.multinomial).  The clip coefficient is
 * clip_grad_norm_'s clamp(max_norm / (total + 1e-6), max=1): a NaN gradient element makes it NaN, and the whole group
 * NaN, as in the reference.  sumsq (both modes), adam_step, adam_step_wd, rmsprop_step and ema are held to a float64
 * reference with per-element first-order bounds, every step from the kernel's own state, at the float4 tails, unaligned
 * views, several grid-stride passes, step counts up to 1e6 and non-finite gradients (tests/test_gpu_optim_precision.py),
 * and so are copy2d, axpy, affine, symlog, tanh_fwd and tanh_bwd below. */
int b200rl_sumsq(const float* x, long long n, double* out, cudaStream_t stream);
int b200rl_adam_step(float* p, const float* g, float* m, float* v, const double* normsq, const int* step_dev,
                     float* norm_out, long long n, float max_norm, float lr, float b1, float b2, float eps,
                     cudaStream_t stream);
/* adam_step with torch.optim.Adam's L2 weight decay (Dreamer-V2's optimizers, configs/algo/dreamer_v2.yaml:99,118,133):
 * weight_decay * p is added to the clipped gradient before the moments.  weight_decay = 0 runs adam_step's kernel, bit
 * for bit; weight_decay < 0 is refused.  Covered by tests/test_gpu_adam_wd.py. */
int b200rl_adam_step_wd(float* p, const float* g, float* m, float* v, const double* normsq, const int* step_dev,
                        float* norm_out, long long n, float max_norm, float lr, float b1, float b2, float eps,
                        float weight_decay, cudaStream_t stream);
/* fabric.clip_gradients + torch.optim.RMSprop.step (single-tensor path; A2C, a2c/a2c.py:102-105) in one pass, with
 * adam_step's normsq / norm_out contract and clip coefficient.  square_avg always; momentum_buf read and written only when momentum > 0;
 * grad_avg non-NULL selects `centered`.  eps is added after the square root; the step count does not enter the update. */
int b200rl_rmsprop_step(float* p, const float* g, float* square_avg, float* momentum_buf, float* grad_avg,
                        const double* normsq, float* norm_out, long long n, float max_norm, float lr, float alpha,
                        float eps, float weight_decay, float momentum, cudaStream_t stream);
int b200rl_ema(float* target, const float* src, long long n, float tau, cudaStream_t stream);
int b200rl_fill_exponential(float* out, long long n, unsigned long long seed, unsigned int stream_id,
                            const int* counter_dev, cudaStream_t stream);
int b200rl_zero(float* x, long long n, cudaStream_t stream);
int b200rl_copy2d(const float* src, float* dst, long long M, int C, long long lds, long long ldd, cudaStream_t stream);
int b200rl_axpy(const float* x, float* y, long long n, float alpha, cudaStream_t stream);
int b200rl_affine(const float* x, float* y, long long n, float alpha, float beta, cudaStream_t stream);
/* y[M,C] = symlog(x[M,C]) = sign(x) log(1 + |x|)  (sheeprl/utils/utils.py:148): the squashing of vector observations in
 * MLPEncoder.forward (dreamer_v3/agent.py:150) and the regression target of SymlogDistribution (utils/distribution.py:180). */
int b200rl_symlog(const float* x, float* y, long long M, int C, long long ldx, long long ldy, cudaStream_t stream);
int b200rl_tanh_fwd(const float* x, float* y, long long n, cudaStream_t stream);
int b200rl_tanh_bwd(const float* y, const float* dy, float* dx, long long n, int accumulate, cudaStream_t stream);
int b200rl_increment(int* p, cudaStream_t stream);

/* ---- replay storage / PPO -------------------------------------------------------------------------------
 * SequentialReplayBuffer._get_samples buffers.py:467-526 (+ get_tensor :1158-1180), ReplayBuffer.add
 * buffers.py:145-221, gae utils/utils.py:63-100.  idx: int64 flat row indices in (sample, batch, time)
 * order exactly as the reference computes them on the host; out rows in (sample, time, batch) order. */
int b200rl_replay_gather(const void* storage, const long long* idx, void* out, int n_samples, int batch, int seq_len,
                         long long row_bytes, cudaStream_t stream);
int b200rl_replay_scatter(const void* src, const long long* dst_rows, void* storage, long long n_rows,
                          long long row_bytes, cudaStream_t stream);
int b200rl_gae(const float* rewards, const float* values, const float* dones, const float* next_value, float* returns,
               float* advantages, int T, int E, float gamma, float lmbda, cudaStream_t stream);

/* ---- SAC / PPO dense layers and SAC element-wise stages ---------------------------------------------------
 * b200rl_bgemm: `nets` independent products C[n] = epi(A[n] * B[n] + bias[n]) in one launch; A(m,k) = A[m*sam+k*sak],
 * B(k,n) = B[k*sbk+n*sbn] (covers NN/NT/TN), C row-major with ldc.  epilogue: 0 none, 1 ReLU, 2 Tanh, 3 multiply by
 * ReLU'(aux), 4 multiply by Tanh'(aux) = 1-aux^2 (aux = the layer's saved activation output).  rsum (optional):
 * rsum[m] = sum_k A(m,k), i.e. the bias gradient when A = dY^T.  Replaces nn.Linear + activation forward/backward
 * of models/models.py:16-119 as used by sac/agent.py:19-108 and ppo/agent.py:84-177.  Every tile config, epilogue and
 * split-K form, up to the A2C weight gradients' K = 65536, is checked against a float64 reference
 * (tests/test_gpu_simt_precision.py). */
int b200rl_bgemm(const float* A, long long sam, long long sak, long long strideA, const float* B, long long sbk,
                 long long sbn, long long strideB, float* C, long long ldc, long long strideC, const float* bias,
                 long long strideBias, const float* aux, long long ldaux, long long strideAux, float* rsum,
                 long long strideRsum, int M, int N, int K, int nets, int epilogue, int accumulate, cudaStream_t stream);
/* SACActor._get_actions_and_log_probs sac/agent.py:110-142: head = [mean | log_std] (B x 2A), eps ~ N(0,1);
 * writes the rescaled tanh action into `action` (row stride ld_action: straight into the critics' input buffer),
 * logp[B], and tanh(x_t) for the backward. */
int b200rl_sac_sample_fwd(const float* head, const float* eps, const float* scale, const float* abias, float* action,
                          long long ld_action, float* logp, float* tanh_out, int B, int A, cudaStream_t stream);
/* autograd of the above for the policy loss (loss.py:9-11): d(action) = sum over `nets` critics' input gradients,
 * d(logp) = exp(log_alpha)/B. */
int b200rl_sac_sample_bwd(const float* head, const float* eps, const float* tanh_y, const float* scale,
                          const float* dact, long long stride_net, int nets, const float* log_alpha, float* dhead, int B,
                          int A, cudaStream_t stream);
/* SACAgent.get_next_target_q_values sac/agent.py:254-262 (alpha read from the device log_alpha) */
int b200rl_sac_target(const float* q_target, long long stride_net, int nets, const float* logp, const float* rewards,
                      const float* terminated, const float* log_alpha, float gamma, float* y, int B, cudaStream_t stream);
/* critic_loss sac/loss.py:14-20 + its gradient w.r.t. q */
int b200rl_sac_critic_loss(const float* q, long long stride_net, int nets, const float* y, float* dq, float* loss_out,
                           int B, cudaStream_t stream);
/* policy_loss + entropy_loss sac/loss.py:9-11,23-26 with torch.min over critics (sac.py:62-63): gradients w.r.t. q
 * and log_alpha */
int b200rl_sac_actor_loss(const float* q, long long stride_net, int nets, const float* logp, const float* log_alpha,
                          float target_entropy, float* dq, float* actor_loss, float* alpha_loss, float* dlog_alpha, int B,
                          cudaStream_t stream);
/* N(0,1) noise (Philox4x32-10 + Box-Muller), same counter scheme as b200rl_fill_exponential; replaces
 * Normal.rsample's torch.normal draw (sac/agent.py:126) */
int b200rl_fill_normal(float* out, long long n, unsigned long long seed, unsigned int stream_id, const int* counter_dev,
                       cudaStream_t stream);

/* ---- DroQ critics (csrc/droq.cu) ----------------------------------------------------------------------------
 * DroQ's policy loss: b200rl_sac_actor_loss with the mean over the critics in place of the min (droq/droq.py:147-150):
 * actor_loss = mean(alpha*logp - mean_n q[n]), dq[n,b] = -1/(nets*B); alpha loss and its gradient as SAC's. */
int b200rl_droq_actor_loss(const float* q, long long stride_net, int nets, const float* logp, const float* log_alpha,
                           float target_entropy, float* dq, float* actor_loss, float* alpha_loss, float* dlog_alpha,
                           int B, cudaStream_t stream);
/* nn.Dropout's keep masks (Bernoulli(1-p), droq/agent.py:40-42) for n_words 32-bit words, bit-packed: a [n, B, H]
 * activation takes [n, B, ceil(H/32)] words, bit j of word k keeping column 32k + j.  Philox4x32-10 keyed by (seed,
 * stream_id, *counter_dev) as b200rl_fill_normal, so one launch fills the masks of every critic forward of a train()
 * call without a host synchronisation. */
int b200rl_dropout_mask(unsigned int* mask, long long n_words, float p, unsigned long long seed, unsigned int stream_id,
                        const int* counter_dev, cudaStream_t stream);
/* The miniblock after each hidden Linear of the DroQ critic (utils/model.py:34-88: Dropout(p) -> LayerNorm(H, eps) ->
 * ReLU) for all `nets` critics in one launch: y = relu(LN(z * mask / (1-p)) * gamma + beta).  z, y [nets, B, H]
 * contiguous; mask [nets, B, ceil(H/32)] words (NULL iff p == 0; bits past column H are never read); gamma / beta of
 * critic i at i * stride_param; stats [nets, B, 2] = (mean, 1/std) per row, kept for the backward.  1 <= H <= 1024:
 * `_supported` answers for H. */
int b200rl_dropout_ln_relu_supported(int H);
int b200rl_dropout_ln_relu_fwd(const float* z, const unsigned int* mask, float p, const float* gamma, const float* beta,
                               long long stride_param, float eps, float* y, float* stats, int nets, int B, int H,
                               cudaStream_t stream);
/* its autograd backward: dReLU, LayerNorm backward, then the mask scale, giving dz [nets, B, H] from dy.  dgamma / dbeta
 * (both or neither, same stride as gamma) are reduced over the rows in a fixed order, bit-identical run to run; NULL
 * gives the input-gradient-only pass of the policy loss. */
int b200rl_dropout_ln_relu_bwd(const float* dy, const float* y, const float* z, const unsigned int* mask, float p,
                               const float* stats, const float* gamma, long long stride_param, float* dz, float* dgamma,
                               float* dbeta, int nets, int B, int H, cudaStream_t stream);

/* ---- PPO --------------------------------------------------------------------------------------------------
 * Channel-last patch gather / scatter for NatureCNN's unpadded convolutions (models/models.py:288-328):
 * col[(b,oy,ox),(ky,kx,c)] = x[b,oy*s+ky,ox*s+kx,c]; col2im is its transpose (sum over overlapping patches), optionally
 * masked by ReLU'(act) of the activation that fed the convolution.  im2col is checked bit for bit and col2im against a
 * float64 bound on the overlap sum (tests/test_gpu_optim_precision.py). */
int b200rl_im2col(const float* x, float* col, int B, int H, int W, int C, int k, int stride, cudaStream_t stream);
int b200rl_col2im(const float* dcol, const float* act, float* dx, int B, int H, int W, int C, int k, int stride,
                  cudaStream_t stream);
/* PPO objective on one minibatch: log-prob + entropy of the taken actions from the actor head (OneHotCategorical per
 * head / Independent Normal, ppo/agent.py:179-239), optional advantage normalisation (utils/utils.py:121-130),
 * policy / value / entropy losses (ppo/loss.py:6-75, reduction mean) and the gradients of
 * policy + vf_coef*value + ent_coef*entropy w.r.t. the head outputs and the values.  losses[3].
 * is_continuous: 0 discrete, 1 `normal`, 2 `tanh_normal` (stored actions are tanh-squashed, agent.py:194-206). */
int b200rl_ppo_loss(const float* head, const float* actions, const float* old_logp, const float* adv,
                    const float* values, const float* old_values, const float* returns, float* dhead, float* dvalues,
                    float* losses, int B, const int* head_dims, int n_heads, int is_continuous, int clip_vloss,
                    int normalize_adv, float clip_coef, float vf_coef, float ent_coef, cudaStream_t stream);

/* The same objective over the rows whose mask[b] != 0 (recurrent PPO, ppo_recurrent.py:77-101): means over their
 * count n (computed on the device), advantages normalised over them only when n > 1, zero dhead / dvalues on the other
 * rows.  n == 0 gives zero losses and gradients. */
int b200rl_ppo_loss_masked(const float* head, const float* actions, const float* old_logp, const float* adv,
                           const float* values, const float* old_values, const float* returns, const float* mask,
                           float* dhead, float* dvalues, float* losses, int B, const int* head_dims, int n_heads,
                           int is_continuous, int clip_vloss, int normalize_adv, float clip_coef, float vf_coef,
                           float ent_coef, cudaStream_t stream);
/* A2C objective (a2c/a2c.py:60-100, a2c/loss.py, ppo/loss.py:44-75) of every minibatch of a rollout in one launch,
 * one CTA per minibatch.  Rows are the gathered rollout in sampler order; minibatch i is rows [i*seg, min(N, (i+1)*seg))
 * (the last one may be short).  Per minibatch: optional advantage normalisation (unbiased std + 1e-8), policy
 * -(logp*adv), value (value - return)^2 and entropy -entropy losses reduced by mean (reduce_sum 0) or sum (1);
 * dhead / dvalues = gradient of policy + vf_coef*value + ent_coef*entropy of the row's own minibatch; losses[n_seg, 3].
 * Distributions as b200rl_ppo_loss.  normalize_adv needs at least two rows in every minibatch. */
int b200rl_a2c_loss(const float* head, const float* actions, const float* adv, const float* values, const float* returns,
                    float* dhead, float* dvalues, float* losses, int N, int seg, const int* head_dims, int n_heads,
                    int is_continuous, int normalize_adv, int reduce_sum, float vf_coef, float ent_coef,
                    cudaStream_t stream);
/* Single-layer LSTM over padded time-major sequences in one launch (recurrent PPO, ppo_recurrent/agent.py:67-80; torch
 * gate order i, f, g, o).  xw [T, B, 4H] = x W_ih^T + b_ih + b_hh; W_hh [4H, H]; h0, c0 [B, H]; lengths [B] int32 in
 * [1, T] (sequence b is valid for t < lengths[b]).  out [T, B, H] (0 at padded steps); gates [T, B, 4H] (activated)
 * and cs [T, B, H] (cell state) are kept for the backward, both or neither (NULL when acting); hT, cT [B, H]
 * (nullable): the state after each sequence's last valid step. */
int b200rl_lstm_seq_fwd(const float* xw, const float* W_hh, const float* h0, const float* c0, const int* lengths,
                        float* out, float* gates, float* cs, float* hT, float* cT, int T, int B, int H,
                        cudaStream_t stream);
/* Backward through time in one launch: d_gates [T, B, 4H] = gradient w.r.t. the pre-activation gates from d_out
 * [T, B, H] and what the forward kept; zero at padded steps.  h0 / c0 get no gradient.  The weight, bias and input
 * gradients are dense products of d_gates done by the caller.  Both kernels are checked against a float64 reference with
 * propagated error bounds, for every sequences-per-CTA width (tests/test_gpu_simt_precision.py). */
int b200rl_lstm_seq_bwd(const float* d_out, const float* W_hh, const float* gates, const float* cs, const float* c0,
                        const int* lengths, float* d_gates, int T, int B, int H, cudaStream_t stream);

/* Linear([z, a]) for a one-hot z (S groups of K classes, straight-through categorical sample) as a gather-sum over the
 * transposed weight WT [S*K + A, N]: RecurrentModel.mlp's first Linear (agent.py:328-341) inside the imagination
 * rollout.  z: [M, S*K] (row stride ldz), act: [M, A], out: [M, N].  S <= 64 groups, A <= 32: `_supported` is 1 for
 * the dims the launch runs. */
int b200rl_onehot_linear_supported(int S, int K, int A, int N);
int b200rl_onehot_linear(const float* z, const float* act, const float* WT, float* out, long long M, int S, int K, int A,
                         int N, long long ldz, long long lda, long long ldo, cudaStream_t stream);
/* The same gather followed, in the same launch, by the miniblock's LayerNorm(eps) + SiLU: out = SiLU(LN(Linear([z, a])));
 * `pre` (optional) keeps the Linear output.  The dims of b200rl_onehot_linear_supported, N a multiple of 128 up to 1024
 * (one float4 of the row per thread), 16-byte aligned WT / gamma / beta / out / pre rows.  `_ln_supported` answers the
 * terms beyond b200rl_onehot_linear_supported's from the pointer values, without reading through them; a NULL pointer
 * passes its alignment term (the launch refuses a NULL gamma or beta on its own). */
int b200rl_onehot_linear_ln_supported(const float* WT, const float* gamma, const float* beta, const float* out,
                                      const float* pre, int N, long long ldo, long long ldpre);
int b200rl_onehot_linear_ln(const float* z, const float* act, const float* WT, const float* gamma, const float* beta,
                            float eps, float* pre, long long ldpre, float* out, long long M, int S, int K, int A, int N,
                            long long ldz, long long lda, long long ldo, cudaStream_t stream);

/* ---- Dreamer-V3 continuous actions (policy gradient through the imagined rollout) -------------------------
 * Actor.forward `scaled_normal` branch agent.py:803-825: head = [mean | std_raw] (M x 2A), eps ~ N(0,1);
 * action (row stride lda) = clip-rescaled tanh(mean) + std*eps, ent[M] = Independent(Normal).entropy().  The four
 * entry points below are held to a float64 reference with first-order error bounds (tests/test_gpu_loss_precision.py). */
int b200rl_cont_action_fwd(const float* head, const float* eps, float* action, long long lda, float* ent, long long M,
                           int A, float min_std, float max_std, float init_std, float clip, cudaStream_t stream);
/* its backward: d_action (row stride ldd) and the entropy bonus d_ent[m] = ent_scale * discount[m] -> dhead */
int b200rl_cont_action_bwd(const float* head, const float* eps, const float* d_action, long long ldd,
                           const float* discount, float* dhead, long long M, int A, float min_std, float max_std,
                           float init_std, float clip, float ent_scale, cudaStream_t stream);
/* continuous objective dreamer_v3.py:276-296 + backward of compute_lambda_values (dreamer_v3/utils.py:66-77):
 * rows[H,N] = discount*(advantage + ent_coef*entropy); d_val / d_rew [H+1,N] = d(policy_loss)/d(values, rewards) */
int b200rl_lambda_returns_bwd(const float* cont_logit, const float* discount, const float* moments, const float* lam,
                              const float* val, const float* ent, float* d_val, float* d_rew, float* rows, int H, int N,
                              float gamma, float lmbda, float ent_coef, float scale, cudaStream_t stream);
/* backward of TwoHotEncodingDistribution.mean (distribution.py:245-247): d_logits = d_mean * dsymexp * softmax' */
int b200rl_twohot_mean_bwd(const float* logits, const float* d_mean, float* d_logits, long long M, int nb, long long ldl,
                           long long ldd, float low, float high, cudaStream_t stream);

/* Convolution weight gradient with both operands read in place as MN-major tiles (no im2col, no transposes):
 * G[(tap, cb), cs] = sum over small pixels p of big[patch(p)][tap][cb] * small[p][cs]; big [NB,2h,2w,Cb] and small
 * [NB,h,w,Cs] channel-last, G [16*Cb][Cs] (unpacked to the reference's [Cs][Cb][4][4] by b200rl_conv_wgrad_tc).
 * Replaces the autograd weight-gradient of CNNEncoder / CNNDecoder convolutions (agent.py:78-91, :199-222). */
int b200rl_conv_wgrad_mn_supported(int NB, int h, int w, int Cs, int Cb);
int b200rl_conv_wgrad_mn(const float* small_, const float* big, float* G, int NB, int h, int w, int Cs, int Cb,
                         cudaStream_t stream);

/* PPOPlayer.forward / get_actions (ppo/agent.py:269-322): per-head categorical sample (Exp(1) noise; mode when greedy or
 * noise == NULL) or Normal sample (N(0,1) noise; mean when greedy) from the actor head, its log-probability logp[B];
 * actions: one-hot [B, sum(head_dims)] or [B, A].  is_continuous: 0 discrete, 1 `normal`, 2 `tanh_normal` as
 * forward() returns it (safetanh + corrected log-prob, :257-268), 3 `tanh_normal` as get_actions() returns it (:306-311). */
int b200rl_ppo_act(const float* head, const float* noise, float* actions, float* logp, int B, const int* head_dims,
                   int n_heads, int is_continuous, int greedy, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H_ */
