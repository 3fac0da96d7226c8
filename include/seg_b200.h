/*
 * seg_b200.h — C ABI of the H100-native segmentation hot path.
 *
 * Drop-in boundary for the forward/backward hot path of yassouali/pytorch-segmentation
 * (dilated-ResNet encoder -> ASPP / PSP head -> bilinear upsample -> per-pixel loss).  The reference is
 * 100 % Python and dispatches every op below to ATen/cuDNN; each entry point here names the reference call
 * site(s) whose ATen op it replaces (path:line relative to the reference tree).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; seg_last_error() gives the message
 *     (thread-local).  Python wrappers turn a non-zero status into RuntimeError (the reference's convention is
 *     Python exceptions, e.g. trainer.py:58-59).
 *   - all pointers are BORROWED device pointers; the library allocates nothing the caller must free.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream).
 *   - activations are NHWC; `ld*` is the channel pitch (elements) of the buffer a tensor lives in, so a tensor
 *     can be a channel slice of a wider concat buffer (replaces torch.cat, deeplabv3_plus.py:293,329).
 *   - bf16 = raw uint16 storage of __nv_bfloat16.  dtype codes: 0 = bf16, 1 = fp32.
 *   - packed conv weights: bf16 [R*S][K][C] (tap-major, then output channel, input channel contiguous).
 *   - nothing here falls back to the CPU; a missing GPU / wrong arch is an error.
 */
#ifndef SEG_B200_H
#define SEG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SEG_DT_BF16 0
#define SEG_DT_F32 1

/* implementation selector for the conv entry points */
#define SEG_IMPL_AUTO 0 /* wgmma where the shape and the operand base addresses allow (the TMA-read operands —
                         * fprop x, dgrad dy, wgrad dy and x, packed weights — 16-byte aligned), else SIMT */
#define SEG_IMPL_SIMT 1 /* CUDA-core implicit GEMM (any shape) */
#define SEG_IMPL_TC 2   /* wgmma + TMA implicit GEMM, error if shape unsupported */

typedef struct seg_conv_desc {
  int32_t N, H, W, C;   /* input  [N,H,W,C]  (C = input channels)                 */
  int32_t K;            /* output channels                                           */
  int32_t R, S;         /* filter taps                                               */
  int32_t stride, pad, dil;
  int32_t P, Q;         /* output spatial size                                       */
  int32_t ldx;          /* channel pitch of the input buffer  (>= C, multiple of 8)  */
  int32_t ldy;          /* channel pitch of the output buffer (>= K)                 */
} seg_conv_desc;

/* SyncBN exchange handle (seg_comm_*): device array of every rank's symmetric-buffer pointer + this rank.  Passed to the
 * kernels that produce BatchNorm statistics so the cross-GPU exchange (utils/sync_batchnorm/batchnorm.py:105-126:
 * ReduceAddCoalesced + Broadcast + thread pipes) rides inside them, with no launch of its own (csrc/seg_sync.cuh): the
 * producer's last block performs the whole exchange and leaves the WORLD's totals in its output (stats / sums), so the
 * consumers (seg_bn_apply_train, seg_bn_bwd_apply) take no handle.  32 bytes. */
typedef struct seg_sync_desc {
  void* const* peers;        /* DEVICE array of `world` base pointers; peers[rank] is this rank's buffer */
  int32_t rank, world, n_max;
  int64_t timeout_clocks;    /* spin-wait bound in GPU clocks (<= 0: unbounded) */
} seg_sync_desc;

const char* seg_last_error(void);
int seg_version(void);
/* 0 if the current device is sm_90 and kernels can be launched */
int seg_device_ok(void);
/* number of kernel launches issued by this library since the last reset (gpu_launches in bench.py) */
int64_t seg_launch_count(void);
void seg_launch_count_reset(void);

/* ---- convolution: replaces nn.Conv2d (models/deeplabv3_plus.py:21,256,268,306,312-319; torchvision
 *      Bottleneck conv1/2/3 + downsample.0 mutated at deeplabv3_plus.py:35-53; models/resnet.py:43-48,80-86) ---- */
/* y[N,P,Q,K] = conv(x, w) (+bias[K]);  y = beta*y + result.  y_dtype in {bf16, fp32}.
 * stats (optional): fp64 [2*K], ZERO at launch: per-channel sum and sum of squares of the result as stored — the reduction
 * half of nn.BatchNorm2d, produced by the conv epilogue.  Every CTA adds its (fixed-order) fp32 column sums with one fp64
 * atomic per channel: a sum of fp32 values in fp64 is exact while their exponents span < 2^17, so the order of the atomics
 * cannot change the result — the statistics are bit-reproducible (fp32 atomics would not be).
 * sync (optional, with stats): SyncBN — the last CTA to finish also exchanges the totals (as fp64) with every peer and
 * leaves the WORLD's totals in stats (csrc/seg_sync.cuh); sync_ticket = one zeroed uint32.  The consumer is
 * seg_bn_apply_train with the world's count.  stats requires beta == 0 (an error otherwise, on both implementations).
 * beta != 0 with a bf16 y: the wgmma epilogue rounds the convolution (+bias) to bf16 before it adds beta*y, so the result
 * is rounded twice; the SIMT kernel adds in fp32 and rounds once. */
int seg_conv2d_fwd(const seg_conv_desc* d, const void* x, const void* w_packed, void* y, int y_dtype,
                   const float* bias, float beta, double* stats, const seg_sync_desc* sync, void* sync_ticket,
                   int impl, void* stream);
/* dx[N,H,W,C] = beta*dx + conv_transpose(dy, w)   (autograd of the above w.r.t. x).  Input pixels that no filter tap
 * reaches (a parity class of a strided convolution with no matching tap) become beta*dx.  beta != 0 with the wgmma path:
 * the convolution is rounded to bf16 before beta*dx is added, as in seg_conv2d_fwd. */
int seg_conv2d_dgrad(const seg_conv_desc* d, const void* dy, const void* w_packed, void* dx, float beta,
                     int impl, void* stream);
/* dw_packed (fp32 [R*S][K][C]) += dy^T * im2col(x)   (autograd w.r.t. the weight; caller zeroes dw first).
 * workspace: fp32 scratch of seg_conv2d_wgrad_workspace_floats(d, impl) floats (NULL when that is 0) holding the k-split
 * partial sums, which are added in a fixed order: the result is bit-reproducible.  The SIMT kernel (no workspace) adds
 * its k-splits with fp32 atomics, so its result may differ in the last bits from run to run. */
int64_t seg_conv2d_wgrad_workspace_floats(const seg_conv_desc* d, int impl);
int seg_conv2d_wgrad(const seg_conv_desc* d, const void* dy, const void* x, float* dw_packed, float* workspace, int impl,
                     void* stream);

/* ---- depthwise 3x3 (atrous) convolution: SeparableConv2d.conv1 of the Aligned-Xception backbone
 *      (models/deeplabv3_plus.py:77-78, groups = C).  desc: K == C, R = S = 3.  Packed weights: fp32 [9][C]. ---- */
int64_t seg_dwconv_scratch_floats(int C);
/* y = dw(x); stats (optional, fp64 [2C], zero at launch) += per-channel sum / sum of squares of y as stored (bf16-rounded)
 * (exact fp64 accumulation); sync / sync_ticket: as seg_conv2d_fwd.  All four entry points refuse C or pitches that are
 * not multiples of 8 and x / y / dy / dx base pointers that are not 16-byte aligned. */
int seg_dwconv3x3_fwd(const seg_conv_desc* d, const void* x, const float* w9, void* y, double* stats,
                      const seg_sync_desc* sync, void* sync_ticket, void* stream);
/* dx = beta*dx + dw^T(dy) */
int seg_dwconv3x3_bwd_data(const seg_conv_desc* d, const void* dy, const float* w9, void* dx, float beta, void* stream);
/* dw9 (fp32 [9][C]) = beta*dw9 + sum_pixels dy * x_shifted; scratch: seg_dwconv_scratch_floats(C) floats */
int seg_dwconv3x3_bwd_weight(const seg_conv_desc* d, const void* dy, const void* x, float* dw9, float beta,
                             float* scratch, void* stream);
/* [C][1][3][3] fp32 <-> [9][C] fp32 */
int seg_dw_pack_weight(const float* w_c133, float* w9, int C, void* stream);
int seg_dw_unpack_wgrad(const float* g9, float* g_c133, int C, float beta, void* stream);

/* OIHW fp32 master weight -> packed bf16 [R*S][K][Cpad]; Cpad >= C zero padded */
int seg_pack_weight(const float* w_oihw, void* w_packed, int K, int C, int R, int S, int Cpad, void* stream);
/* packed fp32 grad [R*S][K][Cpad] -> OIHW fp32:  g = beta*g + packed */
int seg_unpack_wgrad(const float* dw_packed, float* g_oihw, int K, int C, int R, int S, int Cpad, float beta,
                     void* stream);
/* Batched forms: one launch for every conv of a model.  `table` is a DEVICE array of n entries
 *   struct { const float* oihw; void* packed; int32 K, C, R, S, Cpad, explicit_rsc; int64 start; }  (48 bytes,
 *   seg_pack_entry_bytes()); `start` = prefix sum of work items (pack: packed elements; unpack: OIHW elements),
 *   explicit_rsc = 1 for the stem-style single-tap [K][(r,s,c)->Cpad] matrix. */
int seg_pack_entry_bytes(void);
int seg_pack_weights_batched(const void* table, int n, int64_t total, void* stream);
int seg_unpack_wgrads_batched(const void* table, int n, int64_t total, float beta, void* stream);
/* explicit im2col for convs TMA cannot address (C % 8 != 0: the 7x7/3-channel stem, deeplabv3_plus.py:21):
 * col[N*P*Q][Kpad] bf16, column order (r, s, c), zero padded to Kpad.  x is NCHW fp32 (x_nchw_f32=1) or NHWC bf16. */
int seg_im2col(const seg_conv_desc* d, const void* x, int x_nchw_f32, void* col, int Kpad, void* stream);

/* ---- batch norm (nn.BatchNorm2d everywhere on the path; sync_batchnorm/batchnorm.py:128-145 for the multi-GPU
 *      variant): statistics, finalize, apply(+residual+ReLU+dropout), backward ---- */
/* stats[0:C] += sum_x, stats[C:2C] += sum_x^2 over M rows of x[M][ldx] (bf16); stats fp64, zero at launch (exact, order-
 * independent accumulation); sync / sync_ticket as seg_conv2d_fwd */
int seg_bn_stats(const void* x, int64_t M, int C, int ldx, double* stats, const seg_sync_desc* sync, void* sync_ticket,
                 void* stream);
/* mean/var from (possibly all-reduced) sums over `count` elements; writes scale_shift[0:C]=gamma*inv_std,
 * [C:2C]=beta-mean*scale, save_mean_istd[0:C]=mean,[C:2C]=inv_std; updates running stats with momentum and the
 * unbiased variance.  clamp_eps=0: inv_std=(var+eps)^-1/2 (F.batch_norm); 1: clamp(var,eps)^-1/2
 * (sync_batchnorm/batchnorm.py:145). */
int seg_bn_finalize(const double* stats, double count, int C, const float* gamma, const float* beta, float eps,
                    float momentum, int clamp_eps, float* running_mean, float* running_var, float* scale_shift,
                    float* save_mean_istd, void* stream);
/* eval-mode (or frozen, BaseModel.freeze_bn): scale/shift from running stats; optionally also (mean, inv_std) */
int seg_bn_eval_scale_shift(int C, const float* gamma, const float* beta, const float* running_mean,
                            const float* running_var, float eps, float* scale_shift, float* save_mean_istd,
                            void* stream);
/* out = dropout(relu?(x*scale+shift (+res)))  — x,res,out bf16 [M][ld*]; drop_p = 0 disables dropout
 * (nn.ReLU(inplace) + residual add torchvision Bottleneck; nn.Dropout deeplabv3_plus.py:282,318).
 * drop_hw = 0: nn.Dropout (one draw per element); drop_hw = H*W: nn.Dropout2d (one draw per image and channel —
 * models/pspnet.py:22,68, upernet.py:22), rows being the pixels of consecutive images. */
int seg_bn_apply(const void* x, int ldx, const float* scale_shift, const void* res, int ldr, void* out, int ldo,
                 int64_t M, int C, int relu, float drop_p, uint64_t seed, const uint64_t* step_ctr, int drop_hw,
                 void* stream);
/* stats: fp64 [2C] from seg_conv2d_fwd / seg_dwconv3x3_fwd / seg_bn_stats over `count` elements (under SyncBN the world's
 * totals and the WORLD's element count).
 * seg_bn_finalize + seg_bn_apply in ONE launch (training mode): coefficients are derived from the batch sums inside the
 * kernel; save[2C] = (mean, 1/std) for the backward pass and the running statistics are written by one block row.
 * mask (optional, needs relu): the ReLU bit mask for the backward passes, uint8 [M][C/8] with its own pitch C/8 (independent
 * of ldo): bit j of mask[m][g] = (stored out[m][8g+j] > 0).
 * growth > 0: `stats` is a dense block's statistics table and x its channel prefix [0, C): fp64 records [sum(w), sum^2(w)]
 * back to back in channel order, the block input's (w = c0) first, then one per layer (w = growth), each written once by
 * its producer (and, under SyncBN, exchanged there).  Channel c's sums are read from its record.  growth == 0: stats is
 * [2C] (the launch without a table). */
int seg_bn_apply_train(const void* x, int ldx, const double* stats, double count, const float* gamma, const float* beta,
                       float eps, float momentum, int clamp_eps, float* running_mean, float* running_var, float* save,
                       const void* res, int ldr, void* out, int ldo, uint8_t* mask, int64_t M, int C, int relu, float drop_p,
                       uint64_t seed, const uint64_t* step_ctr, int drop_hw, int c0, int growth, void* stream);
/* device-side step counter (*ctr += inc): mixed into dropout seeds and SyncBN epochs so a captured CUDA graph of the
 * train step stays correct on every replay */
int seg_counter_add(uint64_t* ctr, uint64_t inc, void* stream);
/* backward, pass 1: sums[0:C] = sum(dz), sums[C:2C] = sum(dz*xhat), dz = dout * (out>0) * 1/(1-drop_p) if relu.  ONE
 * launch: every block adds its partial sums to one of seg_bn_bwd_reduce_slots() copies of `acc` (fp64 [slots][2C], ZERO at
 * launch; exact, order-independent accumulation; the copies spread the atomics); the
 * last block (ticket: one zeroed uint32) rounds them into sums[] and, if given, dbeta (=|+=) sums[0:C] and dgamma (=|+=)
 * sums[C:2C] — the parameter gradients from the LOCAL sums.  sync: SyncBN — that block then exchanges the sums with every
 * peer and leaves the WORLD's in sums[]; the consumer is seg_bn_bwd_apply with the world's count.
 * out == NULL with relu (both backward passes): the ReLU mask is recomputed from x with the forward's own coefficients
 * (sc = gamma/std, sh = fma(-mean, sc, beta)) instead of being read from the stored activation — valid for
 * conv -> BN(batch statistics) -> ReLU with no residual and no dropout; needs gamma and beta.
 * Dropout in the backward (all three backward entry points) needs relu != 0: the keep mask is read from the stored
 * activation (out > 0), which without the ReLU does not tell a dropped element from a negative one, so relu == 0 with
 * drop_p > 0 is rejected.
 * mask != NULL with relu (all three backward entry points): the ReLU / dropout keep mask is read from the bit mask that
 * seg_bn_apply_train wrote for this activation (1/16 of the bytes of out; out is then not read); it takes precedence over
 * out and over the recomputation. */
int seg_bn_bwd_reduce_slots(void);
int seg_bn_bwd_reduce(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                      const float* save_mean_istd, int64_t M, int C, int relu, float drop_p, float* sums, double* acc,
                      void* ticket, float* dgamma, float* dbeta, int accumulate, const float* gamma, const float* beta,
                      const seg_sync_desc* sync, void* stream);
/* backward, pass 2: dx = beta_dx*dx + gamma*istd*(dz - sums0/count - xhat*sums1/count); dres = beta_res*dres + dz (optional).
 * `sums` are the sums over `count` elements (under SyncBN the world's, from seg_bn_bwd_reduce).  beta_dx is 0 or 1; with 1
 * the sum is taken in fp32 and rounded to bf16 once (a pre-activation BN adding into its concat's gradient). */
int seg_bn_bwd_apply(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                     const float* save_mean_istd, const float* gamma, const float* sums, double count, int64_t M,
                     int C, int relu, float drop_p, void* dx, int lddx, void* dres, int lddres, float beta_res,
                     const float* beta, float beta_dx, void* stream);
/* BatchNorm backward in ONE cooperative launch = seg_bn_bwd_reduce + (SyncBN exchange) + seg_bn_bwd_apply: partial sums per
 * block -> grid barrier -> the cross-block sum spread over all blocks in fixed order (bit-reproducible) -> grid barrier ->
 * dx / dres.  dgamma / dbeta (optional) receive the parameter gradients from the LOCAL totals.  count_total = rows summed
 * over the world.  zero_sums != 0: frozen BatchNorm (BaseModel.freeze_bn): dx = gamma*istd*dz.  sync != NULL: one block
 * exchanges the totals with the SyncBN peers inside the kernel.  sums[2C] receives the totals dx is computed from (the WORLD's
 * under SyncBN).  Workspace from seg_bn_bwd_fused_workspace: rows (uninitialised floats) and tickets (uint32, ZERO at launch).
 * The grid is sized to be co-resident.  beta_dx (0 or 1): as seg_bn_bwd_apply's. */
int seg_bn_bwd_fused_workspace(int64_t M, int C, int64_t* rows_floats, int64_t* tickets);
int seg_bn_bwd_fused(const void* dout, int lddo, const void* out, int ldo, const uint8_t* mask, const void* x, int ldx,
                     const float* save_mean_istd, const float* gamma, const float* beta, double count_total, int64_t M,
                     int C, int relu, float drop_p, float* sums, float* rows, void* tickets, float* dgamma, float* dbeta,
                     int accumulate, void* dx, int lddx, void* dres, int lddres, float beta_res, int zero_sums,
                     const seg_sync_desc* sync, float beta_dx, void* stream);
/* parameter grads from the LOCAL sums: dbeta (=|+=) sums[0:C], dgamma (=|+=) sums[C:2C] */
int seg_bn_param_grad(const float* sums, int C, float* dgamma, float* dbeta, int accumulate, void* stream);

/* ---- pooling ---- */
/* nn.MaxPool2d(3, stride 2, pad 1) (deeplabv3_plus.py:24; resnet.py:151); idx (uint8) saves the arg-max tap */
int seg_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C, int P, int Q,
                         void* stream);
int seg_maxpool3x3s2_bwd(const void* dy, const uint8_t* idx, void* dx, int N, int H, int W, int C, int P, int Q,
                         void* stream);
/* nn.MaxPool2d(2, 2, return_indices=True) (segnet.py:30, called at segnet.py:87-103) and nn.MaxUnpool2d(2, 2) with
 * output_size = the pre-pool size (segnet.py:62, called at segnet.py:106-118).  H, W: the PRE-pool size (H, W >= 2);
 * P = H/2, Q = W/2 (floor: an odd last row / column is never read).  code[N,P,Q,C] (uint8) = 2r + s of the window
 * element chosen by ATen's rule (row-major scan, v > best || isnan(v): first maximum on ties, last NaN wins).  C % 8 == 0.
 * Selections of raw bf16 bits; every output element is written exactly once (no memset, no beta). */
int seg_maxpool2x2_fwd(const void* x, void* y, uint8_t* code, int N, int H, int W, int C, void* stream);
/* dx[N,H,W,C] = dy at the coded position of each window, 0 elsewhere and on a dropped odd row / column */
int seg_maxpool2x2_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream);
/* y[N,H,W,C] from x[N,P,Q,C]: x at the coded position, zeros in the other three and past rows 2P / columns 2Q */
int seg_maxunpool2x2_fwd(const void* x, const uint8_t* code, void* y, int N, int H, int W, int C, void* stream);
/* dx[N,P,Q,C] = dy[N,H,W,C] gathered at the coded positions */
int seg_maxunpool2x2_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream);
/* F.relu followed by nn.MaxPool2d(2, 2, ceil_mode=True) (FCN8's VGG trunk, fcn.py:20-22), over the raw conv output x[N,H,W,C]
 * (H, W >= 1): y[N,P,Q,C] = relu(window max), P = ceil(H/2), Q = ceil(W/2); the last windows of an odd H / W hold 1 or 2
 * elements.  code (uint8, y's shape) = 2r + s by ATen's rule where the window max is > 0 or NaN (there it equals the index
 * ATen's pool of relu(x) picks); a window whose max is <= 0 gets 4 + (2r + s).  C % 8 == 0, dense NHWC. */
int seg_relu_maxpool2x2_ceil_fwd(const void* x, void* y, uint8_t* code, int N, int H, int W, int C, void* stream);
/* dx[N,H,W,C] = dy at the coded position of windows whose max was > 0 or NaN, 0 everywhere else (relu + pool autograd) */
int seg_relu_maxpool2x2_ceil_bwd(const void* dy, const uint8_t* code, void* dx, int N, int H, int W, int C, void* stream);
/* nn.AvgPool2d(2, 2), floor mode (DenseNet's transition1): y [N][H/2][W/2][C] (channel pitch ldy: may be a concat slice)
 * = the mean of each 2x2 window, summed in fp32 and rounded once; a trailing odd row / column is dropped.  Backward:
 * dx = beta*dx + dy/4 over every element of dx (0 for the dropped row / column). */
int seg_avgpool2x2_fwd(const void* x, int ldx, void* y, int ldy, int N, int H, int W, int C, void* stream);
int seg_avgpool2x2_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int H, int W, int C, float beta, void* stream);
/* nn.AdaptiveAvgPool2d(bins) (deeplabv3_plus.py:274 bins=1; pspnet.py:26 bins 1,2,3,6): y[N,b,b,C] bf16 */
int seg_adaptive_avgpool_fwd(const void* x, int ldx, void* y, int N, int H, int W, int C, int bins, void* stream);
/* dx = beta*dx + scatter(dy) */
int seg_adaptive_avgpool_bwd(const void* dy, void* dx, int lddx, int N, int H, int W, int C, int bins, float beta,
                             void* stream);

/* ---- bilinear resize, F.interpolate(mode='bilinear') (deeplabv3_plus.py:291,328,361; pspnet.py:35,86,91) ---- */
/* NHWC bf16 -> NHWC bf16 (channel-slice output allowed) */
int seg_bilinear_fwd(const void* x, int ldx, void* y, int ldy, int N, int Hi, int Wi, int Ho, int Wo, int C,
                     int align_corners, void* stream);
/* dx = beta*dx + bilinear^T(dy) */
int seg_bilinear_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                     int align_corners, float beta, void* stream);
/* final logits: NHWC fp32 [N,Hi,Wi,C] -> NCHW fp32 [N,C,Ho,Wo] (the tensor the reference returns, deeplabv3_plus.py:361) */
int seg_bilinear_logits_fwd(const float* x, float* y_nchw, int N, int Hi, int Wi, int Ho, int Wo, int C,
                            int align_corners, void* stream);
/* NCHW fp32 grad -> NHWC bf16 grad at the low resolution */
int seg_bilinear_logits_bwd(const float* dy_nchw, void* dx, int lddx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                            int align_corners, void* stream);

/* ---- pixel shuffle, nn.PixelShuffle(r) (duc_hdc.py:22,30) ---- */
/* NHWC bf16 x [N,H,W,r*r*C] (pitch ldx) -> NHWC bf16 y [N,Ho,Wo,C] (pitch ldy; a channel slice is allowed), cropped to
 * Ho <= r*H, Wo <= r*W: y[n,oy,ox,c] = x[n, oy/r, ox/r, c*r*r + (oy%r)*r + ox%r].  Replaces the DUC block's shuffle and the
 * decoder's crop x[:, :, :Hl, :Wl] (duc_hdc.py:30,206), writing straight into the decoder's concat buffer.  Exact. */
int seg_pixel_shuffle_fwd(const void* x, int ldx, void* y, int ldy, int N, int H, int W, int C, int r, int Ho, int Wo,
                          void* stream);
/* dx = beta*dx + shuffle^T(dy) over all r*r*C channels of dx; source positions the crop dropped get zero */
int seg_pixel_shuffle_bwd(const void* dy, int lddy, void* dx, int lddx, int N, int H, int W, int C, int r, int Ho, int Wo,
                          float beta, void* stream);
/* final logits of DeepLab_DUC_HDC (duc_hdc.py:233): NHWC bf16 [N,h,w,r*r*C] (pitch ldx) -> NCHW fp32 [N,C,r*h,r*w] */
int seg_pixel_shuffle_logits_fwd(const void* x, int ldx, float* y_nchw, int N, int h, int w, int C, int r, void* stream);
/* NCHW fp32 grad -> NHWC bf16 grad [N,h,w,lddx] (channels r*r*C .. lddx-1 zero) */
int seg_pixel_shuffle_logits_bwd(const float* dy_nchw, void* dx, int lddx, int N, int h, int w, int C, int r, void* stream);

/* ---- per-pixel loss ---- */
/* Cross-entropy, class-weighted cross-entropy and focal loss, one family of entry points with the loss picked by `kind`:
 * CrossEntropyLoss2d(weight, reduction) (utils/losses.py:24-31), FocalLoss(gamma, alpha, size_average) (:52-65) and the
 * CE half of CE_DiceLoss(weight, reduction) (:67-77).  With nll = lse(z) - z_t at a pixel labelled t != ignore_index and
 * w = weight (fp32 [C], finite and >= 0; NULL = all ones):
 *   SEG_LOSS_CE     per-pixel loss nll;                             accum[1] += 1 per valid pixel
 *   SEG_LOSS_WCE    per-pixel loss L = w_t*nll;                     accum[1] += w_t per valid pixel
 *   SEG_LOSS_FOCAL  per-pixel loss (1-pt)^gamma * L, pt = exp(-L);  accum[1] += 1 per pixel, ignored ones included
 * (the reference's .mean() over the unreduced loss counts ignored pixels).  accum is fp64 [2], zeroed by the caller:
 * accum[0] += the per-pixel losses, accum[1] += the denominator; it may be summed over ranks before the finalize and the
 * backward.  SEG_LOSS_CE takes weight = NULL and mean = 1, an error otherwise; gamma (finite, >= 0) is read by
 * SEG_LOSS_FOCAL only.  mean = 1: loss = accum[0]/accum[1], or 0 when accum[1] == 0 (ATen gives NaN there); mean = 0
 * ('sum', size_average=False): loss = accum[0].
 * Backward: dL/dz_c = g * w_t (p_c - delta_ct) * F'(L), 0 for ignored pixels, with F' = 1 except for focal, where
 * F' = u^gamma (1 + gamma r), u = -expm1(-L), r = L/expm1(L) (1 at L = 0), so 0 <= F' <= 1 + gamma and a pixel whose pt
 * rounds to 1 gets the finite limit (0 for gamma > 0; the reference's autograd gives NaN for 0 < gamma < 1).
 * g = gscale/accum[1] (0 when accum[1] == 0; SEG_LOSS_CE: gscale/max(accum[1], 1), divided in fp32) or gscale for a sum;
 * gscale = the upstream gradient (fp32 scalar on the device, NULL = 1). */
#define SEG_LOSS_CE 0
#define SEG_LOSS_WCE 1
#define SEG_LOSS_FOCAL 2
/* logits NCHW fp32, target int64 [N,H,W]; dlogits NCHW fp32 */
int seg_loss_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                      const float* weight, int kind, float gamma, double* accum, void* stream);
int seg_loss_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                      const float* weight, int kind, float gamma, int mean, const double* accum, const float* gscale,
                      float* dlogits, void* stream);
/* loss (fp32 scalar on the device) from accum, as above */
int seg_loss_finalize(const double* accum, int mean, float* loss, void* stream);
/* The same losses fused with the bilinear upsample: low-res NHWC fp32 logits [N,Hi,Wi,C] (C <= 160), upsampled as
 * deeplabv3_plus.py:361 / pspnet.py:86 do, + log-softmax + NLL, with no full-resolution logits in HBM.
 * argmax != NULL: also the arg-max label map (int32 [N,Ho,Wo], lowest index wins ties).
 * counters != NULL: also the main head's eval_metrics (trainer.py:62,84 -> utils/metrics.py:59-67) in the same launch, so
 * neither training nor validation needs the full-resolution logits for pixel accuracy and mIoU.  counters: int64
 * [2 + 3*C] = correct, labeled, area_inter[C], area_pred[C], area_lab[C], the layout of seg_eval_metrics_nchw with
 * num_class = C; ADDED to (not zeroed), so a running total needs no extra launch.  The prediction is the arg-max of the
 * interpolated fp32 logits seg_bilinear_logits_fwd produces (lowest index wins ties); a pixel is labeled when
 * 0 <= target < C, independently of ignore_index.  Integer counters: deterministic.
 * Backward: d(logits_lo) is accumulated in 64-bit fixed point in the int64 scratch dlo_fixed [N,Hi,Wi,C] (zeroed here;
 * order-independent, hence bit-reproducible) with the scale derived from the bound |g| * max(w) * (1 + gamma) (the
 * factors the kind has), converted to fp32 dlo_f32 [N,Hi,Wi,C], then written as bf16 NHWC with pitch lddx (channels
 * C..lddx-1 zero) when dx != NULL. */
int seg_upsample_loss_fwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                          int align_corners, int64_t ignore_index, const float* weight, int kind, float gamma, double* accum,
                          int32_t* argmax, int64_t* counters, void* stream);
int seg_upsample_loss_bwd(const float* logits_lo, const int64_t* target, int N, int Hi, int Wi, int Ho, int Wo, int C,
                          int align_corners, int64_t ignore_index, const float* weight, int kind, float gamma, int mean,
                          const double* accum, const float* gscale, float* dlo_f32, void* dlo_fixed, void* dx, int lddx,
                          void* stream);
/* The same losses fused with the pixel shuffle of DeepLab_DUC_HDC's output (duc_hdc.py:233 + trainer.py:60): the logits
 * are the nn.PixelShuffle(r) view of the low-res NHWC bf16 map [N,h,w,r*r*C] (pitch ldlo, C <= 160), read in place, and
 * target is int64 [N, r*h, r*w].  kind, weight, gamma, mean, accum, gscale and counters as for seg_upsample_loss_*; the
 * prediction is the arg-max of the values seg_pixel_shuffle_logits_fwd produces (lowest index wins ties).
 * Backward: every low-res element belongs to exactly one pixel, so dx (bf16 [N,h,w,lddx], channels r*r*C .. lddx-1 zero) is
 * written directly, once per element: deterministic, no scratch. */
int seg_shuffle_loss_fwd(const void* logits_lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r,
                         int64_t ignore_index, const float* weight, int kind, float gamma, double* accum, int64_t* counters,
                         void* stream);
int seg_shuffle_loss_bwd(const void* logits_lo, int ldlo, const int64_t* target, int N, int h, int w, int C, int r,
                         int64_t ignore_index, const float* weight, int kind, float gamma, int mean, const double* accum,
                         const float* gscale, void* dx, int lddx, void* stream);
/* The same losses on logits that are already at the output resolution: UNetResnet's conv7 output (unet.py:204 +
 * trainer.py:60), NHWC fp32 [N,H,W,C] with pitch ld (C <= 160), read in place; target int64 [N,H,W].  kind, weight, gamma,
 * mean, accum, gscale and counters as for seg_shuffle_loss_* (these are its r = 1 instance over an fp32 map).
 * Backward: dx (bf16 [N,H,W,lddx], channels C .. lddx-1 zero) written once per element: deterministic, no atomics. */
int seg_nhwc_loss_fwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                      const float* weight, int kind, float gamma, double* accum, int64_t* counters, void* stream);
int seg_nhwc_loss_bwd(const float* logits, int ld, const int64_t* target, int N, int H, int W, int C, int64_t ignore_index,
                      const float* weight, int kind, float gamma, int mean, const double* accum, const float* gscale, void* dx,
                      int lddx, void* stream);
/* DiceLoss (utils/losses.py:33-50): softmax over C, intersection with the one-hot target, whole-batch ratio.
 * accum (fp64 [2], zeroed by the caller) receives (sum p[target], #pixels); loss = 1 - (2I+s)/(2*#pixels+s).
 * The caller applies the reference's in-place target fix-up (losses.py:40-42) before calling. */
int seg_dice_nchw_fwd(const float* logits, const int64_t* target, int N, int C, int H, int W, float smooth,
                      double* accum, float* loss, void* stream);
/* dlogits = beta*dlogits + gscale * d(dice)/d(logits) */
int seg_dice_nchw_bwd(const float* logits, const int64_t* target, int N, int C, int H, int W, const double* accum,
                      float smooth, const float* gscale, float* dlogits, float beta, void* stream);
/* LovaszSoftmax (utils/losses.py:79-89 -> utils/lovasz_losses.py:153-199,19-31; classes='present', per_image=False):
 * all present classes at once on the device — 64-bit keys [class rank|~error bits|fg|pixel], one LSD radix sort,
 * tiled scans, Jaccard differences — instead of the reference's per-class sort + host sync.
 *   seg_lovasz_count: counts (int32 [C+1], zeroed here): valid pixels per class, counts[C] = all valid pixels.
 *   The caller reads counts back (the one host sync; the reference does C of them), then passes P = counts[C],
 *   n_present = #{c: counts[c] > 0}, two uint64 key buffers of P*n_present elements and a byte workspace.
 *   seg_lovasz_softmax_nchw: loss (fp32 scalar) and dlogits = d loss / d logits (NCHW fp32; also scratch).
 *   Exactly tied errors take ranks in flat pixel order, and the loss is folded in a fixed order: two calls on the same
 *   inputs give bit-identical results. */
int seg_lovasz_count(const int64_t* target, int64_t npix, int C, int64_t ignore_index, int32_t* counts, void* stream);
int64_t seg_lovasz_workspace_bytes(int64_t P, int n_present, int C);
int seg_lovasz_softmax_nchw(const float* logits, const int64_t* target, int N, int C, int H, int W, int64_t ignore_index,
                            const int32_t* counts, int64_t P, int n_present, void* keys0, void* keys1, void* workspace,
                            float* loss, float* dlogits, void* stream);
/* eval_metrics (utils/metrics.py:42-67: argmax, batch_pix_accuracy :41-45, batch_intersection_union :47-57) in one
 * pass over the NCHW fp32 logits.  out: int64 [2 + 3*num_class] (zeroed here) = correct, labeled, area_inter[K],
 * area_pred[K], area_lab[K]; union = pred + lab - inter.  Integer counters: bit-exact with the reference. */
int seg_eval_metrics_nchw(const float* logits, const int64_t* target, int N, int C, int H, int W, int num_class,
                          int64_t* out, void* stream);

/* ---- misc ---- */
/* standalone ReLU on NHWC bf16 (F.relu, deeplabv3_plus.py:210) and its backward dx = beta*dx + dy*(y>0) */
int seg_relu_fwd(const void* x, int ldx, void* y, int ldy, int64_t M, int C, void* stream);
int seg_relu_bwd(const void* dy, int lddy, const void* y, int ldy, void* dx, int lddx, int64_t M, int C, float beta,
                 void* stream);
/* F.relu + nn.Dropout(drop_p) in training (FCN8's conv6 / conv7, fcn.py:49-51): y = relu(x) * keep / (1 - drop_p) with keep =
 * hash_uniform(seed + step_ctr * golden, row * C + c) >= drop_p (bn_apply's stream; step_ctr: device counter or NULL).
 * drop_p = 0 is F.relu.  Backward: dx = beta*dx + (y > 0 ? dy / (1 - drop_p) : 0).  C and pitches % 8 == 0. */
int seg_relu_dropout_fwd(const void* x, int ldx, void* y, int ldy, int64_t M, int C, float drop_p, uint64_t seed,
                         const uint64_t* step_ctr, void* stream);
int seg_relu_dropout_bwd(const void* dy, int lddy, const void* y, int ldy, void* dx, int lddx, int64_t M, int C, float drop_p,
                         float beta, void* stream);
/* ---- class-map transposed convolution (FCN8's frozen score upsamplers, fcn.py:57-97) ----
 * ConvTranspose2d(C, C, k = 2s, stride s, padding 0, no bias) of x[N,h,w,C] (bf16, pitch ldx) -> a [N,(h+1)s,(w+1)s,C] map of
 * which only the window rows [y0, y0+Ho) x cols [x0, x0+Wo) are computed.  1 <= C <= 160, 1 <= s <= 8.  Tensor cores
 * (mma.sync bf16, fp32 accumulation); no atomics: every output element is one thread's fixed-order sum.  Only the C class
 * lanes of pitched operands are read or written.  bf16 operand pitches must be even and their base addresses 4-byte aligned.
 * seg_score_pack: weight w[C][C][k][k] (fp32, any dense values) -> the kernels' bf16 operand (packed_elems bf16 elements);
 * bwd = 0 packs the forward's four-tap parity-class GEMMs, 1 the data gradient's. */
int64_t seg_score_packed_elems(int C, int s);
int seg_score_pack(const float* w, void* packed, int C, int s, int bwd, void* stream);
/* y[n,i,j,c] = convT(x)[n, y0+i, x0+j, c] (+ alpha * skip[n, sy0+i, sx0+j, c] + bias[c] when skip is non-NULL; bias may be
 * NULL).  y_dtype SEG_DT_BF16 / SEG_DT_F32, pitch ldy. */
int seg_score_upsample_fwd(const void* x, int ldx, int N, int h, int w, int C, int s, const void* packed, void* y, int ldy,
                           int y_dtype, int y0, int x0, int Ho, int Wo, const void* skip, int lds, int Hs, int Ws, int sy0, int sx0,
                           float alpha, const float* bias, void* stream);
/* dx[N,h,w,C] (bf16, pitch ldx, written) = the data gradient of the windowed forward for dy[N,Ho,Wo,C] (bf16, pitch lddy) */
int seg_score_upsample_bwd(const void* dy, int lddy, int N, int h, int w, int C, int s, const void* packed_bwd, void* dx, int ldx,
                           int y0, int x0, int Ho, int Wo, void* stream);
/* dskip[N,Hs,Ws,C] (bf16, pitch ldd) = alpha * dy[n, a-sy0, b-sx0, c] inside the window, 0 elsewhere (the skip's gradient) */
int seg_score_skip_bwd(const void* dy, int lddy, int Ho, int Wo, void* dskip, int ldd, int N, int Hs, int Ws, int C, int sy0,
                       int sx0, float alpha, void* stream);
int seg_nhwc_to_nchw_f32(const void* x, int ldx, int x_dtype, float* y, int N, int H, int W, int C, void* stream);
/* y[M][ldy] (bf16) = beta*y + x[M][ldx] (bf16) */
int seg_axpby_bf16(const void* x, int ldx, void* y, int ldy, int64_t M, int C, float beta, void* stream);
/* multi-tensor SGD step (torch.optim.SGD semantics: wd, momentum, dampening 0, no nesterov;
 * base/base_trainer.py:57): n tensors described by device arrays of pointers/sizes; one block row per tensor, so
 * n <= 65535 (a larger n is refused before any launch) */
int seg_sgd_step(float* const* params, float* const* grads, float* const* momentum_bufs, const int64_t* sizes,
                 const float* lrs, int n, float momentum, float weight_decay, int first_step, float grad_scale,
                 void* stream);
/* same step with (momentum, weight_decay) read from DEVICE memory hyper[0..1]: a momentum schedule
 * (OneCycle, utils/lr_scheduler.py:24-59) stays effective when the step is replayed from a CUDA graph */
int seg_sgd_step_dev(float* const* params, float* const* grads, float* const* momentum_bufs, const int64_t* sizes,
                     const float* lrs, int n, const float* hyper, int first_step, float grad_scale, void* stream);
/* ---- input pipeline tail (SURVEY.md §8f row 2): pad + crop + horizontal flip + ToTensor + Normalize on the device ----
 * Replaces, for a batch that crossed PCIe as uint8, base/base_dataset.py:93-123 (copyMakeBorder value 0, crop at
 * (start_h, start_w), np.fliplr) and :129-136 (ToTensor, Normalize, label -> int64).  `arena` holds the B images
 * (HWC uint8, h x w x 3, any sizes) and labels (h x w, uint8 or int32) back to back; `table[b]` says where.  The
 * random draws (crop origin, flip) stay on the host so a seeded run makes the reference's draws; mean3/std3 are HOST
 * pointers.  out_nchw fp32 [B,3,crop_h,crop_w], out_labels int64 [B,crop_h,crop_w] (NULL: images only).
 * Bit-exact: fp32 (u8/255 - mean)/std with IEEE divisions, the operations torchvision performs. */
typedef struct seg_aug_entry {
  int64_t img_off;   /* byte offset of the image in the arena */
  int64_t lbl_off;   /* byte offset of the label map, or -1 */
  int32_t h, w;      /* image size before padding */
  int32_t y0, x0;    /* crop origin in the (bottom/right zero-padded) image */
  int32_t flip;      /* 1: flip the crop horizontally */
  int32_t lbl_bytes; /* 1 (uint8) or 4 (int32) */
} seg_aug_entry;
int seg_aug_entry_bytes(void);
int seg_augment_batch_u8(const uint8_t* arena, const seg_aug_entry* table, int B, int crop_h, int crop_w, const float* mean3,
                         const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
/* The same tail with the random-scale resize of base/base_dataset.py:66-75 fused in front: `arena` holds the RAW samples
 * (src_h x src_w), each output pixel interpolates from the raw image (cv2.resize INTER_LINEAR arithmetic of OpenCV's own
 * float path, truncated to uint8 as `np.uint8(image)` does at base_dataset.py:133; INTER_NEAREST for the label) at the
 * position the crop / flip selects in the resized h x w image.  scale_x = 1.0 / ((double)w / src_w), scale_y likewise —
 * computed by the HOST in float64 exactly as cv::resize does. */
typedef struct seg_aug_scale_entry {
  int64_t img_off;        /* byte offset of the raw image (HWC uint8) in the arena */
  int64_t lbl_off;        /* byte offset of the raw label map, or -1 */
  double scale_x, scale_y;
  int32_t src_h, src_w;   /* raw sample size */
  int32_t h, w;           /* size after the resize (before padding) */
  int32_t y0, x0;         /* crop origin in the (bottom/right zero-padded) resized image */
  int32_t flip;
  int32_t lbl_bytes;      /* 1 (uint8) or 4 (int32) */
} seg_aug_scale_entry;
int seg_aug_scale_entry_bytes(void);
int seg_augment_scale_batch_u8(const uint8_t* arena, const seg_aug_scale_entry* table, int B, int crop_h, int crop_w,
                               const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
/* The validation tail of base/base_dataset.py:40-61 (resize so the short side is the crop, centre crop, np.uint8,
 * ToTensor, Normalize) with the same records: the image arithmetic is seg_augment_scale_batch_u8's, flip = 0 and (y0, x0)
 * the centre origin.  The label follows PIL's Image.resize(NEAREST) instead of cv2's INTER_NEAREST: Pillow accumulates its
 * float64 source coordinate pixel by pixel, so the host computes the indices and appends them to the label map in the
 * arena, at lbl_off + (src_h * src_w * lbl_bytes rounded up to 4): int32 x index [w], then int32 y index [h]. */
int seg_augment_val_batch_u8(const uint8_t* arena, const seg_aug_scale_entry* table, int B, int crop_h, int crop_w,
                             const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
/* the same with the rotation of base/base_dataset.py:77-83
 * between the resize and the tail.  (a11 a12 b1; a21 a22 b2) = the INVERSE of cv2.getRotationMatrix2D((w/2, h/2), angle, 1)
 * computed by the host in float64 exactly as cv::warpAffine does (oracle/data.py::cv_warp_affine); identity = no rotation. */
typedef struct seg_aug_full_entry {
  int64_t img_off;
  int64_t lbl_off;
  double scale_x, scale_y;
  double a11, a12, b1, a21, a22, b2;
  int32_t src_h, src_w;
  int32_t h, w;
  int32_t y0, x0;
  int32_t flip;
  int32_t lbl_bytes;
} seg_aug_full_entry;
int seg_aug_full_entry_bytes(void);
int seg_augment_full_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, int B, int crop_h, int crop_w,
                              const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
/* the same with the Gaussian blur of base/base_dataset.py:114-119 after the flip, on the float crop before np.uint8:
 * cv2.GaussianBlur(k = 3, BORDER_REFLECT_101 at the crop's border), OpenCV's separable fp32 filter (row pass, then column
 * pass, no fma).  blur_taps: DEVICE memory, B x (centre tap, side tap) float32 = getGaussianKernel(3, sigma) in float64
 * rounded to float32, computed by the host; (1, 0) = k = 1 (no blur), bit-identical to seg_augment_full_batch_u8. */
int seg_augment_full_blur_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, const float* blur_taps, int B, int crop_h,
                                   int crop_w, const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels,
                                   void* stream);
/* ---- label maps: the *_mapped twins of the five augmentation entry points take the same arguments and records and also
 * accept lbl_bytes = 1 | SEG_AUG_LABEL_MAP: the sample's uint8 label map is followed, at the next 4-byte boundary, by 256
 * int32 entries `map`, and every label read from the raw map is map[raw] (a dataset's id -> train-id table, applied where
 * the reference applies it: before the resize, rotation and padding).  Fill values — the zero padding of copyMakeBorder and
 * warpAffine's constant-0 border — are post-map values and stay 0.  The validation kernel's PIL index tables follow the
 * map.  The flag is valid with 1-byte labels only (the host packer refuses anything else); records without it read their
 * labels exactly as the entry points above do. */
#define SEG_AUG_LABEL_MAP 256
int seg_augment_mapped_batch_u8(const uint8_t* arena, const seg_aug_entry* table, int B, int crop_h, int crop_w, const float* mean3,
                                const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
int seg_augment_scale_mapped_batch_u8(const uint8_t* arena, const seg_aug_scale_entry* table, int B, int crop_h, int crop_w,
                                      const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
int seg_augment_val_mapped_batch_u8(const uint8_t* arena, const seg_aug_scale_entry* table, int B, int crop_h, int crop_w,
                                    const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
int seg_augment_full_mapped_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, int B, int crop_h, int crop_w,
                                     const float* mean3, const float* std3, float* out_nchw, int64_t* out_labels, void* stream);
int seg_augment_full_blur_mapped_batch_u8(const uint8_t* arena, const seg_aug_full_entry* table, const float* blur_taps, int B,
                                          int crop_h, int crop_w, const float* mean3, const float* std3, float* out_nchw,
                                          int64_t* out_labels, void* stream);
/* ---- inference-side resampling (SURVEY.md §8f row 3; inference.py:26-79), fp32 NCHW score maps, `planes` = N*C ----
 * resize: dst = beta*dst + alpha*flip_x?(bilinear resize of src to Hd x Wd).  mode 0 / 1 = ATen bilinear with
 * align_corners False / True (1 = nn.Upsample(align_corners=True), inference.py:60; same size + flip_x = tensor.flip(-1),
 * :48,:70); mode 2 = scipy.ndimage.zoom(order=1, prefilter=False) (inference.py:65): float64 coordinates and the
 * library's mode='constant' rule that zeroes an output whose coordinate rounds past the last input sample. */
int seg_resize_nchw_f32(const float* src, int64_t planes, int Hs, int Ws, float* dst, int Hd, int Wd, int mode, int flip_x,
                        float alpha, float beta, void* stream);
/* dst[:, y0:y0+h, x0:x0+w] += alpha * flip_x?(src)[:, :h, :w]  — sliding-window accumulation (inference.py:49-53) */
int seg_window_add_nchw_f32(const float* src, int64_t planes, int Hs, int Ws, float* dst, int Hd, int Wd, int y0, int x0, int h,
                            int w, int flip_x, float alpha, void* stream);
/* x[p] /= count  (count fp32 [H,W]; inference.py:55) */
int seg_div_by_count_nchw_f32(float* x, int64_t planes, int H, int W, const float* count_hw, void* stream);
/* labels int64 [N,H,W] = softmax(dim=C).argmax of inference.py:156 without the softmax pass: 0 where a pixel's scores hold
 * a NaN or +inf (the reference's softmax column is all NaN), else the first maximum.  Two finite top scores closer than a
 * float64 softmax resolves (both under ~2e-9) may tie in the reference, which keeps the first; here the larger wins. */
int seg_argmax_nchw_f32(const float* scores, int N, int C, int H, int W, int64_t* labels, void* stream);
/* ---- SyncBN one-shot exchange over NVLink peer memory (replaces ReduceAddCoalesced + Broadcast,
 *      sync_batchnorm/batchnorm.py:117,120 and the thread pipes of sync_batchnorm/comm.py) ----
 * Each rank owns a symmetric buffer of seg_comm_buffer_bytes(world, n_max) bytes (seg_comm_alloc, zeroed), exports it
 * with seg_comm_ipc_get, opens its peers' with seg_comm_ipc_open, and passes the world's pointers (indexed by rank;
 * its own pointer at [rank]) as a DEVICE array in a seg_sync_desc.  seg_syncbn_exchange(sync, vals[n]) leaves the
 * rank-ordered sum over all ranks in vals on every rank (bit-identical everywhere): one block running the same exchange as
 * the statistics producers (csrc/seg_sync.cuh), n <= n_max, world <= 64, spin wait bounded by sync->timeout_clocks.  All
 * ranks must issue the same sequence of exchanges, in-kernel and stand-alone alike; the sequence number lives in the
 * symmetric buffer on the device, so the call can be captured in a CUDA graph. */
size_t seg_comm_buffer_bytes(int world, int n_max);
int seg_comm_alloc(size_t bytes, void** ptr);
int seg_comm_free(void* ptr);
int seg_comm_ipc_get(void* ptr, void* handle64);
int seg_comm_ipc_open(const void* handle64, void** ptr);
int seg_comm_ipc_close(void* ptr);
int seg_syncbn_exchange(const seg_sync_desc* sync, float* vals, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEG_B200_H */
