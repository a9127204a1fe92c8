/* libosvos_b200 - C ABI of the H100-native OSVOS hot path.
 *
 * The reference (kmaninis/OSVOS-PyTorch) has no FFI of its own: its hot path is
 * Python calling torch.nn modules (SURVEY.md section 8b).  This header is the native
 * boundary introduced underneath the unchanged Python API; each entry point
 * names the reference call it replaces (file:line relative to the reference
 * repo).  The binding a maintainer adds on the reference side is the ctypes
 * stub shown in INTEGRATION.md (osvos_pytorch_b200/_native.py is that stub).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name says host;
 *   - no allocation inside: outputs and workspaces are caller-provided;
 *   - every function enqueues on `stream` and returns immediately with an
 *     OSVOS_* status (0 = ok); no exceptions cross the boundary;
 *     osvos_last_error() returns a thread-local message for the last failure;
 *   - "act" = activation tensor, NHWC, stored as split bf16: value ~= hi + lo,
 *     two planes of shape [N,H,W,C] (C a multiple of 64 for 3x3 conv inputs,
 *     16 for the side-branch gradient).  In OSVOS_FLAG_FAST mode only `hi`
 *     exists (lo pointers may be NULL) and a single tensor-core pass is issued;
 *     the default (exact) mode issues the three passes hi*hi + hi*lo + lo*hi
 *     with fp32 accumulation in registers.
 */
#ifndef OSVOS_B200_H_
#define OSVOS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OSVOS_B200_VERSION 100 /* major*10000 + minor*100 + patch */

#if defined(__GNUC__)
#define OSVOS_API __attribute__((visibility("default")))
#else
#define OSVOS_API
#endif

enum {
  OSVOS_OK = 0,
  OSVOS_ERR_INVALID_ARGUMENT = 1,
  OSVOS_ERR_CUDA = 2,
  OSVOS_ERR_UNSUPPORTED = 3
};

enum {
  OSVOS_FLAG_RELU = 1,       /* fwd: y = max(y, 0)            (networks/vgg_osvos.py:143) */
  OSVOS_FLAG_FAST = 2,       /* single-pass bf16 operands (hi planes only)               */
  OSVOS_FLAG_RELU_MASK = 4,  /* dgrad: dx *= (mask_hi > 0)    (autograd of :143)          */
  OSVOS_FLAG_ACCUMULATE = 8, /* add into the existing output instead of overwriting it    */
  OSVOS_FLAG_DEFER_FINISH = 16, /* osvos_conv3x3_wgrad: accumulate into a caller-zeroed workspace only; the
                                  workspace -> OIHW step is done later by osvos_wgrad_finish for many layers */
  OSVOS_FLAG_DETERMINISTIC = 32, /* reduce floats in an order that does not depend on scheduling: partial results go to
                                   per-block / per-tile slots written with plain stores, which are added in a fixed order
                                   (see "Deterministic forms" below).  Without it the kernels add with atomics. */
  OSVOS_FLAG_VOID_LABELS = 64   /* class-balanced BCE (osvos_cbce_fwd, osvos_tail_fwd, osvos_tail_loss_bwd): a label
                                   y < 0 marks a void pixel, counted in neither class and given zero gradient; N is
                                   then the number of pixels with y >= 0, and N == 0 gives loss 0 and gradient 0 */
};

typedef void* osvos_stream_t; /* cudaStream_t */

OSVOS_API int osvos_version(void);
OSVOS_API const char* osvos_last_error(void);
/* Programmatic dependent launch for the kernels enqueued from now on: 1 on, 0 off, -1 = the process default
 * (environment OSVOS_PDL, off).  Returns the previous setting.  Every kernel of the library waits
 * (griddepcontrol.wait) before it first touches memory another kernel may have written, so the switch only decides
 * whether a kernel's prologue may overlap its predecessor's tail.  A captured CUDA graph keeps what it was captured with. */
OSVOS_API int osvos_set_pdl(int mode);

/* ---- weight packing ------------------------------------------------------
 * nn.Conv2d weight, OIHW fp32 (networks/vgg_osvos.py:41,142) -> split-bf16
 * K-major GEMM operand [plane(hi,lo)][tap = 3*r+s][rows][cols]:
 *   transpose_flip == 0 (forward):  rows = Cout, cols = Cin, element = w[co][ci][r][s]
 *   transpose_flip == 1 (dgrad):    rows = Cin,  cols = Cout, element = w[co][ci][2-r][2-s]
 * cols is padded up to a multiple of `col_pad` (64 or 16) with zeros.
 * Bytes needed: osvos_packed_weight_bytes(rows, cols_padded).                      */
OSVOS_API size_t osvos_packed_weight_bytes(int rows, int cols_padded);
OSVOS_API int osvos_pack_conv3x3_weights(const float* w_oihw, void* packed, int cout, int cin, int transpose_flip,
                               int col_pad, osvos_stream_t stream);

/* ---- layout conversion (test / boundary helpers) -------------------------- */
OSVOS_API int osvos_nchw_to_act(const float* x_nchw, void* act_hi, void* act_lo, int n, int c, int h, int w,
                      osvos_stream_t stream);
OSVOS_API int osvos_act_to_nchw(const void* act_hi, const void* act_lo, float* y_nchw, int n, int c, int h, int w,
                      osvos_stream_t stream);

/* ---- conv1_1: nn.Conv2d(3, 64, 3, padding=1) + ReLU ------------------------
 * Replaces stages[0][0..1] (networks/vgg_osvos.py:61,142-143).  Reads the
 * caller's NCHW fp32 frame directly (no layout pass), wgmma over split-bf16
 * operands (conv_first_tc.cu), writes an act [N,H,W,64].                       */
OSVOS_API int osvos_conv_first_fwd(const float* x_nchw, const float* w_oihw, const float* bias, void* y_hi, void* y_lo,
                         int n, int h, int w, int flags, osvos_stream_t stream);

/* ---- 3x3 convolution, padding 1, stride 1, as a wgmma implicit GEMM -------
 * Replaces every other nn.Conv2d(k=3, p=1) on the path: the 12 remaining trunk
 * convs (+ReLU, networks/vgg_osvos.py:142-143, run at :61,:66) and the four
 * side_prep convs (:41, run at :67, no ReLU); with transpose-flipped packed
 * weights it is also their data gradient (autograd of the same lines).
 *   M = N*H*W pixels (tiles of 16 rows x 8 px), N = cout, K = 9 * cin.         */
typedef struct {
  const void* x_hi;      /* act [n,h,w,cin]                                     */
  const void* x_lo;      /* NULL in FAST mode                                   */
  const void* w_packed;  /* osvos_pack_conv3x3_weights output, rows = cout      */
  const float* bias;     /* [cout] or NULL                                      */
  void* y_hi;            /* act [n,h,w,cout] or NULL (cout >= 64 only)          */
  void* y_lo;            /* NULL in FAST mode / when y_hi is NULL               */
  float* y_f32;          /* optional fp32 NHWC copy of the output [n,h,w,cout]  */
  const void* mask_hi;   /* RELU_MASK (cout >= 64 only): act hi plane [n,h,w,cout] of the fwd output this gradient
                            flows into */
  /* side_prep only (cout == 16, whose outputs are y_f32 and / or pq): fused 1x1 projections of the 16 features
   *   pq[px][0] = <y, proj_w[0:16]>  + proj_b[0]   score_dsn (networks/vgg_osvos.py:44,69)
   *   pq[px][1] = <y, proj_w[16:32]>               this scale's slice of fuse (:54,72)  */
  const float* proj_w;   /* [32] or NULL */
  const float* proj_b;   /* [1]  or NULL */
  float* pq;             /* [n,h,w,2] or NULL */
  /* fused MaxPool2d(2,2,ceil_mode=True) of the output (networks/vgg_osvos.py:140): act
   * [n, ceil(h/2), ceil(w/2), cout], written in addition to y (cout >= 64 only) */
  void* pool_hi;
  void* pool_lo;
  /* fused per-channel sum of the (masked) output over all pixels = bias gradient of the layer this
   * gradient belongs to; [cout] fp32, ACCUMULATED with atomics (caller zeroes); cout >= 64 only.
   * With OSVOS_FLAG_DETERMINISTIC: partial rows [osvos_conv3x3_colsum_rows(n, h, w)][cout] instead, each written once
   * (no zeroing needed); osvos_reduce_rows adds them in order. */
  float* colsum;
  int n, h, w, cin, cout;
  int flags;
} osvos_conv3x3_args;
OSVOS_API int osvos_conv3x3(const osvos_conv3x3_args* args /* host */, osvos_stream_t stream);

/* ---- folded side branch (inference and training) ---------------------------------------
 * side_prep has no ReLU (networks/vgg_osvos.py:67), so side_prep followed by score_dsn and this scale's slice of
 * fuse (:44,54,69,72) is ONE 3x3 convolution C -> 2:  W'[o][ci][tap] = sum_co proj_w[16 o + co] * side_w[co][ci][tap],
 * b'[o] = (o == 0 ? proj_b : 0) + sum_co proj_w[16 o + co] * side_b[co].  osvos_fold_side_weights_multi (below) writes
 * W' in the packed operand layout (osvos_packed_weight_bytes(2, cin) bytes) and b' (2 floats); osvos_conv3x3 with
 * cout == 2, w_packed = packed, bias = bias2 and pq set then produces the same pq as the cout == 16 call with
 * projections, at 1/8 of the columns. */
/* The folded side convolutions (cout == 2 calls of osvos_conv3x3) of up to four scales in ONE launch: `args` is an array
 * of `count` argument blocks, each exactly what the single call takes; results are identical.  Inference runs the four
 * scales this way after the last trunk convolution (networks/vgg_osvos.py:67,69,72 for all four stages at once). */
OSVOS_API int osvos_side_folded_multi(const osvos_conv3x3_args* args /* host array */, int count, osvos_stream_t stream);

/* The fold of up to four scales in ONE launch (training re-folds after every optimizer step), optionally with an fp32
 * copy of W' in [tap][o][ci] order (18 * cin floats) - the operand of the folded backward below.                   */
typedef struct {
  const float* side_w;   /* [16,cin,3,3] */
  const float* side_b;   /* [16] or NULL */
  const float* proj_w;   /* [32]: score_dsn.weight | this scale's slice of fuse.weight */
  const float* proj_b;   /* [1] or NULL */
  void* packed;          /* osvos_packed_weight_bytes(2, cin) bytes */
  float* bias2;          /* [2] */
  float* folded_f32;     /* [9][2][cin] or NULL */
  int cin;
} osvos_fold_item;
OSVOS_API int osvos_fold_side_weights_multi(const osvos_fold_item* items /* host */, int count, osvos_stream_t stream);
/* Same contract on CUDA cores (fp32 FMA over hi+lo); debugging cross-check only. */
OSVOS_API int osvos_conv3x3_simt(const osvos_conv3x3_args* args /* host */, osvos_stream_t stream);

/* ---- stage 1 of the trunk as one kernel (inference) -------------------------------------
 * conv1_1 + ReLU + conv1_2 + ReLU (+ the first MaxPool2d(2,2,ceil_mode=True)): networks/vgg_osvos.py:61,140-143.
 * conv1_1 is evaluated inside conv1_2's kernel on the halo patch conv1_2 reads, so the 64-channel full-resolution map
 * between the two layers never touches memory.  Exact mode only.  Outputs: the full-resolution act (y_*), the pooled
 * act (pool_*), or both; all planes 32-byte aligned.  Same results as osvos_conv_first_fwd + osvos_conv3x3 up to the
 * fp32 summation order inside conv1_1.                                                            */
typedef struct {
  const float* x;          /* [n,3,h,w] fp32 frame (NCHW)                    */
  const float* w1;         /* conv1_1 weight [64,3,3,3] fp32 (OIHW)          */
  const float* b1;         /* conv1_1 bias [64] or NULL                      */
  const void* w2_packed;   /* conv1_2 weight, osvos_pack_conv3x3_weights(transpose_flip = 0) */
  const float* b2;         /* conv1_2 bias [64] or NULL                      */
  void* y_hi;              /* [n,h,w,64] or NULL                             */
  void* y_lo;
  void* pool_hi;           /* [n,ceil(h/2),ceil(w/2),64] or NULL             */
  void* pool_lo;
  int n, h, w;
} osvos_stage1_args;
OSVOS_API int osvos_stage1_fused(const osvos_stage1_args* args /* host */, osvos_stream_t stream);

/* ---- MaxPool2d(2, 2, ceil_mode=True) on an act (networks/vgg_osvos.py:140) --- */
OSVOS_API int osvos_maxpool2x2_fwd(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int n, int h, int w, int c,
                         osvos_stream_t stream);

/* ---- side-branch tail ----------------------------------------------------------
 * Replaces, in one bandwidth-bound kernel, upscale_[i](score_dsn[i](.)) + center_crop
 * (networks/vgg_osvos.py:69), upscale[i] + center_crop + cat + fuse (:68,:71-72), the
 * interp_surgery bilinear taps (layers/osvos_layers.py:59-85), the crop offsets
 * (layers/osvos_layers.py:51-56) and, when `label` is given, the per-pixel terms and
 * reductions of class_balanced_cross_entropy_loss (layers/osvos_layers.py:28-41).
 *   out[k][n,0,y,x], k<4 = sum over the <=2x2 low-res taps of scale k of p_k
 *   out[4]               = sum_k (same taps of q_k) + fuse_bias
 *   sums[2k], sums[2k+1] = {sum_{y=1} (softplus(x)-x), sum_{y=0} softplus(x)} of map k,
 *   sums[10] = P = #(label >= .5), sums[11] = number of pixels N,
 *   sums[12], sums[13] = {sum_{y=1} (sigmoid(x_fused)-1), sum_{y=0} sigmoid(x_fused)} (-> d fuse.bias),
 *   sums[14] = arrival counter                         (OSVOS_TAIL_SUMS = 15 doubles, zeroed by the call)
 * and, when `losses` is given (the package's own objective: train_online.py:127, train_parent.py:143-147),
 *   losses[k] = (Nn/N * S_pos_k + P/N * S_neg_k) / divisor,  losses[5] = sum_k loss_weights[k] * losses[k]
 * so that upsample + crop + fuse + the five class-balanced BCE losses are ONE kernel.            */
#define OSVOS_TAIL_SUMS 15
typedef struct {
  const float* pq[4];      /* [n, h_k, w_k, 2], h_k = ceil-halved k+1 times          */
  const float* fuse_bias;  /* [1] */
  float* out[5];           /* each [n,1,h,w] fp32, any may be NULL                   */
  const float* label;      /* [n,1,h,w] or NULL */
  double* sums;            /* [OSVOS_TAIL_SUMS] or NULL (required with label)         */
  float* losses;           /* [6] or NULL (needs label)                               */
  float loss_weights[5];   /* weights of the five losses in losses[5]                 */
  float divisor;           /* batch size (batch_average), numel (size_average) or 1   */
  int n, h, w;
  int flags;               /* OSVOS_FLAG_DETERMINISTIC: then `sums` holds osvos_tail_fwd_sums(n, h, w, flags) doubles -
                              the 15 above, then one row of block partials per block, added in a fixed order.
                              OSVOS_FLAG_VOID_LABELS (needs label): pixels with label < 0 enter no sum, sums[11] = N is
                              the count of the others, and N == 0 gives losses of 0.
                              Added after the other members: zero-initialise the struct (other bits are refused). */
} osvos_tail_fwd_args;
OSVOS_API int osvos_tail_fwd(const osvos_tail_fwd_args* args /* host */, osvos_stream_t stream);
/* doubles of osvos_tail_fwd's `sums` for these flags (OSVOS_TAIL_SUMS without OSVOS_FLAG_DETERMINISTIC), 0 for shapes
 * or flags the call refuses; equal to osvos_tail_fwd_deterministic_sums(n, h, w) for OSVOS_FLAG_DETERMINISTIC alone. */
OSVOS_API size_t osvos_tail_fwd_sums(int n, int h, int w, int flags);

/* Standalone 1x1 projections of a side feature map (used when the features do
 * not come from osvos_conv3x3's fused epilogue): pq as above.                       */
OSVOS_API int osvos_side_project(const float* feat /* [n,h,w,16] */, const float* proj_w, const float* proj_b, float* pq,
                       int n, int h, int w, osvos_stream_t stream);

/* ---- class_balanced_cross_entropy_loss (layers/osvos_layers.py:19-48) -----------
 * forward: sums[0..3] = {S_pos, S_neg, P, N} (osvos_cbce_fwd_sums(numel, flags) doubles; the call zeroes the first 5,
 * sums[4] is an arrival counter), loss[0] = (Nn/N*S_pos + P/N*S_neg)/divisor with divisor = numel (size_average), batch
 * (batch_average) or 1.  backward: grad_in = grad_out[0] * w * (sigmoid(x) - y) / divisor
 * (grad_out == NULL means 1).
 * Void labels: osvos_cbce_fwd with OSVOS_FLAG_VOID_LABELS sums only pixels with y >= 0 and stores their count N in
 * sums[3] (rows of four block sums under OSVOS_FLAG_DETERMINISTIC); osvos_cbce_bwd_void reads those sums and gives
 * pixels with y < 0 zero gradient.  N == 0 gives loss 0 and gradient 0.              */
OSVOS_API size_t osvos_cbce_fwd_sums(size_t numel, int flags);
OSVOS_API int osvos_cbce_fwd(const float* output, const float* label, size_t numel, double divisor, double* sums,
                             float* loss, int flags, osvos_stream_t stream);
OSVOS_API int osvos_cbce_bwd(const float* output, const float* label, const double* sums, const float* grad_out,
                             double divisor, size_t numel, float* grad_in, osvos_stream_t stream);
OSVOS_API int osvos_cbce_bwd_void(const float* output, const float* label, const double* sums, const float* grad_out,
                                  double divisor, size_t numel, float* grad_in, osvos_stream_t stream);

/* ======================= backward (training) entry points ======================= */

/* ---- weight gradient of a 3x3 conv (wgmma GEMM over the pixel axis) -----------
 * Replaces autograd's weight gradient of nn.Conv2d(k=3,p=1) (reference
 * networks/vgg_osvos.py:41,142; backward at train_online.py:141 / train_parent.py:164):
 *   dw[co][ci][r][s] = sum_px dz[px][co] * x[px + (r-1, s-1)][ci]
 * dz has `cout` channels (dz_channels == cout, a multiple of 64).  (side_prep's weight gradient does not come through
 * here: osvos_side_folded_wgrad_multi / osvos_side_grads_finish.)
 * workspace: osvos_wgrad_workspace_bytes(n, h, w, cin, dz_channels, flags & OSVOS_FLAG_DETERMINISTIC) bytes, contents
 * destroyed.  */
typedef struct {
  const void* x_hi;   /* layer input act [n,h,w,cin]        */
  const void* x_lo;
  const void* dz_hi;  /* output-gradient act [n,h,w,dz_channels] */
  const void* dz_lo;
  float* dw;          /* [cout][cin][3][3] fp32, overwritten */
  float* workspace;
  int n, h, w, cin, cout, dz_channels;
  int flags;          /* OSVOS_FLAG_FAST | OSVOS_FLAG_DEFER_FINISH (then dw may be NULL) | OSVOS_FLAG_DETERMINISTIC (then
                         the workspace needs no zeroing) */
} osvos_wgrad_args;
OSVOS_API size_t osvos_wgrad_workspace_bytes(int n, int h, int w, int cin, int dz_channels, int flags);
OSVOS_API int osvos_conv3x3_wgrad(const osvos_wgrad_args* args /* host */, osvos_stream_t stream);

/* Deferred finish of up to OSVOS_WGRAD_FINISH_MAX weight gradients in ONE launch: workspace [9][a][b] -> OIHW,
 * dw = (accumulate ? dw : 0) + scale * ws.  With accumulate the destination can be the parameter's .grad itself
 * (what autograd's AccumulateGrad would do with a separate add kernel, train_online.py:141).  `splits` (host,
 * [count]): the osvos_wgrad_deterministic_splits of each item's shape with OSVOS_FLAG_DETERMINISTIC, NULL without. */
#define OSVOS_WGRAD_FINISH_MAX 24
typedef struct {
  const float* workspace;  /* as passed to osvos_conv3x3_wgrad with OSVOS_FLAG_DEFER_FINISH */
  float* dw;               /* [cout][cin][3][3] */
  int cout, cin, dz_channels;
  int accumulate;
  float scale;
} osvos_wgrad_finish_item;
OSVOS_API int osvos_wgrad_finish(const osvos_wgrad_finish_item* items /* host */, const int* splits, int count, int flags,
                                 osvos_stream_t stream);

/* ---- adjoint of the tail: gradients of the five maps -> low-res dp/dq ------------
 * Backward of osvos_tail_fwd (autograd of networks/vgg_osvos.py:68-72): strided bilinear
 * DOWN-sampling of grad_out[k] (-> dpq[k][..,0]) and of grad_out[4] (-> dpq[k][..,1])
 * through the crop window.  NULL grad_out entries count as zero.                       */
typedef struct {
  const float* grad_out[5]; /* each [n,1,h,w] or NULL */
  float* dpq[4];            /* [n,h_k,w_k,2] */
  int n, h, w;
  int flags;                /* 0 or OSVOS_FLAG_DETERMINISTIC; zero-initialise the struct (other bits are refused) */
} osvos_tail_bwd_args;
OSVOS_API int osvos_tail_bwd(const osvos_tail_bwd_args* args /* host */, osvos_stream_t stream);

/* ---- backward of tail + class-balanced BCE in one launch ---------------------------
 * Autograd of `total = sum_k loss_weights[k] * class_balanced_cross_entropy_loss(out[k], label)` through
 * osvos_tail_fwd (layers/osvos_layers.py:28-46 + networks/vgg_osvos.py:68-72; the parent / online objectives of
 * train_parent.py:143-147 and train_online.py:127): dL/dlogit_k = upstream * loss_weights[k] * w * (sigmoid(x_k) - y)
 * / divisor is formed on the fly from the logit maps and the label while the bilinear adjoint gathers it - the five
 * gradient maps are never written.  `sums` is the forward call's (P, N and the fuse-bias sums are read from it).   */
typedef struct {
  const float* logits[5];   /* the five maps written by osvos_tail_fwd (NULL allowed where the weight is 0) */
  const float* label;       /* [n,1,h,w] */
  const double* sums;       /* [OSVOS_TAIL_SUMS] of the forward call */
  const float* upstream;    /* device scalar d(total) or NULL (= 1) */
  float loss_weights[5];
  float divisor;
  float* dpq[4];            /* [n,h_k,w_k,2] */
  float* fuse_bias_grad;    /* [1] or NULL */
  int n, h, w;
  int flags;                /* OSVOS_FLAG_DETERMINISTIC | OSVOS_FLAG_VOID_LABELS (as passed to the forward call, whose
                               sums[11] is then the non-void count); zero-initialise the struct (other bits are refused) */
} osvos_tail_loss_bwd_args;
OSVOS_API int osvos_tail_loss_bwd(const osvos_tail_loss_bwd_args* args /* host */, osvos_stream_t stream);

/* out[0] = sum(x[0:n]) (fuse.bias gradient); scratch: osvos_sum_f32_scratch_bytes(flags) bytes, 8-byte aligned.  */
OSVOS_API size_t osvos_sum_f32_scratch_bytes(int flags);
OSVOS_API int osvos_sum_f32(const float* x, size_t n, void* scratch, float* out, int flags, osvos_stream_t stream);

/* ---- max-unpool + side-branch add + ReLU mask (autograd of networks/vgg_osvos.py:140,143) ------------------------
 * dz = ReLU'(x) * (unpool(dpool) + side-branch gradient), the side-branch gradient being one of
 *   dside:      an fp32 map [n,h,w,c], 16-byte aligned;
 *   dpq, wfold: the folded form dX[px][c] = sum_{t,o} wfold[t][o][c] dpq[px - t][o] (see the folded side branch
 *               backward below), computed on the fly; dpq [n,h,w,2], wfold [9][2][c] fp32 16-byte aligned, h*w < 2^30;
 *   neither:    zero (stage 1).
 * dpool_hi NULL: no pooling consumer (the deepest stage); at least one of dpool_hi, dside and dpq is set, and dside
 * excludes dpq.  colsum: [c] per-channel sum of dz (the bias gradient), accumulated, or NULL.  c: a multiple of 8 up
 * to 2048 with 256 % (c / 8) == 0.                                                                                  */
OSVOS_API int osvos_unpool_mask(const void* dpool_hi /* or NULL */, const void* dpool_lo, const void* x_hi,
                                const void* x_lo, const float* dside /* or NULL */, const float* dpq /* or NULL */,
                                const float* wfold /* or NULL */, void* dz_hi, void* dz_lo, float* colsum /* or NULL */,
                                int n, int h, int w, int c, int flags, osvos_stream_t stream);

/* ---- side branch backward in folded (rank-2) form -------------------------------------------------------------
 * Autograd of networks/vgg_osvos.py:67,69,72 (side_prep -> score_dsn / fuse slice) expressed on the folded 3x3
 * convolution C -> 2 (see osvos_fold_side_weights_multi): the branch's backward only sees the two gradient channels
 * dpq = (dL/dp, dL/dq).
 *   osvos_side_folded_wgrad_multi: for up to four scales in one launch (x_lo either set for all items or for none),
 *                             g[t][o][c] += sum_px dpq[px - t][o] * x[px][c]  (t = 3r + s <-> offset (r-1, s-1)),
 *                             g[18 c + o] += sum_px dpq[px][o];   g: osvos_side_folded_wgrad_floats(c) floats, PRE-ZEROED,
 *                             16-byte aligned; c a multiple of 128.  workspace: osvos_side_folded_wgrad_workspace_bytes(
 *                             items, count, flags) bytes, 16-byte aligned (0 in the default form: workspace may be NULL).
 *   osvos_side_grads_finish:  every parameter gradient of up to four scales from g, one launch:
 *                             d side_prep.weight[f][c][t] = proj[f] g[t][0][c] + proj[16+f] g[t][1][c],
 *                             d side_prep.bias[f] = proj[f] S0 + proj[16+f] S1,
 *                             d score_dsn.weight[f] = <side_w[f], g[.][0][.]> + side_b[f] S0, d score_dsn.bias = S0,
 *                             d fuse.weight slice[f] = <side_w[f], g[.][1][.]> + side_b[f] S1
 *                             (NULL outputs are skipped; accumulate: add to the destinations instead of overwriting).
 *   osvos_unpool_mask with dpq and wfold (the fp32 folded weights of osvos_fold_side_weights_multi): the gradient
 *                             w.r.t. the stage output, dX[px][c] = sum_{t,o} wfold[t][o][c] dpq[px - t][o].          */
OSVOS_API size_t osvos_side_folded_wgrad_floats(int c);
typedef struct {
  const void* x_hi;
  const void* x_lo;
  const float* dpq;
  float* g;
  int n, h, w, c;
} osvos_side_wgrad_item;
OSVOS_API size_t osvos_side_folded_wgrad_workspace_bytes(const osvos_side_wgrad_item* items /* host */, int count,
                                                         int flags);
OSVOS_API int osvos_side_folded_wgrad_multi(const osvos_side_wgrad_item* items /* host */, int count, void* workspace,
                                            int flags, osvos_stream_t stream);
typedef struct {
  const float* g;        /* as filled by osvos_side_folded_wgrad_multi */
  const float* side_w;   /* [16,c,3,3] */
  const float* side_b;   /* [16] or NULL */
  const float* proj_w;   /* [32] */
  float* d_side_w;       /* [16,c,3,3] */
  float* d_side_b;       /* [16] */
  float* d_score_w;      /* [16] or NULL */
  float* d_score_b;      /* [1] or NULL */
  float* d_fuse_w;       /* [16] (this scale's slice) or NULL */
  int c;
  int accumulate;
} osvos_side_grads_item;
OSVOS_API int osvos_side_grads_finish(const osvos_side_grads_item* items /* host */, int count, osvos_stream_t stream);

/* ---- conv1_1 backward: dw [64][3][3][3] and (optionally) dx [n,3,h,w] ---------------
 * workspace: osvos_conv_first_bwd_workspace_bytes(n, h, w, flags) bytes (default form: replicated partial sums +
 * arrival counter, zeroed by the call).                                                       */
OSVOS_API size_t osvos_conv_first_bwd_workspace_bytes(int n, int h, int w, int flags);
OSVOS_API int osvos_conv_first_bwd(const float* x_nchw, const void* dz_hi, const void* dz_lo, const float* w_oihw,
                                   float* dw, float* dx_nchw /* or NULL */, void* workspace, int n, int h, int w,
                                   int flags, osvos_stream_t stream);

/* ---- Deterministic forms (OSVOS_FLAG_DETERMINISTIC; torch.use_deterministic_algorithms in the package) ----------
 * Every float reduction of the training path has a form whose summation order depends on the shapes (and, where a
 * grid is sized by it, the device's SM count) only, so two runs on one device give bit-identical results.  What the
 * flag changes, per entry point (the size queries take the same flags and return 0 for shapes the calls refuse):
 *   osvos_conv3x3:              colsum is partial rows [osvos_conv3x3_colsum_rows(n, h, w)][cout], 8 per 128-pixel tile.
 *   osvos_conv3x3_wgrad:        one workspace slice per pixel-range split, written with plain stores; the split count
 *                               (osvos_wgrad_deterministic_splits) comes from a nominal 132-SM device, not the H100 variant.
 *   osvos_wgrad_finish:         adds the splits[i] slices of item i in order before it scales and accumulates.
 *   osvos_unpool_mask:          colsum is partial rows [osvos_unpool_colsum_rows(n, h, w, c, pool, side)][c], one per
 *                               block (pool = dpool_hi != NULL, side = dpq != NULL).
 *   osvos_side_folded_wgrad_multi: G += the blocks' partial rows in order, through the workspace.
 *   osvos_conv_first_bwd:       one partial slot per block in the workspace, added by the ordered row reduction.
 *   osvos_cbce_fwd:             one row of block sums per block behind sums[0..4], added in a fixed order by the last
 *                               block (osvos_cbce_bwd reads sums[0..4] either way).
 *   osvos_sum_f32:              a fixed grid of 256 contiguous ranges, their totals added in order by the last block.
 *   osvos_tail_fwd / osvos_tail_bwd / osvos_tail_loss_bwd: the `flags` member of their argument blocks (appended:
 *                               callers zero-initialise the blocks); tail_fwd's sums: osvos_tail_fwd_sums.
 * osvos_reduce_rows adds such partial rows: out[c] = (accumulate ? out[c] : 0) + sum_r rows[r][c], rows [nrows][ncols]
 * fp32, in a fixed order (up to 64 row segments, each summed by 8 interleaved row lanes); scratch:
 * osvos_reduce_rows_scratch_floats(nrows, ncols) floats.                                                            */
OSVOS_API size_t osvos_reduce_rows_scratch_floats(int nrows, int ncols);
OSVOS_API int osvos_reduce_rows(const float* rows, int nrows, int ncols, float* scratch, float* out, int accumulate,
                                osvos_stream_t stream);
OSVOS_API size_t osvos_conv3x3_colsum_rows(int n, int h, int w);
OSVOS_API int osvos_wgrad_deterministic_splits(int n, int h, int w, int cin, int dz_channels);
OSVOS_API size_t osvos_unpool_colsum_rows(int n, int h, int w, int c, int pool, int side);
OSVOS_API size_t osvos_tail_fwd_deterministic_sums(int n, int h, int w);

/* ===================== SURVEY.md 8(f) "next" rows: callers either side ===================== */

/* ---- test-time output path (train_online.py:181-187) --------------------------------
 * The reference copies the fused logits to the host, applies 1/(1+exp(-x)) in numpy and hands
 * the float map to scipy.misc.imsave, which rescales [min,max] of the frame to [0,255]
 * ("bytescale").  Here the 8-bit map is produced on the device so only H*W bytes cross PCIe.
 *   OSVOS_U8_PROB      out = floor(255*sigmoid(x) + 0.5)
 *   OSVOS_U8_BYTESCALE out = floor(clip((p - pmin) * 255/(pmax - pmin), 0, 255) + 0.5), p = sigmoid(x),
 *                      pmin/pmax over each frame (pmax == pmin -> divisor 1): the PNG the reference writes
 *   OSVOS_U8_MASK      out = x > 0 ? 255 : 0   (the thresholded mask, sigmoid(x) > 0.5)
 * logits [frames][per_frame] fp32, out [frames][per_frame] u8, minmax_ws: 2 uint32 per frame
 * (only used by BYTESCALE; zeroed by the call).                                                   */
enum { OSVOS_U8_PROB = 0, OSVOS_U8_BYTESCALE = 1, OSVOS_U8_MASK = 2 };
OSVOS_API int osvos_logits_to_u8(const float* logits, uint8_t* out, uint32_t* minmax_ws, int frames, size_t per_frame,
                                 int mode, osvos_stream_t stream);

/* ---- optimizer step (train_online.py:79-88,147; train_parent.py:87-103,170) -------------
 * torch.optim.SGD(momentum, weight_decay, dampening 0, no nesterov) over every trainable tensor in ONE launch:
 *     g' = g + wd*p ;  m = mu*m + g' ;  p = p - lr*m        (m starts at 0, so the first step gives m = g')
 * with per-tensor lr / wd / mu (the reference's parameter groups), optionally zeroing g in the same pass
 * (optimizer.zero_grad(), train_online.py:148), and - for 3x3 conv weights whose `packed_*` pointers are set -
 * re-emitting the tensor-core operand layouts of osvos_pack_conv3x3_weights (forward, col_pad = colp_fwd multiple;
 * transposed+flipped for dgrad) from the updated values, so no separate repack pass runs after the step.
 * `segments` is a DEVICE array of `count` descriptors (<= OSVOS_SGD_MAX_SEGMENTS); `work_items` of each
 * descriptor = osvos_sgd_work_items(numel, cout, cin) (host helper).  Pad columns of the packed layouts are not
 * touched (they stay zero from the initial osvos_pack_conv3x3_weights call).                           */
#define OSVOS_SGD_MAX_SEGMENTS 64
typedef struct osvos_sgd_segment {
  float* param;         /* [numel] fp32, updated in place                                         */
  float* grad;          /* [numel] fp32 (zeroed when zero_grad != 0)                              */
  float* momentum;      /* [numel] fp32 momentum buffer, updated in place                         */
  uint64_t numel;
  float lr, weight_decay, momentum_coef;
  int32_t cout, cin;    /* 3x3 conv weight [cout][cin][3][3] when packed_fwd/packed_flip are set  */
  int32_t colp_fwd;     /* padded column count of the forward layout  (multiple of its col_pad)   */
  int32_t colp_flip;    /* padded column count of the flipped layout                              */
  uint32_t work_items;  /* osvos_sgd_work_items(numel, cout, cin) when packing, (numel, 0, 0) else */
  void* packed_fwd;     /* or NULL */
  void* packed_flip;    /* or NULL */
} osvos_sgd_segment;
OSVOS_API uint32_t osvos_sgd_work_items(uint64_t numel, int cout, int cin);
OSVOS_API int osvos_sgd_step(const osvos_sgd_segment* segments /* device */, int count, uint32_t total_work_items,
                             int zero_grad, osvos_stream_t stream);

/* ---- data augmentation on the device (dataloaders/custom_transforms.py:7-54 ScaleNRotate, :87-100
 * RandomHorizontalFlip, composed flip-then-warp at train_online.py:92-94 / train_parent.py:108-110) -----
 * The reference warps every sample on the host with cv2.warpAffine(tmp, getRotationMatrix2D(center, rot, sc),
 * (w, h), flags) - INTER_CUBIC for the image, INTER_NEAREST for the 0/1 mask, BORDER_CONSTANT 0.  This entry point
 * restates OpenCV's published algorithm (cv2 is not vendored by the reference and absent from this image):
 * fixed-point source coordinates X = (rint((m1*y+m2)*1024) + delta + rint(m0*x*1024)) >> s with 1/32-pixel
 * sub-positions for cubic (delta 16, s 5) and whole pixels for nearest (delta 512, s 10); bicubic taps with
 * A = -0.75 evaluated in fp32 at the 1/32 position; taps outside the image contribute 0.
 * src/dst [n][c][h][w] fp32; inv_matrices_host: n x 6 doubles, the INVERTED 2x3 matrix (dst -> src) as
 * cv::warpAffine computes it; flips_host[n]: 1 = the source is mirrored horizontally first (cv2.flip(.., 1)).   */
enum { OSVOS_WARP_CUBIC = 0, OSVOS_WARP_NEAREST = 1 };
OSVOS_API int osvos_affine_warp(const float* src, float* dst, const double* inv_matrices_host, const int* flips_host,
                                int n, int c, int h, int w, int mode, osvos_stream_t stream);

/* ---- ingest of decoded frames (dataloaders/davis_2016.py:88-108 make_img_gt_pair, custom_transforms.py:103-122
 * ToTensor) ------------------------------------------------------------------------------------------------------
 * The host decodes with cv2.imread and copies the uint8 bytes; everything after the decode runs here, bit-identical
 * to the reference's float arithmetic.  Any h, w and source alignment; n < 65536.
 *   osvos_image_from_bgr8: src [n][h][w][3] uint8 (BGR, as cv2.imread returns it) -> dst [n][3][h][w] fp32,
 *                          dst = float(v) - mean[c] with one fp32 rounding (np.subtract of two float32 arrays).
 *   osvos_label_stats_u8:  src [n][h][w] uint8 mask -> stats [n][2] = {max byte, binary flag}; the flag is 1 when every
 *                          byte is 0 or the max, i.e. the normalised mask is all 0 / 1.  Zeroes stats itself; run it
 *                          before the two calls below that read stats.
 *   osvos_label_from_u8:   dst [n][1][h][w] fp32 = float(v) / max(float(max), 1e-8f) (gt / np.max([gt.max(), 1e-8]),
 *                          rounded to fp32).
 *   osvos_affine_warp_u8:  RandomHorizontalFlip + ScaleNRotate of the ingested tensors read straight from the bytes,
 *                          same matrices and arithmetic as osvos_affine_warp.  Image (image_src -> image_dst
 *                          [n][3][h][w]): cubic over mean-subtracted taps, so the border is 0 of the mean-subtracted
 *                          image; bit-identical to osvos_image_from_bgr8 + osvos_affine_warp(CUBIC).  Mask (label_src,
 *                          label_stats -> label_dst [n][1][h][w]): nearest where the sample's binary flag is set, cubic
 *                          otherwise (custom_transforms.py:46-49), chosen on the device; bit-identical to
 *                          osvos_label_from_u8 + osvos_affine_warp in that mode.  Either tensor may be NULL (all three
 *                          label pointers together).
 *   osvos_affine_warp_u8_indexed: the same warp over a batch gathered from frame stores that stay on the device
 *                          (image_store [n_store][h][w][3], label_store [n_store][h][w], label_stats [n_store][2]):
 *                          output sample i (image_dst [n][3][h][w], label_dst [n][1][h][w]) is store frame
 *                          index_host[i], bit-identical to osvos_affine_warp_u8 on the gathered contiguous batch.
 *                          index_host[n] is host memory and travels with the matrices as a kernel parameter;
 *                          indices may repeat, and each must lie in [0, n_store).  NULL rules as osvos_affine_warp_u8.
 *                          (custom_transforms.py:7-54, :87-100 applied to frames decoded once per run instead of once
 *                          per epoch.)                                                                             */
OSVOS_API int osvos_image_from_bgr8(const uint8_t* src, float* dst, int n, int h, int w, float mean_b, float mean_g,
                                    float mean_r, osvos_stream_t stream);
OSVOS_API int osvos_label_stats_u8(const uint8_t* src, uint32_t* stats, int n, int h, int w, osvos_stream_t stream);
OSVOS_API int osvos_label_from_u8(const uint8_t* src, const uint32_t* stats, float* dst, int n, int h, int w,
                                  osvos_stream_t stream);
OSVOS_API int osvos_affine_warp_u8(const uint8_t* image_src, const uint8_t* label_src, const uint32_t* label_stats,
                                   float* image_dst, float* label_dst, const double* inv_matrices_host,
                                   const int* flips_host, int n, int h, int w, float mean_b, float mean_g, float mean_r,
                                   osvos_stream_t stream);
OSVOS_API int osvos_affine_warp_u8_indexed(const uint8_t* image_store, const uint8_t* label_store,
                                           const uint32_t* label_stats, float* image_dst, float* label_dst,
                                           const int* index_host, const double* inv_matrices_host,
                                           const int* flips_host, int n, int n_store, int h, int w, float mean_b,
                                           float mean_g, float mean_r, osvos_stream_t stream);

/* ---- labels from object-id maps (DAVIS-2017 annotations: 0 background, 1..K objects, 255 void) ------------------
 * The label of id v is -1 for v == 255 (void, for OSVOS_FLAG_VOID_LABELS), 1 for an object (1 <= v <= 254 when
 * object == 0, v == object otherwise) and 0 else.
 *   osvos_labels_from_ids: ids [n][h][w] uint8 -> dst [n][1][h][w] fp32.
 *   osvos_affine_warp_ids: the mask half of osvos_affine_warp_u8 (index_host == NULL) or of osvos_affine_warp_u8_indexed
 *                          for id maps: output sample i reads store frame index_host[i] (or i) of ids [n_store][h][w],
 *                          always sampled nearest, out-of-frame samples 0.  Equal, bit for bit, to the label of the
 *                          0/255 object mask warped by those calls, set to -1 where the warped 0/255 void mask is 1.
 * object: 0 (every object) or 1..254.  Same size rules as the calls above.                                         */
OSVOS_API int osvos_labels_from_ids(const uint8_t* ids, float* dst, int n, int h, int w, int object,
                                    osvos_stream_t stream);
OSVOS_API int osvos_affine_warp_ids(const uint8_t* ids_store, float* label_dst, const int* index_host,
                                    const double* inv_matrices_host, const int* flips_host, int n, int n_store, int h,
                                    int w, int object, osvos_stream_t stream);

/* ---- resize of decoded frames (dataloaders/davis_2016.py:96-99 inputRes: scipy.misc.imresize, i.e. Pillow's 8-bit
 * Image.resize; DESIGN.md §17) ----------------------------------------------------------------------------------------
 *   osvos_resize_u8: src [n][h][w][c] uint8 -> dst [n][out_h][out_w][c] uint8, c = 1 or 3, bit-identical to Pillow's
 *                    Image.resize((out_w, out_h), BILINEAR) (separable antialiased triangle filter, 22-bit fixed point,
 *                    horizontal pass first) or NEAREST (ImagingScaleAffine's index walk) of an L / RGB image; channels
 *                    are independent, so BGR bytes resize as they are.  Equal sizes are a copy.  n < 65536, h, w,
 *                    out_h, out_w < 32768; src and dst any alignment, not overlapping.  `workspace`:
 *                    osvos_resize_u8_workspace_bytes(...) bytes (the coefficient or index tables and, when both axes
 *                    change size under BILINEAR, the horizontal pass's uint8 intermediate), 4-byte aligned, owned by the
 *                    caller (may be NULL when that is 0); nothing is allocated and nothing waits for the host.
 *   osvos_resize_u8_workspace_bytes: host query; 0 for invalid arguments.                                            */
enum { OSVOS_RESIZE_BILINEAR = 0, OSVOS_RESIZE_NEAREST = 1 };
OSVOS_API size_t osvos_resize_u8_workspace_bytes(int n, int h, int w, int c, int out_h, int out_w, int mode);
OSVOS_API int osvos_resize_u8(const uint8_t* src, uint8_t* dst, void* workspace, int n, int h, int w, int c, int out_h,
                              int out_w, int mode, osvos_stream_t stream);

/* ---- resize of fp32 maps (fused logits back to the annotations' stored size: scipy 1.0's imresize(..., mode='F'),
 * i.e. Pillow's 'F' Image.resize; DESIGN.md §18) ----------------------------------------------------------------------
 *   osvos_resize_f32: src [n][h][w] fp32 -> dst [n][out_h][out_w] fp32, bit-identical to Pillow's
 *                     Image.resize((out_w, out_h), BILINEAR) of an 'F' image: the bilinear coefficient tables of
 *                     osvos_resize_u8 kept in double (not rounded to fixed point), horizontal pass first into an fp32
 *                     intermediate that holds only the source rows the vertical pass reads, each output a double sum
 *                     of (double)src * k rounded once to fp32; an axis that keeps its size has no pass and equal sizes
 *                     are a copy.  n < 65536, h, w, out_h, out_w < 32768; src and dst 4-byte aligned, not
 *                     overlapping.  `workspace`: osvos_resize_f32_workspace_bytes(...) bytes (per axis {xmin, count}
 *                     and the double weights and, when both axes change size, the fp32 intermediate), 8-byte aligned,
 *                     owned by the caller (may be NULL when that is 0); nothing is allocated and nothing waits for
 *                     the host.
 *   osvos_resize_f32_workspace_bytes: host query; 0 for invalid arguments.                                          */
OSVOS_API size_t osvos_resize_f32_workspace_bytes(int n, int h, int w, int out_h, int out_w);
OSVOS_API int osvos_resize_f32(const float* src, float* dst, void* workspace, int n, int h, int w, int out_h, int out_w,
                               osvos_stream_t stream);

/* ---- DAVIS-2016 region and boundary measures (J and F; DESIGN.md §14) -------------------------------------------
 * Per frame, P = logit > 0 (±0.0 is background, as osvos_logits_to_u8 mode MASK) and G = byte != 0.  The boundary map
 * of a mask is b = seg^E | seg^S | seg^SE (E, S, SE: the right, lower and lower-right neighbour, zeros past the frame),
 * with the last row = seg^E, the last column = seg^S and the last pixel 0.  Each boundary map is dilated by the disk
 * dx² + dy² <= r² (pixels outside the frame are background) and ANDed with the other one.
 *   osvos_davis_measures: logits [n][h][w] fp32 (4-byte aligned), masks [n][h][w] uint8 (any alignment) ->
 *                         counts [n][6] int32 = {|P∧G|, |P∨G|, |B(P)|, |B(G)|, |B(P) ∧ dilate(B(G))|,
 *                         |B(G) ∧ dilate(B(P))|}.  1 <= r <= OSVOS_DAVIS_MAX_RADIUS (31 covers frames up to a 3875-pixel
 *                         diagonal at the benchmark's 0.008 tolerance; 1080p needs 18); n < 65536, h, w < 32768.
 *                         `workspace`: osvos_davis_measures_workspace_bytes(n, h, w) bytes, 4-byte aligned, owned by the
 *                         caller; nothing is allocated.  Zeroes counts itself.  Integer counts: the result does not
 *                         depend on the launch configuration.
 *   osvos_davis_measures_workspace_bytes: host query; 0 for a non-positive dimension.                               */
#define OSVOS_DAVIS_MAX_RADIUS 31
OSVOS_API size_t osvos_davis_measures_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_davis_measures(const float* logits, const uint8_t* masks, int* counts, void* workspace, int n, int h,
                                   int w, int r, osvos_stream_t stream);

/* ---- DAVIS-2017 per-object measures and the merge of per-object maps (DESIGN.md §24) ------------------------------
 *   osvos_davis_measures_objects: label maps [n][h][w] uint8 and annotations gt [n][h][w] uint8 (both any alignment) ->
 *                         counts [n][k][6] int32 (4-byte aligned), row (f, j) the six counts of osvos_davis_measures for
 *                         object j + 1 with P = label == j + 1 and G = gt == j + 1, both cleared where gt == 255 (void).
 *                         Boundaries, radius and disk as osvos_davis_measures.  1 <= k <= OSVOS_DAVIS_MAX_OBJECTS,
 *                         n * k < 65536, h, w < 32768.  `workspace`: osvos_davis_measures_objects_workspace_bytes(n, k,
 *                         h, w) bytes, 4-byte aligned, owned by the caller.  Zeroes counts itself.  Integer counts: the
 *                         result does not depend on the launch configuration.
 *   osvos_davis_measures_objects_workspace_bytes: host query; 0 for a non-positive dimension.
 *   osvos_merge_objects:  `maps` (host array of k device pointers, each to `pixels` fp32 values, 4-byte aligned) ->
 *                         out [pixels] uint8 (any alignment): 1 + the first k of the largest value where that value is
 *                         > 0, else 0 (±0 and NaN never win).  1 <= k <= OSVOS_MERGE_MAX_OBJECTS.                    */
#define OSVOS_DAVIS_MAX_OBJECTS 254
#define OSVOS_MERGE_MAX_OBJECTS 254
OSVOS_API size_t osvos_davis_measures_objects_workspace_bytes(int n, int k, int h, int w);
OSVOS_API int osvos_davis_measures_objects(const uint8_t* labels, const uint8_t* gt, int* counts, void* workspace, int n,
                                           int k, int h, int w, int r, osvos_stream_t stream);
OSVOS_API int osvos_merge_objects(const float* const* maps, int k, uint8_t* out, size_t pixels, osvos_stream_t stream);

/* ---- reduced-resolution DAVIS-2017: per-object upsample fused with the merge (DESIGN.md §27) ---------------------
 *   osvos_upsample_merge_objects: `maps` (host array of k device pointers, each to fp32 [n][h][w], 4-byte aligned) ->
 *                         out [n][out_h][out_w] uint8 (any alignment), bit-identical to osvos_merge_objects of the k maps
 *                         each resized by osvos_resize_f32 to out_h x out_w, without the resized maps: two launches (the
 *                         coefficient tables, then one tile kernel that stages each map's horizontal pass in shared memory
 *                         and keeps the running argmax in registers), one when the sizes are equal (a plain merge).
 *                         1 <= k <= OSVOS_MERGE_MAX_OBJECTS, n < 65536, h, w, out_h, out_w < 32768.  A vertical downscale
 *                         too steep to stage one output row's source rows, 128 columns of doubles each, in 48 KiB of
 *                         shared memory is refused (status 1): min(h, 2 * ceil(h / out_h) + 3) > 48, i.e. h / out_h > 22.
 *                         `workspace`: osvos_upsample_merge_objects_workspace_bytes(...) bytes (the tables), 8-byte
 *                         aligned, owned by the caller (may be NULL when that is 0); nothing is allocated and nothing
 *                         waits for the host.
 *   osvos_upsample_merge_objects_workspace_bytes: host query; 0 for equal sizes and for invalid or refused arguments. */
OSVOS_API size_t osvos_upsample_merge_objects_workspace_bytes(int n, int k, int h, int w, int out_h, int out_w);
OSVOS_API int osvos_upsample_merge_objects(const float* const* maps, int k, uint8_t* out, void* workspace, int n, int h,
                                           int w, int out_h, int out_w, osvos_stream_t stream);

/* ---- baseline JPEG decode, bit-identical to cv2.imread (libjpeg-turbo; DESIGN.md §19) ----------------------------
 *   osvos_jpeg_decode: a batch of n JPEGs of one size h x w, packed by osvos_pytorch_b200.jpeg.pack into `blob`
 *                      (blob_bytes bytes, 16-byte aligned; headers, tables and de-stuffed entropy-coded segments) ->
 *                      out [n][h][w][3] uint8 BGR (any alignment) and status [n] int32.  Tables, sampling and quality
 *                      may differ per image.  Huffman decoding is a self-synchronising parallel decode over chunks of
 *                      chunk_bits bits (0: the default, OSVOS_JPEG_DEFAULT_CHUNK_BITS; otherwise >= 32), then the
 *                      DC prefix sums, ISLOW IDCT, fancy upsampling and fixed-point YCbCr -> BGR of libjpeg-turbo.
 *                      status bits: 1 a bad Huffman code, 2 a zig-zag index past 63, 4 entropy data that ended
 *                      before the last MCU (bits past a segment's end read as zero, as libjpeg-turbo does), 8 a
 *                      header inconsistent with the arguments (that image is not decoded).  Output for a stream with
 *                      bad codes is not specified, but the call reads nothing outside the blob and writes nothing
 *                      outside out, status and the workspace.  `nseg` is the blob's segment count.  `workspace`:
 *                      osvos_jpeg_decode_workspace_bytes(...) bytes, 16-byte aligned, owned by the caller; nothing
 *                      is allocated and nothing waits for the host.  n < 65536, h, w < 32768.
 *   osvos_jpeg_decode_workspace_bytes: host query; 0 for invalid arguments.                                          */
#define OSVOS_JPEG_DEFAULT_CHUNK_BITS 512
typedef struct osvos_jpeg_args {
  const void* blob;
  size_t blob_bytes;
  uint8_t* out;
  int32_t* status;
  void* workspace;
  int n, h, w;
  int nseg;
  int chunk_bits;
  int reserved;
} osvos_jpeg_args;
OSVOS_API size_t osvos_jpeg_decode_workspace_bytes(int n, int h, int w, int nseg, size_t blob_bytes, int chunk_bits);
OSVOS_API int osvos_jpeg_decode(const osvos_jpeg_args* args, osvos_stream_t stream);

/* ---- PNG encoding of 8-bit maps (the result files of train_online.py:187, sm.imsave; DESIGN.md §21) ---------------
 *   osvos_png_encode: src [n][h][w] uint8 (any alignment) -> one complete 8-bit grayscale PNG per frame in
 *                     out [n][osvos_png_max_bytes(h, w)] (frame i's file is out + i * max_bytes, lengths[i] bytes long;
 *                     lengths int64 [n], 8-byte aligned).  Colour type 0, bit depth 8, no interlace, no ancillary
 *                     chunks; the row filter is the least-sum-of-residuals heuristic, the zlib stream uses literals
 *                     and distance-1 matches in one dynamic-Huffman or stored block per segment of filtered rows,
 *                     each segment its own IDAT chunk.  The bytes are a function of the frame alone (not of n, the
 *                     stream or the run).  `workspace`: osvos_png_encode_workspace_bytes(n, h, w) bytes, 16-byte
 *                     aligned, owned by the caller; nothing is allocated and nothing waits for the host.  n < 65536.
 *   osvos_png_max_bytes: the per-frame capacity (every segment stored); 0 unless 1 <= h, w <= 32767.
 *   osvos_png_encode_workspace_bytes: host query; 0 for invalid arguments.                                          */
OSVOS_API size_t osvos_png_max_bytes(int h, int w);
OSVOS_API size_t osvos_png_encode_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_png_encode(const uint8_t* src, uint8_t* out, int64_t* lengths, void* workspace, int n, int h, int w,
                               osvos_stream_t stream);
/*   osvos_png_encode_palette: osvos_png_encode with IHDR colour type 3 (depth 8) and a PLTE chunk of `palette` (host
 *                     memory, 3 * entries bytes RGB, 1 <= entries <= 256) after it; the bytes of each map are written as
 *                     palette indices.  Everything after the PLTE chunk is identical to osvos_png_encode's file of the
 *                     same map.  out [n][osvos_png_max_bytes_palette(h, w, entries)]; the workspace is
 *                     osvos_png_encode_workspace_bytes(n, h, w).
 *   osvos_png_max_bytes_palette: osvos_png_max_bytes(h, w) + 12 + 3 * entries; 0 for invalid arguments.              */
OSVOS_API size_t osvos_png_max_bytes_palette(int h, int w, int entries);
OSVOS_API int osvos_png_encode_palette(const uint8_t* src, const uint8_t* palette, int entries, uint8_t* out,
                                       int64_t* lengths, void* workspace, int n, int h, int w, osvos_stream_t stream);

/* ---- PNG decoding of 8-bit and 1-bit grayscale files and palette files (result and annotation masks; §22, §24) ----
 *   osvos_png_decode: a batch of n PNG files of one size h x w, parsed and packed by osvos_pytorch_b200.png.pack into
 *                     `blob` (blob_bytes bytes, 16-byte aligned: per-file records, segment records, the concatenated
 *                     IDAT payloads) -> out [n][h][w] uint8 (any alignment; gray depth 1 as 0 / 255, palette files at
 *                     depth 1, 2, 4 or 8 as their raw indices, samples MSB first) and status [n] int32.
 *                     Each zlib stream is inflated by one warp per segment when the cuts the host proposed (after an
 *                     IDAT payload ending in 00 00 FF FF) are proven by a counting pass, otherwise by one warp in order;
 *                     a wrong proposal changes neither pixels nor status.  Then the Adler-32 check and the row filters.
 *                     status bits: 1 an invalid block type, code-length set or undefined code, 2 a distance beyond the
 *                     bytes written, 4 a stream that ended early or an output that is not h * (rowbytes + 1) bytes,
 *                     8 an Adler-32 mismatch, 16 a filter type above 4, 32 a header inconsistent with the arguments
 *                     (that file is not decoded).  Pixels of a flagged file are not specified, but the call reads
 *                     nothing outside the blob and writes nothing outside out, status, path and the workspace.
 *                     `path` (int32 [n] or NULL): which pass wrote each file, 1 the segment passes, 2 the in-order
 *                     pass, 0 neither.  `nseg` is the blob's segment count.  `workspace`:
 *                     osvos_png_decode_workspace_bytes(...) bytes, 16-byte aligned, owned by the caller; nothing is
 *                     allocated and nothing waits for the host.  n < 65536, h, w < 32768, blob_bytes < 2^31.
 *   osvos_png_decode_workspace_bytes: host query; 0 for invalid arguments.                                          */
typedef struct osvos_png_decode_args {
  const void* blob;
  size_t blob_bytes;
  uint8_t* out;
  int32_t* status;
  void* workspace;
  int32_t* path;
  int n, h, w;
  int nseg;
} osvos_png_decode_args;
OSVOS_API size_t osvos_png_decode_workspace_bytes(int n, int h, int w, int nseg, size_t blob_bytes);
OSVOS_API int osvos_png_decode(const osvos_png_decode_args* args, osvos_stream_t stream);

/* ---- segmentation overlays as JPEG files (replaces the reference's display: dataloaders/helpers.py:15-40
 *      overlay_mask and the vis_res window of train_online.py:160-205; DESIGN.md §23) ---------------------------------
 *   osvos_overlay_mask: frames [n][h][w][3] uint8 BGR (any alignment) and logits [n][h][w] fp32 (4-byte aligned) ->
 *                     out [n][h][w][3] uint8 (may be frames itself).  fg = logit > 0 (+-0 and NaN are background);
 *                     edge = fg with a 4-neighbour in the background or outside the frame (the pixels
 *                     cv2.drawContours(findContours(mask, RETR_TREE, CHAIN_APPROX_SIMPLE), -1, 0, 1) paints).  Each
 *                     pixel is (0, 0, 0) on the edge, (v + c + 1) >> 1 per channel on the rest of fg (c0, c1, c2 the
 *                     colour in the frame's channel order, 0..255), v elsewhere.
 *   osvos_jpeg_encode: src [n][h][w][3] uint8 BGR (any alignment) -> one baseline JPEG file per frame in
 *                     out [n][osvos_jpeg_max_bytes(h, w)] (frame i's file is out + i * max_bytes, lengths[i] bytes long;
 *                     lengths int64 [n], 8-byte aligned), the bytes cv2.imencode('.jpg', frame,
 *                     [IMWRITE_JPEG_QUALITY, quality]) writes: JFIF, 4:2:0, ISLOW FDCT, the Annex K Huffman tables,
 *                     no restart interval.  1 <= quality <= 100, 1 <= h, w <= 65500, n < 65536.  `workspace`:
 *                     osvos_jpeg_encode_workspace_bytes(n, h, w) bytes, 16-byte aligned, owned by the caller; nothing
 *                     is allocated and nothing waits for the host.
 *   osvos_jpeg_max_bytes: the per-frame capacity: header and EOI plus twice the largest scan (every block at
 *                     22 + 63 x 26 bits, every byte stuffed); 0 for invalid sizes.
 *   osvos_jpeg_encode_workspace_bytes: host query; 0 for invalid arguments.                                          */
OSVOS_API int osvos_overlay_mask(const uint8_t* frames, const float* logits, uint8_t* out, int n, int h, int w, int c0,
                                 int c1, int c2, osvos_stream_t stream);
/*   osvos_overlay_labels: the overlay of a label map of K objects (replaces the reference's dataloaders/helpers.py
 *                     overlay_mask, extended to K objects; DESIGN.md §25): frames [n][h][w][3] uint8 BGR and labels
 *                     [n][h][w] uint8 object ids (both any alignment) -> out [n][h][w][3] uint8 (may be frames itself;
 *                     must not overlap labels).  Per pixel of id k: k == 0 keeps v; k != 0 is (0, 0, 0) on its edge (a
 *                     4-neighbour with another id or outside the frame: per object, the pixels
 *                     cv2.drawContours(findContours(labels == k, RETR_TREE, CHAIN_APPROX_SIMPLE), -1, 0, 1) paints),
 *                     else (v + c_k + 1) >> 1 per channel, c_k = colors->bgr[k] for k < n_colors and (0, 0, 0) past
 *                     it.  `colors` is host memory, passed to the kernel by value; 0 <= n_colors <= 256.  With one id
 *                     and bgr[1] = (0, 0, 255) the bytes are osvos_overlay_mask's.                                  */
#define OSVOS_OVERLAY_MAX_COLORS 256
typedef struct osvos_overlay_colors {
  uint8_t bgr[OSVOS_OVERLAY_MAX_COLORS][3];
} osvos_overlay_colors;
OSVOS_API int osvos_overlay_labels(const uint8_t* frames, const uint8_t* labels, uint8_t* out, int n, int h, int w,
                                   const osvos_overlay_colors* colors /* host */, int n_colors, osvos_stream_t stream);
OSVOS_API size_t osvos_jpeg_max_bytes(int h, int w);
OSVOS_API size_t osvos_jpeg_encode_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_jpeg_encode(const uint8_t* src, uint8_t* out, int64_t* lengths, void* workspace, int n, int h, int w,
                                int quality, osvos_stream_t stream);

/* ---- side-branch tail with general deconvolution weights (DESIGN.md §20)------------------------------------------
 * The reference's eight ConvTranspose2d layers with ANY weights (networks/vgg_osvos.py:45-46,68-69), their centre crop
 * (layers/osvos_layers.py:51-56), cat + fuse (:71-72) and, with a label, the class-balanced BCE terms
 * (layers/osvos_layers.py:28-41); their autograd at train_online.py:141 / train_parent.py:164, including the gradients
 * of upscale[i] / upscale_[i] that the bilinear path never forms.  Scale k: stride s = 2^(k+1), T_k = (2s)^2 taps
 * t = ty * 2s + tx; the four scales' taps are concatenated (offsets 0, 16, 80, 336; OSVOS_UPSAMPLING_TAPS in all).
 *   osvos_upsampling_fold:   vtab [OSVOS_UPSAMPLING_TAPS][16]: V_k[t][ci] = sum_co fuse_w[16k + co] upscale_w[k][ci][co][t]
 *                            (upscale[k] folded with its slice of fuse), atab [OSVOS_UPSAMPLING_TAPS] = upscale_[k] taps.
 *                            Pass vtab and atab as ONE buffer (atab = vtab + 16 * OSVOS_UPSAMPLING_TAPS), 16-byte aligned.
 *   osvos_tail_general_fwd:  out[k<4](y,x) = sum_{<=2x2 src} atab_k[t] p_k(src), out[4] = fuse_bias + sum_k sum_src
 *                            sum_ci vtab_k[t][ci] feat_k[src][ci], from the 16 side features (osvos_conv3x3 cout == 16,
 *                            y_f32) and p_k = channel 0 of their pq.  `sums` / `losses`: osvos_tail_fwd's contract and
 *                            layout, with osvos_tail_general_fwd_sums(n, h, w) doubles (block rows always added in a
 *                            fixed order).
 *   osvos_tail_general_bwd:  from the five upstream gradient maps g_k (label NULL; NULL maps count as zero) or, with a
 *                            label, from dL/dlogit formed on the fly as osvos_tail_loss_bwd does (src = the forward's
 *                            logits, sums = its sums):
 *                              df_k [n,h_k,w_k,64] split-bf16 act: channels 0..15 = dF_k[ci] = sum_t g_4 vtab_k[t][ci]
 *                                   + dp_k score_w[k][ci] with dp_k = sum_t g_k atab_k[t]; channels 16..63 = 0 (the
 *                                   operand of side_prep's tensor-core weight and data gradients);
 *                              red_k [17 T_k + 33] = {H[t][ci] = sum g_4 F[ci] (16 T), gA[t] = sum g_k p (T),
 *                                   sum dp F[ci] (16), sum dp, sum dF[ci] (16)};
 *                              fuse_bias_grad (label mode only).
 *                            workspace: osvos_tail_general_bwd_workspace_bytes(n, h, w) bytes, 4-byte aligned.
 *   osvos_upsampling_grads_finish: d upscale[k][ci][co][t] = fuse_w[16k+co] H_k[t][ci], d upscale_[k] = gA_k,
 *                            d fuse.weight[16k+co] = sum_{ci,t} upscale_w[k][ci][co][t] H_k[t][ci], d score_dsn[k].weight
 *                            = sum dp F, .bias = sum dp, d side_prep[k].bias = sum dF; NULL outputs are skipped, with
 *                            accumulate the values are added to the destinations.
 * Every float reduction of these calls is fixed-order (OSVOS_FLAG_DETERMINISTIC is accepted and changes nothing).  On
 * this path the side branch's gradient w.r.t. a stage output enters the trunk as osvos_unpool_mask's fp32 dside map. */
#define OSVOS_UPSAMPLING_TAPS 1360
typedef struct {
  const float* upscale_w[4];    /* upscale[k].weight [16][16][2s][2s] ([in][out][kH][kW]) */
  const float* upscale1_w[4];   /* upscale_[k].weight [1][1][2s][2s] */
  const float* fuse_w;          /* fuse.weight [64] */
  float* vtab;
  float* atab;
} osvos_upsampling_fold_args;
OSVOS_API int osvos_upsampling_fold(const osvos_upsampling_fold_args* args /* host */, osvos_stream_t stream);
typedef struct {
  const float* feat[4];    /* [n,h_k,w_k,16] fp32 */
  const float* pq[4];      /* [n,h_k,w_k,2] fp32 */
  const float* vtab;
  const float* atab;
  const float* fuse_bias;  /* [1] or NULL */
  float* out[5];           /* each [n,1,h,w] fp32 or NULL */
  const float* label;      /* [n,1,h,w] or NULL */
  double* sums;            /* osvos_tail_general_fwd_sums(n, h, w) doubles (required with label) */
  float* losses;           /* [6] or NULL */
  float loss_weights[5];
  float divisor;
  int n, h, w;
  int flags;
} osvos_tail_general_fwd_args;
OSVOS_API size_t osvos_tail_general_fwd_sums(int n, int h, int w);
OSVOS_API int osvos_tail_general_fwd(const osvos_tail_general_fwd_args* args /* host */, osvos_stream_t stream);
typedef struct {
  const float* feat[4];
  const float* pq[4];
  const float* score_w[4]; /* score_dsn[k].weight [16] */
  const float* vtab;
  const float* atab;
  const float* src[5];     /* gradient maps (label NULL) or the forward's logit maps (label set) */
  const float* label;
  const double* sums;      /* the forward's sums (label mode) */
  const float* upstream;   /* device scalar d(total) or NULL (= 1), label mode */
  float loss_weights[5];
  float divisor;
  void* df_hi[4];          /* [n,h_k,w_k,64] bf16 */
  void* df_lo[4];          /* or NULL (fast precision) */
  float* red[4];           /* [17 T_k + 33] */
  float* fuse_bias_grad;   /* [1] or NULL (label mode) */
  void* workspace;
  int n, h, w;
  int flags;
} osvos_tail_general_bwd_args;
OSVOS_API size_t osvos_tail_general_bwd_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_tail_general_bwd(const osvos_tail_general_bwd_args* args /* host */, osvos_stream_t stream);
typedef struct {
  const float* red[4];
  const float* upscale_w[4];
  const float* fuse_w;
  float* d_upscale_w[4];   /* [16][16][T_k] or NULL */
  float* d_upscale1_w[4];  /* [T_k] or NULL */
  float* d_fuse_w;         /* [64] or NULL */
  float* d_score_w[4];     /* [16] or NULL */
  float* d_score_b[4];     /* [1] or NULL */
  float* d_side_b[4];      /* [16] or NULL */
  int accumulate;
} osvos_upsampling_grads_args;
OSVOS_API int osvos_upsampling_grads_finish(const osvos_upsampling_grads_args* args /* host */, osvos_stream_t stream);

/* ---- online adaptation targets (DESIGN.md §28) ------------------------------------------------------------------
 *   osvos_adaptation_labels: fused logits [n][h][w] fp32 (4-byte aligned) and the last masks last_mask [n][h][w] uint8
 *                         (any alignment) -> labels [n][h][w] fp32 (4-byte aligned) and counts [n][3] int32 (4-byte
 *                         aligned).  Per frame, M = last_mask != 0; E = the pixels p of M with |p - q|² > e² for every
 *                         background pixel q inside the frame (pixels outside the frame are not background; E = M when
 *                         M fills the frame or e = 0); D(p) = min over q in E of |p - q|², exact.  Negative: E non-empty
 *                         and D > d²; positive: not negative and logit > logit_threshold; labels 0 for a negative pixel,
 *                         1 for a positive one, -1 (void) otherwise.  counts = {|E|, #positive, #negative}.  e, d >= 0,
 *                         n < 65536, h, w < 32768.  Four launches (an exact separable squared distance transform, column
 *                         then row pass, for E and again for D), all integer: the result does not depend on the launch
 *                         configuration.  `workspace`: osvos_adaptation_workspace_bytes(n, h, w) bytes, 4-byte aligned,
 *                         owned by the caller; nothing is allocated.  Zeroes counts itself.
 *   osvos_adaptation_workspace_bytes: host query; 0 for a non-positive dimension.                                    */
OSVOS_API size_t osvos_adaptation_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_adaptation_labels(const float* logits, const uint8_t* last_mask, float* labels, int* counts,
                                      void* workspace, int n, int h, int w, float logit_threshold, int erosion_r,
                                      int distance_r, osvos_stream_t stream);

/* ---- dense CRF refinement (DESIGN.md §29) -------------------------------------------------------------------------
 *   osvos_dense_crf:     frames [n][h][w][3] uint8 BGR (any alignment) and `maps` (host array of k device pointers, each
 *                         to fp32 [n][h][w], 4-byte aligned, as osvos_merge_objects) -> out [k][n][h][w] fp32 (4-byte
 *                         aligned): the refined maps r_k = a_k - a_0 of a Potts mean-field with labels 0 (background)
 *                         and 1..k, unary a⁰ = (0, z_1..z_k), `iterations` updates a = a⁰ + w_a·B + w_g·S, Q = softmax(a).
 *                         B: the permutohedral-lattice bilateral filter on (x/theta_a, y/theta_a, R/theta_b, G/theta_b,
 *                         B/theta_b), normalised by its filter of 1; S: the exact 2-D Gaussian of sigma theta_g
 *                         truncated at ceil(3·theta_g), normalised over the pixels inside the frame.  iterations == 0
 *                         copies the maps.  Each frame has its own lattice; lattice vertices are sorted, not hashed, and
 *                         every sum runs in a fixed order: the result does not depend on the launch configuration.  No
 *                         host synchronisation.  1 <= k <= OSVOS_MERGE_MAX_OBJECTS, 1 <= n <= 2048, h, w < 32768,
 *                         6·n·h·w < 2^31, weights finite and >= 0, thetas finite and > 0; a frame size and thetas whose
 *                         lattice coordinates would not fit the packed 64-bit keys are refused before any launch.
 *                         `workspace`: osvos_dense_crf_workspace_bytes(n, k, h, w) bytes, 256-byte aligned, owned by the
 *                         caller; it starts with the n per-frame lattice vertex counts (int32) and their total.
 *   osvos_dense_crf_workspace_bytes: host query; 0 for invalid sizes.                                               */
OSVOS_API size_t osvos_dense_crf_workspace_bytes(int n, int k, int h, int w);
OSVOS_API int osvos_dense_crf(const uint8_t* frames, const float* const* maps, float* out, void* workspace, int n, int k,
                              int h, int w, int iterations, float w_a, double theta_a, double theta_b, float w_g,
                              double theta_g, osvos_stream_t stream);

/* ---- connected components and the component filter (DESIGN.md §30) ----------------------------------------------
 *   osvos_connected_components: masks [n][h][w] uint8 (any alignment; nonzero = foreground) -> labels [n][h][w] int32
 *                         and counts [n] int32 (4-byte aligned): per frame, scipy.ndimage.label of the foreground with
 *                         the cross structure (connectivity 4) or the 3x3 square (8): 0 background, components numbered
 *                         1..counts[f] in the raster order of their first pixels.  Union-find in 32x16 tiles, then
 *                         across tile borders, every link by atomicMin to the smaller root; the roots' ranks come from a
 *                         CUB scan.  The result does not depend on the launch configuration.  h, w < 32768,
 *                         n·h·w < 2^31.  `workspace`: osvos_connected_components_workspace_bytes(n, h, w) bytes,
 *                         256-byte aligned, owned by the caller.
 *   osvos_filter_components: `maps` (host array of k device pointers, each to fp32 [n][h][w], 4-byte aligned, as
 *                         osvos_merge_objects), prior [k][h][w] uint8 (any alignment, nonzero = object) or NULL -> out
 *                         [k][n][h][w] fp32 (4-byte aligned), kept [k][n][h][w] uint8 (0/1) and stats [k][n][4] int32
 *                         (4-byte aligned).  Per object and frame, F = z > 0 (NaN, ±0 are not) and its components C_i at
 *                         `connectivity`; C* the largest (ties: the smallest label).  OSVOS_COMPONENTS_LARGEST keeps
 *                         C*.  OSVOS_COMPONENTS_NEAR keeps every C_i whose exact minimum squared distance to the prior
 *                         mask P is <= radius², or C* when P is empty or none is; P is `prior` for frame 0 (empty when
 *                         NULL) and the kept mask of frame f - 1 after that, so frames are taken in order.  out = z where
 *                         F is false or the component is kept, -z on the pixels of dropped components; kept = the kept
 *                         mask; stats = {components, components kept, |F|, pixels removed}.  Integer after the z > 0
 *                         test: the result does not depend on the launch configuration.  No host synchronisation.
 *                         1 <= k <= OSVOS_MERGE_MAX_OBJECTS, h, w < 32768, n·k·h·w < 2^31, radius >= 0.
 *                         `workspace`: osvos_filter_components_workspace_bytes(n, k, h, w, mode) bytes, 256-byte aligned,
 *                         owned by the caller.
 *   *_workspace_bytes:   host queries; 0 for invalid sizes or mode.                                                */
#define OSVOS_COMPONENTS_LARGEST 0
#define OSVOS_COMPONENTS_NEAR 1
OSVOS_API size_t osvos_connected_components_workspace_bytes(int n, int h, int w);
OSVOS_API int osvos_connected_components(const uint8_t* masks, int* labels, int* counts, void* workspace, int n, int h,
                                         int w, int connectivity, osvos_stream_t stream);
OSVOS_API size_t osvos_filter_components_workspace_bytes(int n, int k, int h, int w, int mode);
OSVOS_API int osvos_filter_components(const float* const* maps, const uint8_t* prior, float* out, uint8_t* kept,
                                      int* stats, void* workspace, int n, int k, int h, int w, int mode, int radius,
                                      int connectivity, osvos_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OSVOS_B200_H_ */
