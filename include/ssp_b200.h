/* ssp_b200.h -- C ABI of libssp_b200.so: the sm_90a (H100) kernels behind the singleshotpose hot path.
 *
 * The reference (microsoft/singleshotpose) has no FFI: its hot path is the Python surface Darknet.forward / RegionLoss.forward /
 * get_region_boxes / pnp.  Each entry point below names the reference code it replaces (file:line under /root/reference);
 * singleshotpose_b200/*.py are the thin Python mirrors of that surface (INTEGRATION.md).  Their ctypes binding is read from this
 * file at import (signatures, SSP_* integer macros, structs): a new entry point is declared here and defined in its kernel file.
 *
 * Conventions: plain pointers and sizes only; every pointer is a DEVICE pointer unless stated; all
 * functions are asynchronous on `stream` (a cudaStream_t passed as void*), never allocate, never
 * synchronise, and return 0 on success or a negative SSP_ERR_* code (ssp_last_error() gives the text).
 * Thread-compatible: distinct host threads may call concurrently on distinct streams.
 *
 * Activation layout ("padded-flat NHWC"): a (N,C,H,W) feature map is a row-major matrix [rows][ld] with
 *   row(n,h,w) = n*(H+1)*(W+1) + (h+1)*(W+1) + (w+1)
 * (one shared zero pad pixel per image row, one shared zero pad row per image); buffers hold
 * ssp_flat_alloc_rows(N,H,W) rows and must be zero-initialised once: kernels only ever write valid rows
 * of operand planes, the zero pads are what makes a 3x3 tap a constant row shift.
 * 16-bit operand planes come as fp16 "hi" (+ optional fp16 "lo", value = hi + lo) -- see DESIGN.md numerics.
 */
#ifndef SSP_B200_H
#define SSP_B200_H
#ifdef __cplusplus
extern "C" {
#endif

#define SSP_OK 0
#define SSP_ERR_ARG (-1)
#define SSP_ERR_CUDA (-2)
#define SSP_ERR_DRIVER (-3)

#define SSP_FMT_F16 0
#define SSP_FMT_BF16 1
#define SSP_IMPL_TC 0    /* wgmma tensor-core kernel, one implicit-GEMM tile per CTA */
#define SSP_IMPL_SIMT 1  /* fp32 CUDA-core kernel (cross-check / bring-up) */
#define SSP_IMPL_BAND 3  /* narrow 3x3 layers: one activation band per kernel row + resident weights (falls back to TC) */
#define SSP_IMPL_TC2 2   /* the SSP_IMPL_TC kernel on sm_90a (kept so that callers selecting it keep working) */
#define SSP_IMPL_BANDT 4 /* few output channels (<= 64 split-fp16, <= 128 single-term): operands swapped, weights on the M side, 128/256 pixels as N (csrc/conv_bandt.cu; falls back to BAND / TC2 / TC when not eligible) */
#define SSP_EPI_F32 0    /* store fp32 */
#define SSP_EPI_STATS 1  /* store fp32 + per-channel sum / sum of squares over valid pixels (fp64) */
#define SSP_EPI_BIAS 2   /* add bias, store fp32 */
#define SSP_EPI_F16 8    /* store fp16 (saturating to +-65504, NaN stays NaN): `out` points to 16-bit elements, out_ld in elements; data gradients only (TC / TC2 / BANDT kernels) */
#define SSP_ROUTE_NONE 0
#define SSP_ROUTE_DIRECT 1 /* consumer has the same geometry */
#define SSP_ROUTE_POOL 2   /* consumer is behind MaxPool2d(2,2)          (darknet.py:168-176) */
#define SSP_ROUTE_REORG 3  /* consumer is behind Reorg(2), marvis order  (darknet.py:16-35)   */
#define SSP_ROUTE_F16 16   /* OR-ed into a g*_route of ssp_bn_bwd_*: that upstream gradient plane holds fp16 (written with SSP_EPI_F16) instead of fp32 */

int ssp_version(void);
const char* ssp_last_error(void);              /* host pointer, thread-local text of the last failure */
long long ssp_flat_alloc_rows(int N, int H, int W);
long long ssp_flat_row(int n, int h, int w, int H, int W);

/* ---- layout: train.py:83 `data.cuda()` hands NCHW fp32; the conv stack runs on padded-flat rows ---- */
int ssp_pack_nchw(const float* x_nchw, void* hi, void* lo_or_null, int N, int C, int H, int W, int ld, int c0,
                  int fmt, float scale, void* stream);
int ssp_unpack_nchw(const float* y_flat, float* out_nchw, int N, int C, int H, int W, int ld, int c0, void* stream);
int ssp_unpack16_nchw(const void* hi, const void* lo_or_null, float* out_nchw, int N, int C, int H, int W, int ld,
                      int c0, int fmt, void* stream);

/* ---- nn.Conv2d forward and data gradient (darknet.py:156-160; autograd of train.py:103) ----
 * out[m][n] = sum_tap sum_c A[m + shift(tap)][c] * B[n][tap*cin + c],  taps in {1, 9} (3x3 pad 1 / 1x1). */
int ssp_conv_gemm(int impl, const void* a_hi, const void* a_lo_or_null, long long a_rows, int a_ld, int cin,
                  const void* b_hi, const void* b_lo_or_null, int b_rows, int b_ld, int a_fmt, int b_fmt,
                  int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows, int epi,
                  const float* bias, double* stat_sum, double* stat_sq, void* stream);
/* number of launches of the operand-swapped kernel (SSP_IMPL_BANDT) so far in this process: lets a test tell the kernel from its fall-backs */
int ssp_conv_bandt_launches(void);
/* ---- inference: nn.Conv2d + nn.BatchNorm2d(eval) + nn.LeakyReLU as ONE kernel (darknet.py:154-164 under model.eval()):
 *      z = leaky(conv * scale[c] + shift[c]) is written by the GEMM epilogue straight into the consumer's fp16 hi/lo operand
 *      planes (rows [row][d_ld], channel offset d_c0); scale/shift from ssp_bn_finalize(train=0).  fp16 hi/lo operands.
 *      The parts are saturating: hi = fp16(clamp(z, +-65504)), lo = fp16(clamp(z - hi, +-65504)), so a finite z never gives
 *      an infinite part (ssp_bn_apply and ssp_pack_nchw split the same way).  SSP_ERR_ARG unless cout % 32 == 0, d_hi and d_lo
 *      are 16-B aligned, d_ld % 8 == 0, d_c0 % 8 == 0 and d_ld >= d_c0 + cout. ---- */
int ssp_conv_gemm_bnact(int impl, const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                        const void* b_hi, const void* b_lo, int b_rows, int b_ld, int N, int H, int W, int taps, int cout,
                        const float* scale, const float* shift, float slope, void* d_hi, void* d_lo, int d_ld, int d_c0,
                        void* stream);
/* ---- inference split-K for few output tiles (one camera frame): the per-tap tensor-core kernel with each output tile's K range
 *      (taps x ceil(cin/64) k-blocks) cut into `splits` slices; slice s walks k-blocks [s*kb/S, (s+1)*kb/S) and stores its fp32
 *      partial sums unmodified (plain stores, no atomics) into slab s of partial[splits][slab_elems] (rows [row][partial_ld]).
 *      ssp_bn_apply_splitk then sums the slabs in the order s = 0..S-1 and applies BN(running stats) + leaky + routing exactly as
 *      ssp_bn_apply does (no arg-max plane: inference only); splits = 1 runs ssp_bn_apply's kernel.
 *      A result is bit-identical across launches and graph replays; it is NOT bit-identical across batch sizes or shapes whose
 *      split count differs (the partial sums are added in a different order).
 *  ssp_conv_gemm_splitk: fp16 hi/lo operands (3 terms) or single-term fp16 (b_lo / a_lo NULL).  SSP_ERR_ARG for splits < 1,
 *      splits above the k-block count, a NULL or non-16-B-aligned workspace, partial_ld % 4 != 0 or < cout, and slabs
 *      (slab_elems) smaller than ssp_flat_alloc_rows(N, H, W) * partial_ld, i.e. a workspace under splits * that size.
 *  ssp_conv_splitk_count: the split rule, S = min(num_sms / tiles, k-blocks / 8), 1 when that is below 2 (tiles = 128-row x
 *      N-tile output tiles of the per-tap kernel).  Host only. ---- */
int ssp_conv_gemm_splitk(const void* a_hi, const void* a_lo_or_null, long long a_rows, int a_ld, int cin, const void* b_hi,
                         const void* b_lo_or_null, int b_rows, int b_ld, int N, int H, int W, int taps, int cout, int splits,
                         float* partial, long long slab_elems, int partial_ld, void* stream);
int ssp_conv_splitk_count(int N, int H, int W, int taps, int cin, int cout, int num_sms);
int ssp_bn_apply_splitk(const float* partial, int splits, long long slab_elems, int partial_ld, const float* scale, const float* shift,
                        int N, int C, int H, int W, float slope, void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_route,
                        void* d1_hi, void* d1_lo, int d1_ld, int d1_c0, int d1_route, void* stream);
/* ---- blocks 0-1 of cfg/yolo-pose.cfg as a unit -- nn.Conv2d(3,32,3,1,1) + BatchNorm2d + LeakyReLU + MaxPool2d(2,2) (darknet.py:154-167)
 *      and their autograd (train.py:103) -- without materialising the full-resolution conv output (csrc/l0_fused.cu).
 *      gram: double[SSP_L0_GRAM_DOUBLES]; the first 28*28 hold the matrix (upper triangle: sums of q q^T over all pixels, q = (27 patch
 *      values, 1)), kept from forward to backward; the rest is scratch of ssp_l0_gram (shift correlations, border sums);
 *      code: uint8 [pooled rows][32] (bits 0-1 arg-max position of the 2x2 window, bit 2 pre-activation > 0);
 *      t1: double[28*32] scratch (27 x 32 patch-weighted gradient sums + the 32 plain sums).  w = fp32 master weights [32][27].
 *      ssp_l0_stats writes the per-channel sum / sum of squares that ssp_bn_finalize(count = N*H*W) expects. ---- */
#define SSP_L0_GRAM_DOUBLES 2816
int ssp_l0_gram(const float* x_nchw, int N, int H, int W, double* gram, void* stream);
int ssp_l0_stats(const double* gram, const float* w, double* stat_sum, double* stat_sq, void* stream);
int ssp_l0_fused_fwd(const float* x_nchw, const float* w, const float* scale, const float* shift, float slope, int N, int H, int W,
                     void* d_hi, void* d_lo, int d_ld, int d_c0, unsigned char* code_or_null, void* stream);
int ssp_l0_bwd(const float* x_nchw, const void* g_pooled, int g_f16, int g_ld, int g_c0, const unsigned char* code, float slope, int N,
               int H, int W, double* t1, void* stream);   /* g_f16: the pooled gradient plane holds fp16 (SSP_EPI_F16) instead of fp32 */
int ssp_l0_bwd_finalize(const double* t1, const double* gram, const float* w, const float* gamma, const float* mean,
                        const float* invstd, double count, float grad_scale, float* dw, float* dgamma, float* dbeta, void* stream);
/* ---- nn.Conv2d weight gradient: dW[co][tap][ci] += scale * sum_m dY[m][co] * X[m + shift(tap)][ci] ---- */
int ssp_wgrad_gemm(int impl, const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt, const void* x,
                   long long x_rows, int x_ld, int cin, int x_fmt, int N, int H, int W, int taps, float* dw,
                   int dw_ld, int cin_store, float scale, void* stream);

/* ---- nn.BatchNorm2d(eps=1e-4) + nn.LeakyReLU(0.1) + MaxPool2d/Reorg/route placement (darknet.py:96-106,157-176) ---- */
int ssp_bn_finalize(double* stat_sum, double* stat_sq, double count, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, float momentum, float eps, int train, float* mean,
                    float* invstd, float* scale, float* shift, int C, void* stream);
/* ypool (optional, max-pool destinations only): fp32 plane in the POOLED geometry receiving the conv output y at the arg-max
 * position of every 2x2 window.  With it the first pass of the BN backward of a pooled layer runs at a quarter of the
 * resolution: ssp_bn_bwd_reduce(y = ypool, H/2, W/2, g0 = pooled upstream gradient, SSP_ROUTE_DIRECT) accumulates the same
 * S1 / S2 as the full-resolution call (only arg-max positions receive gradient).
 * Layout rules (4-channel vectors; SSP_ERR_ARG before any launch otherwise), for ssp_bn_apply, ssp_bn_apply_splitk and the
 * ssp_bn_bwd_* calls: C % 4 == 0; y (and ypool) 16-B aligned with ld % 4 == 0 and ld >= C; every destination plane (hi, lo) 8-B
 * aligned and every upstream gradient plane 16-B (fp32) or 8-B (SSP_ROUTE_F16) aligned, each with ld % 4 == 0, c0 % 4 == 0 and
 * ld >= c0 + C (c0 + 4C behind SSP_ROUTE_REORG); dy of ssp_bn_bwd_apply 8-B aligned with dy_ld % 4 == 0 and dy_ld >= C. */
int ssp_bn_apply(const float* y, int y_ld, const float* scale, const float* shift, int N, int C, int H, int W,
                 float slope, void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_route, void* d1_hi, void* d1_lo,
                 int d1_ld, int d1_c0, int d1_route, float* ypool_or_null, int ypool_ld, void* stream);
int ssp_bn_bwd_reduce(const float* y, int y_ld, const float* scale, const float* shift, const float* mean,
                      const float* invstd, const float* gamma, int N, int C, int H, int W, float slope,
                      const float* g0, int g0_ld, int g0_c0, int g0_route, const float* g1, int g1_ld, int g1_c0,
                      int g1_route, double* s1, double* s2, void* stream);
int ssp_bn_bwd_apply(const float* y, int y_ld, const float* scale, const float* shift, const float* mean,
                     const float* invstd, const float* gamma, int N, int C, int H, int W, float slope,
                     const float* g0, int g0_ld, int g0_c0, int g0_route, const float* g1, int g1_ld, int g1_c0,
                     int g1_route, double* s1, double* s2, void* dy, int dy_ld, int dy_fmt, float dy_scale,
                     void* stream);
int ssp_bn_bwd_finalize(double* s1, double* s2, float* dgamma, float* dbeta, int C, int accumulate, float scale,
                        void* stream);
int ssp_bias_grad_nchw(const float* g_nchw, float* dbias, int N, int C, int HW, int accumulate, float scale,
                       void* stream);

/* ---- parameters: weight re-pack from the fp32 master [cout][taps][cin]; optim.SGD (train.py:388) ---- */
int ssp_pack_weights(const float* w, int cout, int taps, int cin, void* fwd_hi, void* fwd_lo, int fwd_ld,
                     void* dgrad, int dgrad_ld, int dgrad_fmt, void* stream);
int ssp_sgd_step_flat(float* p, const float* g, float* v, long long n, float lr, float momentum,
                      float weight_decay, float grad_scale, void* stream);
/* SGD and the operand-plane re-pack in ONE pass over the flat buffers (csrc/sgd_pack.cu).  `segments` is a DEVICE array with one
 * entry per parameter tensor in flat-buffer order; taps == 0 marks a tensor without operand planes (BN affine, bias).  A conv
 * weight [cout][taps][cin] owns ssp_sgd_segment_blocks() consecutive blocks starting at block0 (prefix sum, filled by the
 * caller); a launch covers blocks [block_begin, block_end), i.e. any run of whole segments: the data-parallel path updates one
 * gradient bucket at a time.  Writes p, v and -- where the pointers are non-null -- W_hi / W_lo [cout][ld_f] (k = tap*cin + ci)
 * and W_d [cin][ld_d] (k = (taps-1-tap)*cout + co), exactly the bytes ssp_pack_weights would produce from the updated p. */
typedef struct ssp_sgd_segment {
  long long off, n;                 /* element offset and count inside the flat buffers */
  int cout, taps, cin;              /* conv weight geometry; taps == 0: plain tensor */
  int ld_f, ld_d, d_fmt;            /* row pitches (elements) of the planes; SSP_FMT_* of W_d */
  void* f_hi; void* f_lo; void* d;  /* device planes, each may be NULL */
  int block0, reserved;
} ssp_sgd_segment;
int ssp_sgd_segment_blocks(int cout, int taps, int cin, long long n);
int ssp_sgd_pack_step(const ssp_sgd_segment* segments_dev, int n_segments, int block_begin, int block_end, float* p,
                      const float* g, float* v, float lr, float momentum, float weight_decay, float grad_scale,
                      void* stream);

/* ---- RegionLoss.forward + build_targets + gradient (region_loss.py:9-175); acc = 8 doubles:
 *      loss_x, loss_y, loss_conf, nGT, nCorrect, nProposals ---- */
int ssp_region_loss_fwd_bwd(const float* out_nchw, const float* target, float* grad_nchw_or_null, double* acc,
                            int B, int num_keypoints, int num_classes, int H, int W, float coord_scale,
                            float noobject_scale, float object_scale, float thresh, int use_conf,
                            float grad_scale, void* stream);
/* ---- get_region_boxes (utils.py:216-296): boxes[B][2K+3] per image, box_global[2K+3] = reference semantics ---- */
int ssp_region_decode_argmax(const float* out_nchw, int B, int num_keypoints, int num_classes, int H, int W,
                             int only_objectness, float* boxes, float* best_conf, float* box_global_or_null,
                             void* stream);

/* ---- multi-object head (multi_obj_pose_estimation/region_loss_multi.py:9-189, utils_multi.py:266-382).
 *      `anchors` is a HOST array of num_anchors*anchor_step floats; acc[6] additionally holds loss_cls.
 *      decode: dense per (image, cell, anchor) arrays in the reference's visiting order + its sequential fallback maxima ---- */
int ssp_region_loss_multi_fwd_bwd(const float* out_nchw, const float* target, float* grad_nchw_or_null, double* acc,
                                  int B, int num_keypoints, int num_classes, int num_anchors, int H, int W,
                                  const float* anchors_host, int anchor_step, float coord_scale, float noobject_scale,
                                  float object_scale, float class_scale, float thresh, int use_conf, float grad_scale,
                                  void* stream);
int ssp_region_decode_multi(const float* out_nchw, int B, int num_keypoints, int num_classes, int num_anchors, int H,
                            int W, int only_objectness, int correspondingclass, float* boxes, float* conf_sel,
                            float* det_conf, float* cls_corr, long long* max_ind, float* max_conf, float* max_cls,
                            void* stream);
/* ---- multi-object evaluation (valid_multi.py:97-132, train_multi.py:196-240): per image, as the reference's batch-1 call, the
 *      box list of get_multi_region_boxes(..., int(target[b][0]), only_objectness=0) and the box chosen for each ground truth.
 *      target (B, target_stride) fp32 device, rows [cls, x0, y0, ..., x8, y8, w, h]; gt_offset (B+1) device: prefix sums of the
 *      number of ground truths per image (G = gt_offset[B]).  Out: boxes [G][2K+3] the chosen box; flags [G] bit 0 = fallback box,
 *      bit 1 = carried over from the previous ground truth of the image; uv [2G][K][2] pixels, the G ground truths after
 *      fix_corner_order, then the G predictions: the points of ssp_pnp_batched.  num_keypoints must be 9 and
 *      H*W*num_anchors at most 4096 (SSP_ERR_ARG otherwise). ---- */
int ssp_eval_multi_select(const float* out_nchw, int B, int num_keypoints, int num_classes, int num_anchors, int H, int W,
                          const float* target, int target_stride, const int* gt_offset, float conf_thresh, float im_width,
                          float im_height, float* boxes, int* flags, float* uv, void* stream);
/* ---- multi-object prediction (no labels): per image b and requested class classes_host[q], the box ssp_eval_multi_select would
 *      choose for a one-row target of that class -- the listed box of class c with the largest det_conf (first in visiting order),
 *      else the fallback box of get_multi_region_boxes(..., correspondingclass = c) -- each image as its own batch-1 call.
 *      classes_host: n_req distinct class ids in [0, num_classes), a HOST array copied into the launch.  Out: boxes
 *      [B][n_req][2K+3]; flags [B][n_req], bit 0 = fallback box (the class was not listed); uv [B][n_req][K][2] = the box
 *      keypoints times (frame_w, frame_h) in fp32, the points of ssp_pnp_batched.  SSP_ERR_ARG for a null pointer,
 *      num_keypoints != 9, H*W*num_anchors > 4096, num_classes > 256, n_req < 1, or a class out of range or listed twice. ---- */
int ssp_predict_multi_select(const float* out_nchw, int B, int num_keypoints, int num_classes, int num_anchors, int H, int W,
                             const int* classes_host, int n_req, float conf_thresh, float frame_w, float frame_h, float* boxes,
                             int* flags, float* uv, void* stream);
/* ---- every instance in a frame (rules: csrc/detect_core.h): per image b, each as its own call, the candidates are the boxes
 *      get_multi_region_boxes(..., only_objectness=0) lists (det_conf * cls_max_conf > conf_thresh, no fallback box) whose arg-max
 *      class is requested, in descending (det_conf, then lower entry) order; greedy suppression within each class drops a
 *      candidate whose rectangle of the 8 corner keypoints (frame pixels) has fp32 IoU > nms_thresh with a kept box of its class.
 *      The reference's nms (YOLO boxes) is not reproduced.  classes_host: n_req distinct class ids, a HOST array copied into the
 *      launch.  Out: boxes [B][max_instances][2K+3], cls [B][max_instances], uv [B][max_instances][K][2] (the box keypoints times
 *      (frame_w, frame_h) in fp32) of the first max_instances kept boxes in that order; slots >= count[b] are zero with cls -1;
 *      count [B] = min(kept, max_instances), kept [B] = boxes kept before the truncation.  SSP_ERR_ARG for a null pointer,
 *      num_keypoints != 9, H*W*num_anchors > 4096, num_classes > 256, n_req < 1, a class out of range or listed twice,
 *      nms_thresh outside [0, 1] or max_instances outside [1, 256]. ---- */
int ssp_detect_instances(const float* out_nchw, int B, int num_keypoints, int num_classes, int num_anchors, int H, int W,
                         const int* classes_host, int n_req, float conf_thresh, float nms_thresh, int max_instances, float frame_w,
                         float frame_h, float* boxes, int* cls, float* uv, int* count, int* kept, void* stream);

/* ---- pnp (utils.py:86-100 -> cv2.solvePnP ITERATIVE + Rodrigues), compute_projection (utils.py:40-45) ---- */
int ssp_pnp_batched(const float* points3d, int points3d_shared, const float* points2d, const float* K3x3,
                    int num_points, long long n, int max_iter, double* R_out, double* t_out,
                    int* iters_out_or_null, void* stream);
/* same solve; work_out [n][3] int = {Jacobi sweeps of the 12x12 DLT, accepted LM iterations, LM linear solves} per problem: what the
 * bench's achieved-FLOP/s figure is computed from */
int ssp_pnp_batched_work(const float* points3d, int points3d_shared, const float* points2d, const float* K3x3,
                         int num_points, long long n, int max_iter, double* R_out, double* t_out, int* work_out,
                         void* stream);
/* same solve over groups x per_group problems with per-problem points3d [groups*per_group][num_points][3]: problem (g, m) is
 * solved only when m < count[g] (count: DEVICE int [groups], so a graph replay needs no host read-back); the others get zero
 * R and t.  The slots of ssp_detect_instances are such groups. */
int ssp_pnp_batched_counted(const float* points3d, const float* points2d, const float* K3x3, int num_points, int groups,
                            int per_group, const int* count, int max_iter, double* R_out, double* t_out, void* stream);
/* the counted solve where problem i with use_guess[i] != 0 starts Levenberg-Marquardt from guess [i][6] = (rvec, t) and skips the
 * DLT, as cv2.solvePnP(..., useExtrinsicGuess=True) does; the others are solved as by ssp_pnp_batched_counted (bit-identical R, t).
 * guess, use_guess: DEVICE [groups*per_group][6] fp64 and [groups*per_group] int.  Out: params_out [n][6] fp64 = the final LM vector
 * (cv2's rvec, tvec); work_out_or_null [n][3] as ssp_pnp_batched_work (0 DLT sweeps for a warm start).  Empty slots get zeros. */
int ssp_pnp_batched_guess(const float* points3d, const float* points2d, const float* K3x3, int num_points, int groups,
                          int per_group, const int* count, const double* guess, const int* use_guess, int max_iter, double* R_out,
                          double* t_out, double* params_out, int* work_out_or_null, void* stream);
/* ---- consensus PnP over keypoint subsets (rule: csrc/pnp_consensus_core.h): a pose that survives wrong keypoints.  Per problem,
 *      hypothesis 0 is the plain cold solve on all num_points points and hypothesis h >= 1 the cold solve on the 6 points of
 *      subsets_host[h-1]; each is scored on all points (no inliers if any point lies at camera depth <= 0, else point i is an inlier
 *      when its squared reprojection error <= reproj_thresh^2 px^2); the one with the most inliers wins, the lower index on a tie.
 *      If its inliers differ from its own points and number >= 6, LM refines it on them from its pose (useExtrinsicGuess).  When
 *      hypothesis 0 has every point as an inlier the result is bit-identical to ssp_pnp_batched.
 *      points3d [n][num_points][3], or one shared [num_points][3] when points3d_shared != 0; n = groups * per_group problems.
 *      count_or_null: DEVICE int [groups] as ssp_pnp_batched_counted (problem (g, m) is solved only when m < count[g], the others
 *      get zeros), or NULL to solve all n.  subsets_host: n_subsets (1..210) HOST uint16 masks of exactly 6 bits below num_points,
 *      copied into the launch; their order is the tie-break order.  work: DEVICE scratch (8-B aligned) of at least the
 *      *bytes_out (a HOST long long) that ssp_pnp_consensus_work_bytes(num_points, n_subsets, n, bytes_out) writes.  Out: R_out [n][9], t_out [n][3], params_out [n][6] (the
 *      final LM vector: rvec, t), inliers_out [n] int bitmask of the chosen hypothesis's inliers (bit i = point i), hyp_out [n]
 *      (the chosen hypothesis, -1 when none has an inlier: hypothesis 0's pose with an empty mask).  SSP_ERR_ARG for a null pointer,
 *      num_points outside 7..10, a bad table, reproj_thresh <= 0 or not finite, max_iter < 1, groups < 0, per_group < 1 or a
 *      workspace that is too small (ssp_pnp_consensus_work_bytes returns SSP_ERR_ARG for bad sizes or a null bytes_out). ---- */
int ssp_pnp_consensus_work_bytes(int num_points, int n_subsets, long long n, long long* bytes_out);
int ssp_pnp_consensus(const float* points3d, int points3d_shared, const float* points2d, const float* K3x3, int num_points, int groups,
                      int per_group, const int* count_or_null, const unsigned short* subsets_host, int n_subsets, double reproj_thresh,
                      int max_iter, double* R_out, double* t_out, double* params_out, int* inliers_out, int* hyp_out, void* work,
                      long long work_bytes, void* stream);

/* ---- tracking instances across frames (rules: csrc/track_core.h): each row b is its own camera stream with T = max_tracks slots
 *      (1 <= T <= 256).  The state is four DEVICE arrays, zeroed for a fresh start (alive 0, ids from 0):
 *        tracks  int    [B][T][5]  alive, id, cls, misses (consecutive frames unmatched), hits;  fields of a slot with alive 0 are stale
 *        rects   float  [B][T][4]  x0, y0, x1, y1: the corner rectangle of the track's last detection in frame pixels
 *        poses   double [B][T][6]  rvec, t: the final Levenberg-Marquardt vector of the track's last solve
 *        next_id int    [B]        the id the next new track of the stream gets
 *      The detections are ssp_detect_instances' outputs for the frame: count [B], cls [B][max_det], uv [B][max_det][9][2].
 *      ssp_track_associate matches the detections to the alive tracks of their class (highest corner-rectangle IoU > match_iou, in
 *      detector order), ages the unmatched tracks (a track dies at misses > max_misses) and gives each unmatched detection the lowest
 *      free slot and the next id.  Out per detection slot: slot [B][max_det] (the track slot, -1 for an empty or untracked slot),
 *      track_id [B][max_det] (-1 likewise), guess [B][max_det][6] fp64 (the matched track's pose, else 0) and use_guess [B][max_det]
 *      (1 when matched): the inputs of ssp_pnp_batched_guess.  ssp_track_commit then stores each matched or born track's rectangle,
 *      the solve's params [B][max_det][6] (ssp_pnp_batched_guess' params_out), misses = 0 and hits + 1.  SSP_ERR_ARG for a null
 *      pointer, B < 0, max_tracks or max_det outside [1, 256], match_iou outside [0, 1] or max_misses < 0. ---- */
int ssp_track_associate(int B, int max_tracks, int max_det, const int* count, const int* cls, const float* uv, float match_iou,
                        int max_misses, int* tracks, const float* rects, const double* poses, int* next_id, int* slot, int* track_id,
                        double* guess, int* use_guess, void* stream);
int ssp_track_commit(int B, int max_tracks, int max_det, const int* count, const float* uv, const int* slot, const double* params,
                     int* tracks, float* rects, double* poses, void* stream);
int ssp_project_points(const float* X, int rows, int nv, const double* Rt, const double* K3x3, long long n,
                       float* out, void* stream);

/* ---- cameras with lens distortion (utils.py:86-100 with pnp.distCoeffs -> cv2.solvePnP(..., distCoeffs); csrc/pnp_dist.cu).
 *      dist8: DEVICE double [8] = OpenCV's (k1, k2, p1, p2, k3, k4, k5, k6), read in place (a graph replay sees its current values);
 *      NULL is SSP_ERR_ARG: zero distortion is the entry points above.  The PnP undistorts the keypoints as cv2.undistortPoints does
 *      (5 fixed-point iterations) for the DLT and fits the raw keypoints with cv2.projectPoints' distorted model in the LM.
 *  ssp_pnp_dist: groups x per_group problems, points3d shared or [n][num_points][3] as ssp_pnp_batched.  count_or_null: DEVICE int
 *      [groups] as ssp_pnp_batched_counted (empty slots get zeros, also in params and work), NULL to solve all.  guess_or_null with
 *      use_guess_or_null (both or neither): warm starts as ssp_pnp_batched_guess, which need params_out.  params_out_or_null [n][6]
 *      the final LM vector; work_out_or_null [n][3] as ssp_pnp_batched_work.  SSP_ERR_ARG for a null required pointer, num_points
 *      outside 6..16, groups < 0, per_group < 1, guess without use_guess (or the reverse) or guess without params_out.
 *  ssp_pnp_consensus_dist: ssp_pnp_consensus with every solve and the scoring distorted; same workspace (ssp_pnp_consensus_work_bytes),
 *      same checks, plus a null dist8.
 *  ssp_project_points_dist: cv2.projectPoints(X, R, t, K, dist) in ssp_project_points' layout (fp64 math, fp32 out [n][2][nv]; with
 *      rows == 4 the translation is scaled by the homogeneous coordinate).  SSP_ERR_ARG for a null pointer, rows not 3 or 4, nv < 0
 *      or n < 0. ---- */
int ssp_pnp_dist(const float* points3d, int points3d_shared, const float* points2d, const float* K3x3, const double* dist8,
                 int num_points, int groups, int per_group, const int* count_or_null, const double* guess_or_null,
                 const int* use_guess_or_null, int max_iter, double* R_out, double* t_out, double* params_out_or_null,
                 int* work_out_or_null, void* stream);
int ssp_pnp_consensus_dist(const float* points3d, int points3d_shared, const float* points2d, const float* K3x3, const double* dist8,
                           int num_points, int groups, int per_group, const int* count_or_null, const unsigned short* subsets_host,
                           int n_subsets, double reproj_thresh, int max_iter, double* R_out, double* t_out, double* params_out,
                           int* inliers_out, int* hyp_out, void* work, long long work_bytes, void* stream);
int ssp_project_points_dist(const float* X, int rows, int nv, const double* Rt, const double* K3x3, const double* dist8,
                            long long n, float* out, void* stream);

/* ---- pose covariance and the constant-velocity pose filter of tracked instances (rules: csrc/pose_filter_core.h; csrc/pose_filter.cu),
 *      fp64.  A pose is perturbed on the left, x_cam = exp([dth]x) R X + t + dt_, and a 6 x 6 covariance is over (dth, dt_).
 *  ssp_pose_covariance: Sigma = sigma^2 (J^T J)^-1 of the pose (R, t) of each problem, J the pixel projection of its points with
 *      respect to (dth, dt_) (distorted with dist8_or_null, a DEVICE double [8] as ssp_pnp_dist takes it; NULL: no distortion).  The
 *      keypoints do not enter: J is taken at the solved pose.  points3d shared or [n][num_points][3], K3x3 fp32, count_or_null as
 *      ssp_pnp_dist; R [n][9], t [n][3] the solutions (ssp_pnp_* outputs).  Out: cov_out [n][6][6], status_out [n] = 0 (usable) or
 *      SSP_POSE_COV_SINGULAR (a Cholesky pivot <= 1e-12 x the largest diagonal entry of J^T J) | SSP_POSE_COV_DEPTH (a point at
 *      depth <= 0); an unusable or empty slot gets zeros.  SSP_ERR_ARG for a null required pointer, num_points outside 3..16,
 *      groups < 0, per_group < 1 or sigma not > 0 and finite.
 *  The filter of each (stream, track slot) is filter [B][max_tracks][SSP_FILTER_DOUBLES] fp64 = R [9], t [3], w [3] (rad/s, camera
 *      frame), v [3] (mesh units / s), P [12][12] over (dth, dt_, dw, dv), valid; zeros for a fresh start.
 *  ssp_track_predict: for every alive slot whose filter has started, moves the filter by dt [B] seconds (DEVICE fp64, one per stream)
 *      in place, and writes the predicted LM vector (log R, t) to pred_poses [B][max_tracks][6] and the predicted corner rectangle to
 *      pred_rects [B][max_tracks][4]: the 8 corners points3d_table [cls][1..8] (fp32 [num_classes][9][3]) of the slot's class
 *      projected with K3x3 (fp64; distorted with dist8_or_null) and rounded to fp32.  Any other slot, and a slot with a predicted
 *      corner at depth <= 0, passes its rects / poses on.  The two outputs take the place of rects / poses in ssp_track_associate.
 *      SSP_ERR_ARG for a null required pointer, B < 0, max_tracks outside [1, 256], num_classes < 1 or an accel sigma not > 0 and finite.
 *  ssp_track_filter_update: after ssp_track_commit, per detection slot with a track slot (slot >= 0, m < count[b]): a new track
 *      (use_guess 0) starts its filter from the measurement R, t (the frame's PnP) with covariance cov / cov_status
 *      (ssp_pose_covariance), a matched one is gated (y^T S^-1 y > gate restarts it) and updated.  Out per detection slot: R_filt
 *      [9], t_filt [3], pose_cov [6][6], velocity [6] = (w, v), reinit (1: the filter was started from this measurement); zeros
 *      elsewhere.  SSP_ERR_ARG for a null pointer, B < 0, max_tracks or max_det outside [1, 256], or an init velocity sigma or the
 *      gate not > 0 and finite. ---- */
#define SSP_POSE_COV_SINGULAR 1
#define SSP_POSE_COV_DEPTH 2
#define SSP_FILTER_DOUBLES 163
int ssp_pose_covariance(const float* points3d, int points3d_shared, const float* K3x3, const double* dist8_or_null, int num_points,
                        int groups, int per_group, const int* count_or_null, const double* R, const double* t, double sigma,
                        double* cov_out, int* status_out, void* stream);
int ssp_track_predict(int B, int max_tracks, const int* tracks, const float* rects, const double* poses, double* filter, const double* dt,
                      const float* points3d_table, int num_classes, const double* K3x3, const double* dist8_or_null,
                      double accel_sigma_rot, double accel_sigma_trans, double* pred_poses, float* pred_rects, void* stream);
int ssp_track_filter_update(int B, int max_tracks, int max_det, const int* count, const int* slot, const int* use_guess,
                            const double* R, const double* t, const double* cov, const int* cov_status, double* filter,
                            double init_velocity_sigma_rot, double init_velocity_sigma_trans, double gate, double* R_filt,
                            double* t_filt, double* pose_cov, double* velocity, int* reinit, void* stream);

/* ---- refinement of poses against registered depth frames: projective point-to-plane ICP (rules: csrc/refine_depth_core.h;
 *      csrc/refine_depth.cu), fp64, one 256-thread CTA per problem, every iteration in one launch.
 *  ssp_refine_depth: groups x per_group problems, group g = depth frame depth [g][H][W] (uint16, 0 = no measurement; depth_scale
 *      mesh units per depth unit, 0.001 for millimetre depth and metre meshes), registered to the camera K3x3 (DEVICE fp64) with
 *      dist8_or_null (a DEVICE double [8] as ssp_pnp_dist takes it; NULL: no distortion).  model [total][6] fp64 = (x, y, z, nx,
 *      ny, nz) of every class's points with unit outward normals, class c's rows offsets[c] .. offsets[c + 1] - 1 (DEVICE int
 *      [num_classes + 1]), diam [num_classes] (DEVICE fp64) its diameter; cls [groups][per_group] (DEVICE int) each problem's class.
 *      count_or_null: DEVICE int [groups] as ssp_pnp_batched_counted (problems at m >= count[g] get zeros and status 0).  R [n][9],
 *      t [n][3] the input poses (camera from model).  iters fixed iterations at the gates diam * g_k, g_k = gate_start *
 *      (gate_end / gate_start)^(k / (iters - 1)): a pair whose depths differ by more is dropped.  Out: R_out, t_out the refined
 *      pose; points_out [n] the pair count and rmse_out [n] the point-to-plane RMS residual of the last iteration (before its
 *      update); status_out [n] 0 or SSP_REFINE_FEW_POINTS (an iteration had fewer than SSP_REFINE_MIN_POINTS pairs; also a class
 *      outside [0, num_classes)) | SSP_REFINE_SINGULAR (a Cholesky pivot of J^T J <= 1e-12 x its largest diagonal entry) |
 *      SSP_REFINE_BAD_POSE (the input pose is not finite or has t_z <= 0).  With a status bit the output pose is the input pose.
 *      SSP_ERR_ARG for a null required pointer, W or H outside [1, 16384], num_classes < 1, groups < 0, per_group < 1, iters
 *      outside [1, SSP_REFINE_MAX_ITERS], a gate not > 0 and finite or gate_end > gate_start, or depth_scale not > 0 and finite. ---- */
#define SSP_REFINE_MIN_POINTS 50
#define SSP_REFINE_MAX_ITERS 100
#define SSP_REFINE_FEW_POINTS 1
#define SSP_REFINE_SINGULAR 2
#define SSP_REFINE_BAD_POSE 4
int ssp_refine_depth(const unsigned short* depth, int W, int H, double depth_scale, const double* K3x3, const double* dist8_or_null,
                     const double* model, const int* offsets, const double* diam, int num_classes, const int* cls, int groups,
                     int per_group, const int* count_or_null, const double* R, const double* t, int iters, double gate_start,
                     double gate_end, double* R_out, double* t_out, int* points_out, double* rmse_out, int* status_out, void* stream);

/* ---- fusing the poses of several calibrated cameras (rules: csrc/multiview_core.h; csrc/multiview_rows.cu, csrc/multiview.cu), fp64.
 *      A rig is `views` = C cameras (1..SSP_RIG_MAX_VIEWS): K3x3_f32 [C][9] (DEVICE fp32, the PnP's K), K3x3 [C][9] (DEVICE fp64, the
 *      projection's K), dist8_or_null [C][8] (DEVICE fp64; a camera whose 8 values are all zero, or NULL, is the pinhole model) and
 *      extrinsics camera-from-world x_c = R_rig[c] x_w + t_rig[c] (DEVICE fp64 [C][9], [C][3]).  Rows b = g * C + c (g < groups) are
 *      camera c of capture g, each with `slots` objects: points3d [rows][slots][num_points][3] (or one shared [num_points][3]),
 *      points2d [rows][slots][num_points][2] raw pixels, valid [rows][slots] (DEVICE bytes, nonzero: the view takes part).
 *  ssp_fuse_views: step 1 solves every (row, slot) with its camera (max_iter LM iterations) into R_out [rows][slots][9], t_out
 *      [rows][slots][3] and projects its points into corners_out [rows][slots][num_points][2]: the bits of ssp_pnp_batched /
 *      ssp_pnp_dist and ssp_project_points / ssp_project_points_dist with that camera.  Per (capture, slot): each valid view's pose in
 *      the world frame is a hypothesis; the views that agree with it (mean squared reprojection error <= gate^2, every point in
 *      front) are fused by LM (at most max_iter steps), the views that agree with the result at reproj_thresh are fused again, and
 *      while a fused view lies beyond reproj_thresh it leaves and the rest is refitted; the
 *      hypothesis with the most views, then the lowest cost, then the lowest index wins.  Out: R_world [groups][slots][9], t_world
 *      [3], world_cov [36] (keypoint_sigma^2 (J^T J)^-1 over the final views, world axes, left perturbation), views_out [C] bytes,
 *      view_err [C] (RMS px of every valid view under the fused pose, -1 for the others), fuse_hyp (the winning view, -1 for none),
 *      fuse_status (SSP_FUSE_NO_VALID | SSP_FUSE_NO_VIEW: zero pose, no views, view_err -1; SSP_FUSE_SINGULAR: world_cov zeros) and
 *      corners_world [rows][slots][num_points][2] (the fused pose in each row's camera; zeros without one).  work: DEVICE scratch
 *      (8-B aligned) of at least the *bytes_out that ssp_fuse_views_work_bytes(groups, views, slots, bytes_out) writes.  SSP_ERR_ARG
 *      for a null pointer, views outside 1..16, num_points outside 7..10, groups < 0, slots < 1, max_iter < 1, a threshold or sigma
 *      not > 0 and finite, gate < reproj_thresh or a short workspace. ---- */
#define SSP_RIG_MAX_VIEWS 16
#define SSP_FUSE_NO_VALID 1
#define SSP_FUSE_NO_VIEW 2
#define SSP_FUSE_SINGULAR 4
int ssp_fuse_views_work_bytes(int groups, int views, int slots, long long* bytes_out);
int ssp_fuse_views(const float* points3d, int points3d_shared, const float* points2d, const unsigned char* valid, int num_points, int groups,
                   int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null, const double* R_rig,
                   const double* t_rig, double gate, double reproj_thresh, double keypoint_sigma, int max_iter, double* R_out,
                   double* t_out, float* corners_out, double* R_world, double* t_world, double* world_cov, unsigned char* views_out,
                   double* view_err, int* fuse_hyp, int* fuse_status, float* corners_world, void* work, long long work_bytes,
                   void* stream);

/* ---- refinement of a rig's world poses against every camera's registered depth frame: one point-to-plane ICP in world axes
 *      (rules: csrc/refine_rig_core.h; csrc/refine_rig.cu), fp64, one thread-block cluster of min(views, 8) 256-thread CTAs per
 *      problem, every iteration in one launch.  The rig is ssp_fuse_views' (`views` = C cameras, 1..SSP_RIG_MAX_VIEWS; K3x3 [C][9]
 *      DEVICE fp64, the projection's K; dist8_or_null [C][8]; R_rig [C][9], t_rig [C][3] camera from world); depth [groups * C][H][W]
 *      uint16, row b = g * C + c registered to camera c, depth_scale as ssp_refine_depth takes it.  model, offsets, diam, iters and
 *      the gates are ssp_refine_depth's; cls [groups][slots] (DEVICE int) each problem's class; points3d_table [num_classes]
 *      [num_points][3] (DEVICE fp32) the points drawn into corners_world_ref.  count_or_null: DEVICE int [groups] (slots at
 *      m >= count[g] get zeros and status 0); fuse_status_or_null: DEVICE int [groups][slots], ssp_fuse_views' status.
 *  ssp_refine_depth_rig: refines each world pose R_world [groups][slots][9], t_world [3] (world from object) against the pairs of
 *      every camera at once: each camera pairs the model points under its camera pose exactly as ssp_refine_depth does, the terms
 *      are taken in world axes and one solve per iteration updates the world pose (left perturbation, as world_cov).  Out: R_out,
 *      t_out; points_out, rmse_out of the last iteration over every camera; view_points [groups][slots][C] and view_rmse [C] each
 *      camera's pairs and RMS point-to-plane residual of the last iteration (0: no pairs); status_out: SSP_REFINE_FEW_POINTS (fewer
 *      than SSP_REFINE_MIN_POINTS pairs in all), SSP_REFINE_SINGULAR, SSP_REFINE_BAD_POSE (a pose that is not finite, or a
 *      fuse_status with SSP_FUSE_NO_VALID or SSP_FUSE_NO_VIEW); with a bit set the output pose is the input pose.
 *      corners_world_ref [groups * C][slots][num_points][2]: the output pose in every row's camera, ssp_fuse_views' corners_world
 *      arithmetic (zeros where the fusion has no pose).  With C = 1 and identity extrinsics the outputs are ssp_refine_depth's bit
 *      for bit.  SSP_ERR_ARG as ssp_refine_depth, and for views outside 1..16, num_points outside 7..10 or a null required
 *      pointer. ---- */
int ssp_refine_depth_rig(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                         const double* dist8_or_null, const double* R_rig, const double* t_rig, const double* model, const int* offsets,
                         const double* diam, const float* points3d_table, int num_points, int num_classes, const int* cls, int groups,
                         int slots, const int* count_or_null, const int* fuse_status_or_null, const double* R_world,
                         const double* t_world, int iters, double gate_start, double gate_end, double* R_out, double* t_out,
                         int* points_out, double* rmse_out, int* status_out, int* view_points, double* view_rmse,
                         float* corners_world_ref, void* stream);

/* ---- refinement of every world instance of a rig's capture against every camera's depth frame, each depth pixel owned by the
 *      instance drawn in front of it (rules: csrc/refine_instances_core.h; csrc/refine_instances.cu), fp64.  The rig, depth,
 *      depth_scale, model, offsets, diam, points3d_table, iters and the gates are ssp_refine_depth_rig's; the problems are the world
 *      slots of ssp_fuse_instances: world_cls [groups][slots] (slots 1..SSP_FUSE_MAX_SLOTS; a class outside [0, num_classes) is an
 *      empty slot), world_count_or_null [groups] (slots at w >= world_count[g] get zeros and status 0), fuse_status_or_null, R_world,
 *      t_world.  faces [total][3] (DEVICE int32) class c's triangles at face_offsets[c] .. face_offsets[c + 1] - 1 (DEVICE int
 *      [num_classes + 1]) as class-local vertex indices into its model rows (every index must lie in [0, its vertex count));
 *      max_faces the largest face count of a class.
 *  ssp_refine_instances_rig: per iteration, every non-empty slot with a usable input pose is drawn at its current pose (its input
 *      pose once a status bit has stopped it) into one z-buffer of 64-bit keys (float depth << 32 | slot) per camera; each slot
 *      then pairs as ssp_refine_depth_rig does, dropping a pair whose pixel another slot owns, and solves.  Out: ssp_refine_depth_rig's
 *      outputs per slot, view_hidden [groups][slots][C] the pairs dropped for ownership in the last iteration that ran, and
 *      instance_map [groups * C][H][W] int16: the slot drawn in front at each pixel under the output poses (-1: none).  A capture
 *      whose only drawn slot is w gives ssp_refine_depth_rig's outputs for w bit for bit.  work: DEVICE scratch (8-B aligned) of at
 *      least the *bytes_out that ssp_refine_instances_rig_work_bytes(groups, views, slots, W, H, bytes_out) writes: the owner
 *      buffers (8 B per pixel per frame) and the pose state.  SSP_ERR_ARG as ssp_refine_depth_rig, and for slots outside 1..256,
 *      max_faces < 0, a null pointer or a short workspace. ---- */
int ssp_refine_instances_rig_work_bytes(int groups, int views, int slots, int W, int H, long long* bytes_out);
int ssp_refine_instances_rig(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                             const double* dist8_or_null, const double* R_rig, const double* t_rig, const double* model, const int* offsets,
                             const double* diam, const int* faces, const int* face_offsets, int max_faces, const float* points3d_table,
                             int num_points, int num_classes, const int* world_cls, int groups, int slots, const int* world_count_or_null,
                             const int* fuse_status_or_null, const double* R_world, const double* t_world, int iters, double gate_start,
                             double gate_end, double* R_out, double* t_out, int* points_out, double* rmse_out, int* status_out,
                             int* view_points, double* view_rmse, int* view_hidden, float* corners_world_ref, short* instance_map,
                             void* work, long long work_bytes, void* stream);

/* ---- fusing every detected instance across the cameras of a rig (rules: csrc/multiview_instances_core.h; csrc/multiview_rows.cu,
 *      csrc/multiview_instances.cu), fp64.  The rig, the rows b = g * C + c and max_iter are ssp_fuse_views'; each row has `slots` = M
 *      detection slots (1..SSP_FUSE_MAX_SLOTS): points3d_table [num_classes][num_points][3] (DEVICE fp32, the PnP points of each class
 *      id), points2d [rows][M][num_points][2] raw pixels, cls [rows][M] and count [rows] (DEVICE int32; slot m of row b is a detection
 *      when m < count[b] and 0 <= cls < num_classes; ssp_detect_instances' outputs).
 *  ssp_fuse_instances: step 1 solves and projects every (row, slot) with m < count[b] as ssp_fuse_views does (the bits of
 *      ssp_pnp_batched_counted / ssp_pnp_dist and ssp_project_points(_dist) with that camera) into R_out [rows][M][9], t_out [3],
 *      corners_out [num_points][2]; empty slots get zeros.  Per capture: each detection's pose in the world frame is a hypothesis;
 *      in each view the closest available detection of its class within gate px joins, the set is fused by LM, and again with the
 *      detections within reproj_thresh px of that fit, members beyond reproj_thresh leave; the hypothesis with the most views, then
 *      the lowest cost, then the lowest index is emitted as a world instance and its detections leave; repeated until no hypothesis
 *      keeps a view or M instances are out.  Out per capture: world_count, unfused (the detections left) [groups]; per world slot
 *      w < M: world_cls [groups][M] (-1 for an empty slot), R_world [groups][M][9], t_world [3], world_cov [36] (keypoint_sigma^2
 *      (J^T J)^-1 over the members), members [groups][M][C] int32 (view c's fused slot, -1 for none), view_err [groups][M][C] (RMS px
 *      of the members, -1 for the others), fuse_hyp [groups][M] (the winning detection's index c * M + m, -1 for an empty slot),
 *      fuse_status [groups][M] (SSP_FUSE_SINGULAR: world_cov zeros); empty world slots are zeros.  Per row: world_index [rows][M]
 *      (the world slot each detection joined, -1 for none) and corners_world [rows][M][num_points][2] (world instance w of the row's
 *      capture drawn in the row's camera, zeros past world_count).  work: DEVICE scratch (8-B aligned) of at least the *bytes_out
 *      that ssp_fuse_instances_work_bytes(groups, views, slots, bytes_out) writes.  SSP_ERR_ARG as ssp_fuse_views, and for slots
 *      outside 1..256 or num_classes < 1. ---- */
#define SSP_FUSE_MAX_SLOTS 256
int ssp_fuse_instances_work_bytes(int groups, int views, int slots, long long* bytes_out);
int ssp_fuse_instances(const float* points3d_table, int num_classes, const float* points2d, const int* cls, const int* count, int num_points,
                       int groups, int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null,
                       const double* R_rig, const double* t_rig, double gate, double reproj_thresh, double keypoint_sigma, int max_iter,
                       double* R_out, double* t_out, float* corners_out, int* world_count, int* unfused, int* world_cls, double* R_world,
                       double* t_world, double* world_cov, int* members, double* view_err, int* fuse_hyp, int* fuse_status,
                       int* world_index, float* corners_world, void* work, long long work_bytes, void* stream);

/* ---- calibrating a camera rig from the object it sees (rules: csrc/calibrate_rig_core.h; csrc/multiview_rows.cu,
 *      csrc/calibrate_rig.cu), fp64.  The cameras (`views` = C, 1..SSP_RIG_MAX_VIEWS: K3x3_f32, K3x3, dist8_or_null), the rows
 *      b = g * C + c, points3d, points2d and valid are ssp_fuse_views'; the extrinsics are unknown.  Observation o = g * slots + s.
 *  ssp_calibrate_rig: step 1 solves every (row, slot) with its camera into R_rows [rows][slots][9], t_rows [3] (the bits of
 *      ssp_fuse_views' R_out, t_out).  Each camera pair scores up to 256 relative-pose hypotheses, one per co-observation, over all
 *      its co-observations (both views carried across within gate px); a maximum spanning tree over the winners' agreement counts
 *      (>= 3) rooted at camera `reference` gives the initial rig, whose world frame is the reference camera's (R = I, t = 0).  Then
 *      at most 4 rounds of: ssp_fuse_views' fusion of every observation under the current rig, and a bundle adjustment (LM, at most
 *      max_iter steps, Schur complement on the device) of the free cameras' extrinsics and the world poses of the observations fused
 *      in >= 2 cameras (linked); the rounds stop when no linked view set changes, and the fusion runs once more under the final
 *      rig.  Out per camera: R_cam [C][9], t_cam [C][3] (camera-from-world), cam_cov [C][36] (keypoint_sigma^2 times the camera's
 *      block of the reduced system's inverse, left perturbation in the camera frame; zeros for the reference), cam_obs [C] (linked
 *      observations it is fused in), cam_rmse [C] (RMS px of those views, -1 for none), tree_parent [C] (-1 for the root and
 *      unconnected cameras), edge_agree [C] (the tree edge's agreement count) and cam_status [C] (SSP_CALIB_UNCONNECTED: no tree
 *      path to the reference, zero extrinsics; SSP_CALIB_SINGULAR: cam_cov zeros).  Per observation: R_world [groups][slots][9],
 *      t_world [3], views_out [C] bytes and view_err [C] as ssp_fuse_views writes them under the final rig, linked [groups][slots]
 *      bytes.  Global: rounds, iterations (LM steps over all rounds), cost (the final sum of squared residuals).  work: DEVICE
 *      scratch (8-B aligned) of at least the *bytes_out that ssp_calibrate_rig_work_bytes(groups, views, slots, bytes_out) writes.
 *      SSP_ERR_ARG as ssp_fuse_views, and for a reference outside 0..views-1. ---- */
#define SSP_CALIB_UNCONNECTED 1
#define SSP_CALIB_SINGULAR 2
int ssp_calibrate_rig_work_bytes(int groups, int views, int slots, long long* bytes_out);
int ssp_calibrate_rig(const float* points3d, int points3d_shared, const float* points2d, const unsigned char* valid, int num_points, int groups,
                      int views, int slots, const float* K3x3_f32, const double* K3x3, const double* dist8_or_null, int reference,
                      double gate, double reproj_thresh, double keypoint_sigma, int max_iter, double* R_rows, double* t_rows,
                      double* R_cam, double* t_cam, double* cam_cov, int* cam_obs, double* cam_rmse, int* tree_parent, int* edge_agree,
                      int* cam_status, double* R_world, double* t_world, unsigned char* views_out, double* view_err,
                      unsigned char* linked, int* rounds, int* iterations, double* cost, void* work, long long work_bytes, void* stream);

/* ---- calibrating an RGB-D rig against depth: a point-to-plane bundle adjustment of the extrinsics and the observations' world
 *      poses (rules: csrc/calibrate_rig_depth_core.h; csrc/calibrate_rig_depth.cu), fp64, the second stage after ssp_calibrate_rig.
 *      The cameras (`views` = C, 2..SSP_RIG_MAX_VIEWS; K3x3 [C][9] DEVICE fp64, dist8_or_null [C][8]) with ssp_calibrate_rig's
 *      reference, cam_status_in [C] (DEVICE int), R_cam_in [C][9], t_cam_in [C][3] (camera-from-world; the reference R = I, t = 0);
 *      observation o = g * slots + s with ssp_calibrate_rig's R_world_in [O][9], t_world_in [O][3], obs_views [O][C] and linked [O]
 *      (DEVICE bytes).  One mesh for every observation: model [num_vertices][6] (DEVICE fp64 vertices and outward normals) and its
 *      diameter diam; depth [groups * C][H][W] uint16, row g * C + c camera c's frame of capture g, depth_scale, iters and the
 *      gates as ssp_refine_depth_rig takes them.
 *  ssp_calibrate_rig_depth: iters Gauss-Newton steps, with no accept test, of the free cameras' extrinsics (connected, not the
 *      reference) and the linked observations' world poses.  Each active view pairs the mesh with its depth as ssp_refine_depth_rig
 *      does; the reduced system over the free cameras is solved by a Cholesky factorisation.  Out per camera: R_cam, t_cam,
 *      cam_cov [C][36] (the RMS residual squared times the camera's block of the last reduced system's inverse: a lower bound, the
 *      pairs taken as independent; zeros for the reference, held and unconnected cameras), cam_points [C], cam_rmse [C] (its pairs
 *      and RMS point-to-plane residual in the last iteration), cam_status [C] (SSP_CALIB_DEPTH_UNCONNECTED passed through;
 *      SSP_CALIB_DEPTH_FEW_POINTS: held, fewer than SSP_REFINE_MIN_POINTS pairs, its extrinsics kept; SSP_CALIB_DEPTH_SINGULAR).
 *      Per observation: R_world, t_world, obs_points, obs_rmse of its last iteration, obs_status (SSP_REFINE_FEW_POINTS or
 *      SSP_REFINE_SINGULAR stop it, with the input pose; an observation that is not linked keeps its pose with zeros).  Global:
 *      status [1] (SSP_CALIB_DEPTH_SINGULAR: the reduced system could not be factored; every output pose is then its input) and
 *      iter_rmse [iters] (the RMS residual over every active pair before each iteration's update, 0 for iterations not run).
 *      work: DEVICE scratch (8-B aligned) of at least the *bytes_out that ssp_calibrate_rig_depth_work_bytes(groups, views, slots,
 *      bytes_out) writes.  SSP_ERR_ARG as ssp_refine_depth_rig and ssp_calibrate_rig, and for views < 2, num_vertices < 1 or a
 *      diameter not > 0 and finite. ---- */
#define SSP_CALIB_DEPTH_UNCONNECTED 1
#define SSP_CALIB_DEPTH_FEW_POINTS 2
#define SSP_CALIB_DEPTH_SINGULAR 4
int ssp_calibrate_rig_depth_work_bytes(int groups, int views, int slots, long long* bytes_out);
int ssp_calibrate_rig_depth(const unsigned short* depth, int W, int H, double depth_scale, int views, const double* K3x3,
                            const double* dist8_or_null, int reference, const int* cam_status_in, const double* R_cam_in,
                            const double* t_cam_in, const double* model, int num_vertices, double diam, int groups, int slots,
                            const unsigned char* obs_views, const unsigned char* linked, const double* R_world_in,
                            const double* t_world_in, int iters, double gate_start, double gate_end, double* R_cam, double* t_cam,
                            double* cam_cov, int* cam_points, double* cam_rmse, int* cam_status, double* R_world, double* t_world,
                            int* obs_points, double* obs_rmse, int* obs_status, int* status, double* iter_rmse, void* work,
                            long long work_bytes, void* stream);

/* ---- tracking the world instances of a rig over time (rules: csrc/world_track_core.h; csrc/world_track.cu), fp64.  Each capture g
 *      of ssp_fuse_instances (rows g * views .. g * views + views - 1, M = slots world slots) is its own stream with T = max_tracks
 *      (1..256) slots, state in DEVICE arrays the caller keeps between calls (zeros for a fresh start):
 *        tracks  int    [groups][T][5]   alive, id, cls, misses, hits (as ssp_track_associate's)
 *        poses   double [groups][T][12]  R (row-major), t of the track's last fused world pose
 *        next_id int    [groups]
 *        filter  double [groups][T][SSP_FILTER_DOUBLES] or NULL: the pose filter of ssp_track_filter_update, in world axes.
 *      The inputs are ssp_fuse_instances' world_count, world_cls, R_world, t_world, world_cov, fuse_status and world_index.
 *  ssp_world_track_associate: with a filter, every alive slot whose filter has started moves by dt [groups] seconds (DEVICE fp64)
 *      in place (dt is NULL exactly when filter is).  Then the world instances, in slot order, each take the alive, not yet taken
 *      track of their class whose position (the started filter's t, else the last fused t) lies nearest, strictly within
 *      match_dist * class_size[cls] (class_size: DEVICE fp64 [num_classes], the largest distance between two of the class's 8 box
 *      corners), the lower slot on ties; unmatched tracks age (they die at misses > max_misses) and unmatched instances take the
 *      lowest free slot and the next id.  Out per world slot: wslot [groups][M] (the track slot, -1 for an empty or untracked world
 *      slot), world_track_id [groups][M] (-1 likewise), matched [groups][M] (1: an existing track); per detection: track_id
 *      [groups * views][M] = its world instance's world_track_id through world_index (-1 for none).
 *  ssp_world_track_commit: each matched or born track stores its instance's R_world, t_world, misses 0, hits + 1; with a filter, a
 *      new track starts it from (R_world, t_world, world_cov) and a matched one is gated and updated (world_cov is unusable when
 *      fuse_status has SSP_FUSE_SINGULAR).  Out per world slot with a filter: R_filt [9], t_filt [3], pose_cov [6][6], velocity
 *      [6] = (w rad/s, v mesh units/s, world axes), reinit (1: the filter was started from this measurement); zeros elsewhere.
 *  SSP_ERR_ARG for a null required pointer, groups < 0, max_tracks or slots outside 1..256, views outside 1..16, num_classes < 1,
 *  max_misses < 0, or match_dist, an acceleration or initial velocity sigma or the gate not > 0 and finite. ---- */
int ssp_world_track_associate(int groups, int views, int max_tracks, int slots, const int* world_count, const int* world_cls,
                              const double* t_world, const int* world_index, const double* class_size, int num_classes, double match_dist,
                              int max_misses, int* tracks, const double* poses, double* filter, const double* dt, double accel_sigma_rot,
                              double accel_sigma_trans, int* next_id, int* wslot, int* world_track_id, int* matched, int* track_id,
                              void* stream);
int ssp_world_track_commit(int groups, int max_tracks, int slots, const int* world_count, const double* R_world, const double* t_world,
                           const double* world_cov, const int* fuse_status, const int* wslot, const int* matched, int* tracks, double* poses,
                           double* filter, double init_velocity_sigma_rot, double init_velocity_sigma_trans, double gate, double* R_filt,
                           double* t_filt, double* pose_cov, double* velocity, int* reinit, void* stream);

/* ---- pose errors over the mesh (utils.py:50-64, valid.py:69-72, 173-177), fp64 throughout (csrc/adds.cu, csrc/adds_core.h).
 *      X [nv][3] fp64 vertices; Rt_est, Rt_gt [n][3][4] fp64 poses [R | t].
 *  ssp_adds_batched: adds_out[p] = mean_i min_j |Rt_gt[p] x_i - Rt_est[p] x_j|, the reference's adi(pts_est, pts_gt) (ADD-S, for
 *      symmetric objects); add_out[p] (optional) = mean_i |Rt_gt[p] x_i - Rt_est[p] x_i| (ADD).  Each pose's result is computed in
 *      a fixed order: bit-identical on every launch, whatever n and the pose's position in the batch.  work: device scratch of at
 *      least ssp_adds_work_bytes(nv, n) bytes (8-B aligned).  n = 0 does nothing.
 *  ssp_mesh_diameter: *diam_out = the largest distance between two vertices, bit-identical to calc_pts_diameter on float64.
 *  SSP_ERR_ARG for a null pointer, nv < 1, nv > SSP_ADDS_MAX_VERTICES, n < 0 or n > 2^31 - 1 (ssp_adds_work_bytes returns
 *  SSP_ERR_ARG for these sizes too). ---- */
#define SSP_ADDS_MAX_VERTICES 1048576 /* 1 << 20 */
long long ssp_adds_work_bytes(int nv, long long n);
int ssp_adds_batched(const double* X, int nv, const double* Rt_est, const double* Rt_gt, long long n, double* adds_out,
                     double* add_out_or_null, void* work, long long work_bytes, void* stream);
int ssp_mesh_diameter(const double* X, int nv, double* diam_out, void* stream);

/* ---- silhouette masks of a mesh under n poses: the mask/<n>.png files a training set needs (image.py:131,135), which the
 *      reference leaves to the user (label_file_creation.md).  csrc/render.cu; the rules are in csrc/render_core.h.
 *      X [rows][nv] fp32 vertices, rows 3 or 4 (as ssp_project_points); faces [nf][3] int32; Rt [n][3][4] fp64; K3x3 fp64.
 *  ssp_render_masks: masks [n][H][W] uint8, 255 where the pixel centre (x, y) -- compute_projection's coordinates -- lies inside
 *      a non-degenerate triangle of either winding, else 0.  The vertices are the fp32 coordinates ssp_project_points returns,
 *      snapped to 1/256 px (round half to even); edge functions are exact int64, and a centre on an edge counts for top and left
 *      edges only (Direct3D's rule).  status [n] int32: bit 0 a vertex at camera depth <= 0, bit 1 a projected coordinate that
 *      is not finite or outside +-2^20 px, bit 2 a face index outside [0, nv); a pose with any bit set gets an all-zero mask.
 *      work: device scratch of at least ssp_render_work_bytes(nv, nf, n, W, H) bytes (256-B aligned).  Each pose's mask depends
 *      on nothing but its own inputs.  SSP_ERR_ARG for a null pointer, rows not 3 or 4, nv < 3, nf < 1, W or H outside
 *      [1, 16384], n < 0 or a work buffer that is too small (ssp_render_work_bytes returns SSP_ERR_ARG for bad sizes).
 *      n = 0 does nothing. ---- */
long long ssp_render_work_bytes(int nv, int nf, long long n, int W, int H);
int ssp_render_masks(const float* X, int rows, int nv, const int* faces, int nf, const double* Rt, const double* K3x3,
                     long long n, int W, int H, unsigned char* masks, int* status, void* work, long long work_bytes,
                     void* stream);

/* ---- training-image pipeline (SURVEY 8f.3): byte-exact with the Pillow routines image.py calls.  Images are device
 *      uint8 HWC RGB, dense.  resample = PIL.Image.Resampling value (0 NEAREST, 2 BILINEAR, 3 BICUBIC = resize()'s default
 *      in Pillow >= 7).  `work` is caller-provided device scratch (16-B aligned) of at least *_work_bytes() bytes.
 *  ssp_aug_resize_u8: Image.crop((x0, y0, x0+in_w, y0+in_h)).resize((out_w, out_h), resample) (image.py:64,69; dataset.py:103);
 *      the crop window may stick out of the source (zero fill), pass (0, 0, src_w, src_h) for a plain resize.
 *  ssp_aug_rgb2hsv_u8 / hsv2rgb_u8: Image.convert('HSV') / ('RGB') (image.py:15,30).
 *  ssp_aug_to_tensor_u8: torchvision ToTensor (the `transform` of dataset.py:103-118) of a dense uint8 HWC image: float32 CHW,
 *      byte / 255 as an IEEE division (what the CPU reference computes; a reciprocal multiply differs by 1 ulp). ---- */
long long ssp_aug_resize_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample);
int ssp_aug_resize_u8(const void* src, int src_w, int src_h, int x0, int y0, int in_w, int in_h, void* dst, int out_w,
                      int out_h, int resample, void* work, long long work_bytes, void* stream);
int ssp_aug_rgb2hsv_u8(const void* rgb, void* hsv, long long n_pixels, void* stream);
int ssp_aug_hsv2rgb_u8(const void* hsv, void* rgb, long long n_pixels, void* stream);
int ssp_aug_to_tensor_u8(const void* hwc_u8, long long n_pixels, float* out_chw, void* stream);

/* Training-image batch: change_background (image.py:110-127) -> crop -> resize -> distort_image (image.py:14-32) -> ToTensor
 * (dataset.py transform) for every sample, with ONE launch per pipeline stage for the whole batch (<= 10 launches).
 *   ssp_aug_item, one per sample, with DEVICE pointers: img and mask (ow x oh), bg (bw x bh); luts = 5 x 256 bytes: posmask,
 *     negmask (image.py:121-122), hue, saturation, value (image.py:17-27) point() tables, built by the host exactly as
 *     Image.point() builds them; crop window (pleft, ptop, cw, ch) with cw = swidth - 1, ch = sheight - 1 (image.py:64); its own
 *     work buffer of ssp_aug_sample_work_bytes() bytes; out_u8 (HWC) and out_chw (float32 CHW in [0,1]) are both optional, at
 *     least one required.
 *   ssp_aug_batch_plan (host only, no device access): writes the op table (table_bytes >= ssp_aug_batch_table_bytes(n)) into
 *     HOST memory -- typically the tail of the pinned staging buffer, so that it travels in the batch's single host->device
 *     copy -- and stage_dims[20].
 *   ssp_aug_batch_run: table_dev = the device copy of that table; launches the stages on `stream`. */
long long ssp_aug_sample_work_bytes(int ow, int oh, int bw, int bh, int cw, int ch, int out_w, int out_h, int resample);
typedef struct ssp_aug_item {
  const void* img; const void* mask; int ow, oh; const void* bg; int bw, bh; const void* luts; int pleft, ptop, cw, ch;
  void* work; long long work_bytes; void* out_u8; float* out_chw;
} ssp_aug_item;
long long ssp_aug_batch_table_bytes(int n);
int ssp_aug_batch_plan(const ssp_aug_item* items_host, int n, int out_w, int out_h, int resample, void* table_host,
                       long long table_bytes, int* stage_dims_host20);
int ssp_aug_batch_run(const void* table_dev, int n, const int* stage_dims_host20, void* stream);

/* ---- multi-object training-image pipeline (multi_obj_pose_estimation/image_multi.py load_data_detection), byte-exact with the
 *      Pillow routines it calls.  Per sample the caller owns four network-size (out_w x out_h x 3 bytes) device images --
 *      main_img, main_mask, total_img, total_mask -- and counts[4] (unsigned): [S, I, accepted, unused].  luts = posmask | negmask
 *      (2 x 256 bytes, as in ssp_aug_item).  Every item needs its own 16-B aligned work buffer of
 *      ssp_augm_work_bytes(in_w, in_h, out_w, out_h) bytes, with (in_w, in_h) = the crop window (cw, ch) for begin / attempt
 *      and the background size for finish.  The plan calls only write HOST memory (no allocation, no device access, no
 *      synchronisation); ssp_augm_run launches the planned stages of one phase (<= 16 launches for the whole batch) on
 *      `stream`, reading the device copy of the table.
 *  ssp_augm_plan_begin: main object of each sample -- crop (pleft, ptop, cw, ch) of img / mask (src_w x src_h), resize,
 *      ImageChops.offset(shift_x, shift_y), FLIP_LEFT_RIGHT if flip, mask_background (image_multi.py:184-228, 38-50); sets
 *      main_* and initialises total_* (:316-322).
 *  ssp_augm_plan_attempt: one candidate object per item (n = samples still placing objects).  img / mask = the candidate at
 *      source resolution; mask_bg = 1 masks img IN PLACE first (mask_background, :338), 0 = img is already masked.  Crop,
 *      resize, flip (:230-263); S = bytes > 200 of the candidate mask, I = those also > 200 in total_mask; accepted =
 *      S != 0 && (double)I / S < 0.2, computed on the device and written to counts[2]; if accepted, superimpose_masks and
 *      superimpose_masked_imgs (:265-297) update total_mask / total_img.  Nothing waits for the host; it reads counts after
 *      the round to decide what to draw next.
 *  ssp_augm_plan_finish: img = background (src_w x src_h), resized to out_w x out_h; main object on top (:363),
 *      change_background (:380), then out_u8 (HWC) and / or out_chw (float32 CHW, byte / 255, ToTensor). ---- */
typedef struct ssp_augm_item {
  void* img; const void* mask; int src_w, src_h;
  int pleft, ptop, cw, ch;
  int flip, shift_x, shift_y, mask_bg;
  void* main_img; void* main_mask; void* total_img; void* total_mask;
  unsigned* counts;
  const void* luts;
  void* work; long long work_bytes; void* out_u8; float* out_chw;
} ssp_augm_item;
long long ssp_augm_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample);
long long ssp_augm_table_bytes(int n);
int ssp_augm_plan_begin(const ssp_augm_item* items_host, int n, int out_w, int out_h, int resample, void* table_host,
                        long long table_bytes, int* stage_dims_host32);
int ssp_augm_plan_attempt(const ssp_augm_item* items_host, int n, int out_w, int out_h, int resample, void* table_host,
                          long long table_bytes, int* stage_dims_host32);
int ssp_augm_plan_finish(const ssp_augm_item* items_host, int n, int out_w, int out_h, int resample, void* table_host,
                         long long table_bytes, int* stage_dims_host32);
int ssp_augm_run(const void* table_dev, int n, const int* stage_dims_host32, void* stream);

/* ---- JPEG decode (dataset.py / image.py open every training and test image with Pillow): baseline Huffman JPEGs decoded for a
 *      whole batch, byte-identical to PIL's Image.open(f).convert('RGB') on libjpeg-turbo (ISLOW IDCT, fancy upsampling)
 *      (csrc/jpeg.cu, rules in csrc/jpeg_core.h).
 *  ssp_jpeg_parse (host only): header of one file.  Returns 0 if the GPU path takes it (1 component, or YCbCr with luma sampling
 *      in {1,2}x{1,2} and 1x1 chroma, 8-bit, one sequential Huffman scan, ending with EOI), a positive decline code otherwise
 *      (ssp_jpeg_decline_reason gives the text), SSP_ERR_ARG for a null pointer.  info receives the size either way when known.
 *  ssp_jpeg_stage_bytes / ssp_jpeg_work_bytes (host only): pinned staging and device workspace sizes of a batch of takeable
 *      files (SSP_ERR_ARG if one is declined).
 *  ssp_jpeg_batch_plan (host only, no device access): writes the batch's records, entropy-coded data (without stuffed bytes and
 *      restart markers) and interval tables into stage_host; dims_host4 receives {largest block count, largest pixel count,
 *      workspace bytes, staging bytes actually used}.  items[i].out is the DEVICE (height, width, 3) uint8 output.
 *  ssp_jpeg_batch_run: stage_dev = the device copy of the first dims[3] bytes of the staging buffer (16-B aligned); three
 *      launches on `stream`, no allocation, no synchronisation.  status[3n] (device int): status[i] | status[n + i] is 0 when
 *      the output was written, otherwise SSP_JPEG_ST_* bits (the output is left untouched and the image is for Pillow);
 *      status[2n + i] = the subsequences of image i whose state no speculative candidate linked to, decoded serially.
 *      n = 0 does nothing. ---- */
#define SSP_JPEG_ST_ENTROPY 1    /* invalid code, coefficient index past 63, data missing or left over, ... */
#define SSP_JPEG_ST_RANGE 2      /* a block where libjpeg-turbo's SIMD and C IDCT can differ */
#define SSP_JPEG_ST_STRUCTURE 4  /* restart markers missing, extra or out of sequence, or another marker inside the scan */
#define SSP_JPEG_ST_OVERFLOW 8   /* a DC value leaves int32 */
typedef struct ssp_jpeg_info { int width, height, components, h_samp, v_samp, restart_interval; } ssp_jpeg_info;
typedef struct ssp_jpeg_item { const void* data; long long size; void* out; } ssp_jpeg_item;
int ssp_jpeg_parse(const void* data, long long size, ssp_jpeg_info* info);
const char* ssp_jpeg_decline_reason(int code);
long long ssp_jpeg_stage_bytes(const ssp_jpeg_item* items_host, int n);
long long ssp_jpeg_work_bytes(const ssp_jpeg_item* items_host, int n);
int ssp_jpeg_batch_plan(const ssp_jpeg_item* items_host, int n, void* stage_host, long long stage_bytes, long long* dims_host4);
int ssp_jpeg_batch_run(const void* stage_dev, int n, const long long* dims_host4, void* work, long long work_bytes, int* status,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif
