// extern "C" surface of libssp_b200.so (declared in include/ssp_b200.h): argument plumbing only.
#include "ssp_common.cuh"
#include "../../include/ssp_b200.h"
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

namespace ssp {
static thread_local char g_err[512] = "";
int fail_cuda(cudaError_t e, const char* file, int line) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s:%d", (int)e, cudaGetErrorString(e), file, line);
  return SSP_ERR_CUDA;
}
int fail_msg(int code, const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg); return code; }

int conv_gemm_tc(const void*, const void*, long long, int, int, const void*, const void*, int, int, int, int, int, int, int, int, int,
                 float*, int, long long, int, const float*, double*, double*, cudaStream_t, const FusedAct*, const SplitK* = nullptr);
int conv_splitk_count(int, int, int, int, int, int, int);
int conv_gemm_band(const void*, const void*, long long, int, int, const void*, const void*, int, int, int, int, int, int, int, int, int,
                   float*, int, long long, int, const float*, double*, double*, cudaStream_t);
int conv_gemm_simt(const void*, const void*, long long, int, int, const void*, const void*, int, int, int, int, int, int, int, int, int,
                   float*, int, long long, int, const float*, double*, double*, cudaStream_t);
int conv_gemm_bandt(const void*, const void*, long long, int, int, const void*, const void*, int, int, int, int, int, int, int, int, int,
                    float*, int, long long, int, const float*, double*, double*, cudaStream_t);
int conv_bandt_launch_count();
int l0_gram(const float*, int, int, int, double*, cudaStream_t);
int l0_stats(const double*, const float*, double*, double*, cudaStream_t);
int l0_fused_fwd(const float*, const float*, const float*, const float*, float, int, int, int, void*, void*, int, int, uint8_t*, cudaStream_t);
int l0_bwd(const float*, const void*, int, int, int, const uint8_t*, float, int, int, int, double*, cudaStream_t);
int l0_bwd_finalize(const double*, const double*, const float*, const float*, const float*, const float*, double, float, float*, float*, float*, cudaStream_t);
int wgrad_gemm_tc(const void*, long long, int, int, int, const void*, long long, int, int, int, int, int, int, int, float*, int, int, float, cudaStream_t);
int wgrad_gemm_simt(const void*, long long, int, int, int, const void*, long long, int, int, int, int, int, int, int, float*, int, int, float, cudaStream_t);
int pack_nchw(const float*, void*, void*, int, int, int, int, int, int, int, float, cudaStream_t);
int unpack_nchw(const float*, float*, int, int, int, int, int, int, cudaStream_t);
int unpack16_nchw(const void*, const void*, float*, int, int, int, int, int, int, int, cudaStream_t);
int bn_finalize(double*, double*, double, const float*, const float*, float*, float*, float, float, int, float*, float*, float*, float*, int, cudaStream_t);
int bn_apply(const float*, int, const float*, const float*, int, int, int, int, float, void*, void*, int, int, int, void*, void*, int, int, int, float*, int, cudaStream_t);
int bn_apply_splitk(const float*, int, long long, int, const float*, const float*, int, int, int, int, float, void*, void*, int, int, int, void*, void*,
                    int, int, int, cudaStream_t, float* = nullptr, int = 0);
int bn_bwd_reduce(const float*, int, const float*, const float*, const float*, const float*, const float*, int, int, int, int, float,
                  const float*, int, int, int, const float*, int, int, int, double*, double*, cudaStream_t);
int bn_bwd_apply(const float*, int, const float*, const float*, const float*, const float*, const float*, int, int, int, int, float,
                 const float*, int, int, int, const float*, int, int, int, double*, double*, void*, int, int, float, cudaStream_t);
int bn_bwd_finalize(double*, double*, float*, float*, int, int, float, cudaStream_t);
int bias_grad_nchw(const float*, float*, int, int, int, int, float, cudaStream_t);
int pack_weights(const float*, int, int, int, void*, void*, int, void*, int, int, cudaStream_t);
int sgd_step_flat(float*, const float*, float*, long long, float, float, float, float, cudaStream_t);
int sgd_pack_step(const ssp_sgd_segment*, int, int, int, float*, const float*, float*, float, float, float, float, cudaStream_t);
int region_loss_fwd_bwd(const float*, const float*, float*, double*, int, int, int, int, int, float, float, float, float, int, float, cudaStream_t);
int region_decode_argmax(const float*, int, int, int, int, int, int, float*, float*, float*, cudaStream_t);
int region_loss_multi_fwd_bwd(const float*, const float*, float*, double*, int, int, int, int, int, int, const float*, int, float, float, float,
                              float, float, int, float, cudaStream_t);
int region_decode_multi(const float*, int, int, int, int, int, int, int, int, float*, float*, float*, float*, long long*, float*, float*, cudaStream_t);
int eval_multi_select(const float*, int, int, int, int, int, int, const float*, int, const int*, float, float, float, float*, int*, float*,
                      cudaStream_t);
int predict_multi_select(const float*, int, int, int, int, int, int, const int*, int, float, float, float, float*, int*, float*, cudaStream_t);
int pnp_batched(const float*, int, const float*, const float*, int, long long, int, double*, double*, int*, int*, cudaStream_t);
int project_points(const float*, int, int, const double*, const double*, long long, float*, cudaStream_t);
long long adds_work_bytes(int, long long);
int adds_batched(const double*, int, const double*, const double*, long long, double*, double*, void*, long long, cudaStream_t);
int mesh_diameter(const double*, int, double*, cudaStream_t);
int jpeg_parse(const void*, long long, ssp_jpeg_info*);
const char* jpeg_decline_reason(int);
long long jpeg_stage_bytes(const ssp_jpeg_item*, int);
long long jpeg_work_bytes(const ssp_jpeg_item*, int);
int jpeg_batch_plan(const ssp_jpeg_item*, int, void*, long long, long long*);
int jpeg_batch_run(const void*, int, const long long*, void*, long long, int*, cudaStream_t);
long long aug_resize_work_bytes(int, int, int, int, int);
long long aug_sample_work_bytes(int, int, int, int, int, int, int, int, int);
int aug_resize_u8(const uint8_t*, int, int, int, int, int, int, uint8_t*, int, int, int, uint8_t*, long long, cudaStream_t);
int aug_convert_u8(const uint8_t*, uint8_t*, long long, int, cudaStream_t);
int aug_to_tensor_u8(const uint8_t*, long long, float*, cudaStream_t);
long long aug_batch_table_bytes(int);
int aug_batch_plan(const ssp_aug_item*, int, int, int, int, void*, long long, int*);
int aug_batch_run(const void*, int, const int*, cudaStream_t);
long long augm_work_bytes(int, int, int, int, int);
long long augm_table_bytes(int);
int augm_plan(int, const ssp_augm_item*, int, int, int, int, void*, long long, int*);
int augm_run(const void*, int, const int*, cudaStream_t);
int aug_sample(const uint8_t*, const uint8_t*, int, int, const uint8_t*, int, int, const uint8_t*, int, int, int, int, int, int, int, uint8_t*,
               long long, uint8_t*, float*, cudaStream_t);
}  // namespace ssp

using namespace ssp;
#define ST(s) ((cudaStream_t)(s))

extern "C" {
int ssp_version(void) { return 100; }
const char* ssp_last_error(void) { return g_err; }
long long ssp_flat_alloc_rows(int N, int H, int W) { return flat_alloc_rows(N, H, W); }
long long ssp_flat_row(int n, int h, int w, int H, int W) { Geom g{1, H, W}; return g.row(n, h, w); }

int ssp_pack_nchw(const float* x, void* hi, void* lo, int N, int C, int H, int W, int ld, int c0, int fmt, float scale, void* s) {
  return pack_nchw(x, hi, lo, N, C, H, W, ld, c0, fmt, scale, ST(s));
}
int ssp_unpack_nchw(const float* y, float* out, int N, int C, int H, int W, int ld, int c0, void* s) { return unpack_nchw(y, out, N, C, H, W, ld, c0, ST(s)); }
int ssp_unpack16_nchw(const void* hi, const void* lo, float* out, int N, int C, int H, int W, int ld, int c0, int fmt, void* s) {
  return unpack16_nchw(hi, lo, out, N, C, H, W, ld, c0, fmt, ST(s));
}
int ssp_conv_gemm(int impl, const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo,
                  int b_rows, int b_ld, int a_fmt, int b_fmt, int N, int H, int W, int taps, int cout, float* out, int out_ld,
                  long long out_rows, int epi, const float* bias, double* ssum, double* ssq, void* s) {
  if (epi == SSP_EPI_F16) {          // fp16 data-gradient planes: the operand-swapped kernel where eligible, the per-tap kernel otherwise
    if (impl != SSP_IMPL_BANDT && impl != SSP_IMPL_TC2) return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm: SSP_EPI_F16 needs SSP_IMPL_BANDT or SSP_IMPL_TC2");
    if (impl == SSP_IMPL_BANDT) {
      const int rc = conv_gemm_bandt(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s));
      if (rc != 1) return rc;
    }
    return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s), nullptr);
  }
  if (impl == SSP_IMPL_SIMT)
    return conv_gemm_simt(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s));
  if (impl == SSP_IMPL_BANDT) {
    const int rc = conv_gemm_bandt(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s));
    if (rc != 1) return rc;          // 1 = not eligible: the kernels for wider layers below
    impl = (taps == 9 && cout < 128) ? SSP_IMPL_BAND : SSP_IMPL_TC;
  }
  if (impl == SSP_IMPL_BAND) {
    const int rc = conv_gemm_band(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s));
    if (rc != 1) return rc;          // 1 = layer not eligible (weights do not fit): per-tap kernel below
  }
  return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s), nullptr);
}
int ssp_conv_bandt_launches(void) { return conv_bandt_launch_count(); }
int ssp_l0_gram(const float* x, int N, int H, int W, double* gram, void* s) { return l0_gram(x, N, H, W, gram, ST(s)); }
int ssp_l0_stats(const double* gram, const float* w, double* ssum, double* ssq, void* s) { return l0_stats(gram, w, ssum, ssq, ST(s)); }
int ssp_l0_fused_fwd(const float* x, const float* w, const float* scale, const float* shift, float slope, int N, int H, int W, void* d_hi,
                     void* d_lo, int d_ld, int d_c0, unsigned char* code, void* s) {
  return l0_fused_fwd(x, w, scale, shift, slope, N, H, W, d_hi, d_lo, d_ld, d_c0, code, ST(s));
}
int ssp_l0_bwd(const float* x, const void* g, int g_f16, int g_ld, int g_c0, const unsigned char* code, float slope, int N, int H, int W, double* t1, void* s) {
  return l0_bwd(x, g, g_f16, g_ld, g_c0, code, slope, N, H, W, t1, ST(s));
}
int ssp_l0_bwd_finalize(const double* t1, const double* gram, const float* w, const float* gamma, const float* mean, const float* invstd,
                        double count, float gscale, float* dw, float* dgamma, float* dbeta, void* s) {
  return l0_bwd_finalize(t1, gram, w, gamma, mean, invstd, count, gscale, dw, dgamma, dbeta, ST(s));
}
int ssp_conv_gemm_bnact(int impl, const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo,
                        int b_rows, int b_ld, int N, int H, int W, int taps, int cout, const float* scale, const float* shift, float slope,
                        void* d_hi, void* d_lo, int d_ld, int d_c0, void* s) {
  FusedAct fa{scale, shift, slope, (uint16_t*)d_hi, (uint16_t*)d_lo, d_ld, d_c0};
  if (impl == SSP_IMPL_TC || impl == SSP_IMPL_TC2 || impl == SSP_IMPL_BAND)
    return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, SSP_FMT_F16, SSP_FMT_F16, N, H, W, taps, cout, nullptr, 0, 0, EPI_BNACT,
                        nullptr, nullptr, nullptr, ST(s), &fa);
  return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm_bnact: tensor-core implementations only");
}
int ssp_conv_gemm_splitk(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo, int b_rows,
                         int b_ld, int N, int H, int W, int taps, int cout, int splits, float* partial, long long slab_elems, int partial_ld,
                         void* s) {
  const SplitK sk{splits, slab_elems};
  return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, SSP_FMT_F16, SSP_FMT_F16, N, H, W, taps, cout, partial, partial_ld, 0,
                      EPI_F32, nullptr, nullptr, nullptr, ST(s), nullptr, &sk);
}
int ssp_conv_splitk_count(int N, int H, int W, int taps, int cin, int cout, int num_sms) { return conv_splitk_count(N, H, W, taps, cin, cout, num_sms); }
int ssp_bn_apply_splitk(const float* partial, int splits, long long slab_elems, int partial_ld, const float* scale, const float* shift, int N, int C,
                        int H, int W, float slope, void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_route, void* d1_hi, void* d1_lo, int d1_ld,
                        int d1_c0, int d1_route, void* s) {
  return bn_apply_splitk(partial, splits, slab_elems, partial_ld, scale, shift, N, C, H, W, slope, d0_hi, d0_lo, d0_ld, d0_c0, d0_route, d1_hi, d1_lo,
                         d1_ld, d1_c0, d1_route, ST(s));
}
int ssp_wgrad_gemm(int impl, const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt, const void* x, long long x_rows, int x_ld,
                   int cin, int x_fmt, int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, void* s) {
  if (impl == SSP_IMPL_SIMT) return wgrad_gemm_simt(dy, dy_rows, dy_ld, cout, dy_fmt, x, x_rows, x_ld, cin, x_fmt, N, H, W, taps, dw, dw_ld, cin_store, scale, ST(s));
  return wgrad_gemm_tc(dy, dy_rows, dy_ld, cout, dy_fmt, x, x_rows, x_ld, cin, x_fmt, N, H, W, taps, dw, dw_ld, cin_store, scale, ST(s));
}
int ssp_bn_finalize(double* ssum, double* ssq, double count, const float* gamma, const float* beta, float* rm, float* rv, float momentum,
                    float eps, int train, float* mean, float* invstd, float* scale, float* shift, int C, void* s) {
  return bn_finalize(ssum, ssq, count, gamma, beta, rm, rv, momentum, eps, train, mean, invstd, scale, shift, C, ST(s));
}
int ssp_bn_apply(const float* y, int y_ld, const float* scale, const float* shift, int N, int C, int H, int W, float slope,
                 void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_route, void* d1_hi, void* d1_lo, int d1_ld, int d1_c0, int d1_route,
                 float* ypool, int ypool_ld, void* s) {
  return bn_apply(y, y_ld, scale, shift, N, C, H, W, slope, d0_hi, d0_lo, d0_ld, d0_c0, d0_route, d1_hi, d1_lo, d1_ld, d1_c0, d1_route, ypool, ypool_ld, ST(s));
}
int ssp_bn_bwd_reduce(const float* y, int y_ld, const float* scale, const float* shift, const float* mean, const float* invstd, const float* gamma,
                      int N, int C, int H, int W, float slope, const float* g0, int g0_ld, int g0_c0, int g0_route,
                      const float* g1, int g1_ld, int g1_c0, int g1_route, double* s1, double* s2, void* s) {
  return bn_bwd_reduce(y, y_ld, scale, shift, mean, invstd, gamma, N, C, H, W, slope, g0, g0_ld, g0_c0, g0_route, g1, g1_ld, g1_c0, g1_route, s1, s2, ST(s));
}
int ssp_bn_bwd_apply(const float* y, int y_ld, const float* scale, const float* shift, const float* mean, const float* invstd, const float* gamma,
                     int N, int C, int H, int W, float slope, const float* g0, int g0_ld, int g0_c0, int g0_route,
                     const float* g1, int g1_ld, int g1_c0, int g1_route, double* s1, double* s2, void* dy, int dy_ld, int dy_fmt, float dy_scale, void* s) {
  return bn_bwd_apply(y, y_ld, scale, shift, mean, invstd, gamma, N, C, H, W, slope, g0, g0_ld, g0_c0, g0_route, g1, g1_ld, g1_c0, g1_route, s1, s2, dy, dy_ld, dy_fmt, dy_scale, ST(s));
}
int ssp_bn_bwd_finalize(double* s1, double* s2, float* dgamma, float* dbeta, int C, int accumulate, float scale, void* s) { return bn_bwd_finalize(s1, s2, dgamma, dbeta, C, accumulate, scale, ST(s)); }
int ssp_bias_grad_nchw(const float* g, float* db, int N, int C, int HW, int accumulate, float scale, void* s) { return bias_grad_nchw(g, db, N, C, HW, accumulate, scale, ST(s)); }
int ssp_pack_weights(const float* w, int cout, int taps, int cin, void* f_hi, void* f_lo, int ld_f, void* d, int ld_d, int d_fmt, void* s) {
  return pack_weights(w, cout, taps, cin, f_hi, f_lo, ld_f, d, ld_d, d_fmt, ST(s));
}
int ssp_sgd_segment_blocks(int cout, int taps, int cin, long long n) {
  if (taps == 0) return (int)((n + 1023) / 1024);
  return ((cin + 63) / 64) * ((cout + 63) / 64) * taps;
}
int ssp_sgd_pack_step(const ssp_sgd_segment* segs, int n_seg, int b0, int b1, float* p, const float* g, float* v, float lr, float mu, float wd,
                      float gscale, void* s) {
  return sgd_pack_step(segs, n_seg, b0, b1, p, g, v, lr, mu, wd, gscale, ST(s));
}
int ssp_sgd_step_flat(float* p, const float* g, float* v, long long n, float lr, float mu, float wd, float gscale, void* s) { return sgd_step_flat(p, g, v, n, lr, mu, wd, gscale, ST(s)); }
int ssp_region_loss_fwd_bwd(const float* out, const float* target, float* grad, double* acc, int B, int K, int nC, int H, int W, float coord_scale,
                            float noobject_scale, float object_scale, float thresh, int use_conf, float grad_scale, void* s) {
  return region_loss_fwd_bwd(out, target, grad, acc, B, K, nC, H, W, coord_scale, noobject_scale, object_scale, thresh, use_conf, grad_scale, ST(s));
}
int ssp_region_decode_argmax(const float* out, int B, int K, int nC, int H, int W, int only_objectness, float* boxes, float* best_conf, float* box_global, void* s) {
  return region_decode_argmax(out, B, K, nC, H, W, only_objectness, boxes, best_conf, box_global, ST(s));
}
int ssp_region_loss_multi_fwd_bwd(const float* out, const float* target, float* grad, double* acc, int B, int K, int nC, int nA, int H, int W,
                                  const float* anchors_host, int anchor_step, float coord_scale, float noobject_scale, float object_scale,
                                  float class_scale, float thresh, int use_conf, float grad_scale, void* s) {
  return region_loss_multi_fwd_bwd(out, target, grad, acc, B, K, nC, nA, H, W, anchors_host, anchor_step, coord_scale, noobject_scale, object_scale,
                                   class_scale, thresh, use_conf, grad_scale, ST(s));
}
int ssp_region_decode_multi(const float* out, int B, int K, int nC, int nA, int H, int W, int only_objectness, int corr, float* boxes, float* conf_sel,
                            float* det, float* cls_corr, long long* max_ind, float* max_conf, float* max_cls, void* s) {
  return region_decode_multi(out, B, K, nC, nA, H, W, only_objectness, corr, boxes, conf_sel, det, cls_corr, max_ind, max_conf, max_cls, ST(s));
}
int ssp_eval_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const float* target, int target_stride,
                          const int* gt_offset, float conf_thresh, float im_width, float im_height, float* boxes, int* flags, float* uv,
                          void* s) {
  return eval_multi_select(out, B, K, nC, nA, H, W, target, target_stride, gt_offset, conf_thresh, im_width, im_height, boxes, flags, uv, ST(s));
}
int ssp_predict_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const int* classes_host, int n_req, float conf_thresh,
                             float frame_w, float frame_h, float* boxes, int* flags, float* uv, void* s) {
  return predict_multi_select(out, B, K, nC, nA, H, W, classes_host, n_req, conf_thresh, frame_w, frame_h, boxes, flags, uv, ST(s));
}
int ssp_pnp_batched(const float* P3, int shared, const float* uv, const float* K, int np, long long n, int max_iter, double* R, double* t, int* iters, void* s) {
  return pnp_batched(P3, shared, uv, K, np, n, max_iter, R, t, iters, nullptr, ST(s));
}
int ssp_pnp_batched_work(const float* P3, int shared, const float* uv, const float* K, int np, long long n, int max_iter, double* R, double* t,
                         int* work, void* s) {
  return pnp_batched(P3, shared, uv, K, np, n, max_iter, R, t, nullptr, work, ST(s));
}
int ssp_project_points(const float* X, int rows, int nv, const double* Rt, const double* K, long long n, float* out, void* s) {
  return project_points(X, rows, nv, Rt, K, n, out, ST(s));
}
long long ssp_adds_work_bytes(int nv, long long n) { return adds_work_bytes(nv, n); }
int ssp_adds_batched(const double* X, int nv, const double* Rt_est, const double* Rt_gt, long long n, double* adds_out, double* add_out,
                     void* work, long long work_bytes, void* s) {
  return adds_batched(X, nv, Rt_est, Rt_gt, n, adds_out, add_out, work, work_bytes, ST(s));
}
int ssp_mesh_diameter(const double* X, int nv, double* diam_out, void* s) { return mesh_diameter(X, nv, diam_out, ST(s)); }
int ssp_jpeg_parse(const void* data, long long size, ssp_jpeg_info* info) { return jpeg_parse(data, size, info); }
const char* ssp_jpeg_decline_reason(int code) { return jpeg_decline_reason(code); }
long long ssp_jpeg_stage_bytes(const ssp_jpeg_item* items, int n) { return jpeg_stage_bytes(items, n); }
long long ssp_jpeg_work_bytes(const ssp_jpeg_item* items, int n) { return jpeg_work_bytes(items, n); }
int ssp_jpeg_batch_plan(const ssp_jpeg_item* items, int n, void* stage_host, long long stage_bytes, long long* dims) {
  return jpeg_batch_plan(items, n, stage_host, stage_bytes, dims);
}
int ssp_jpeg_batch_run(const void* stage_dev, int n, const long long* dims, void* work, long long work_bytes, int* status, void* s) {
  return jpeg_batch_run(stage_dev, n, dims, work, work_bytes, status, ST(s));
}
long long ssp_aug_resize_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) { return aug_resize_work_bytes(in_w, in_h, out_w, out_h, resample); }
int ssp_aug_resize_u8(const void* src, int src_w, int src_h, int x0, int y0, int in_w, int in_h, void* dst, int out_w, int out_h, int resample,
                      void* work, long long work_bytes, void* s) {
  return aug_resize_u8((const uint8_t*)src, src_w, src_h, x0, y0, in_w, in_h, (uint8_t*)dst, out_w, out_h, resample, (uint8_t*)work, work_bytes, ST(s));
}
int ssp_aug_rgb2hsv_u8(const void* rgb, void* hsv, long long n_pixels, void* s) { return aug_convert_u8((const uint8_t*)rgb, (uint8_t*)hsv, n_pixels, 1, ST(s)); }
int ssp_aug_hsv2rgb_u8(const void* hsv, void* rgb, long long n_pixels, void* s) { return aug_convert_u8((const uint8_t*)hsv, (uint8_t*)rgb, n_pixels, 2, ST(s)); }
int ssp_aug_to_tensor_u8(const void* hwc, long long n_pixels, float* out_chw, void* s) { return aug_to_tensor_u8((const uint8_t*)hwc, n_pixels, out_chw, ST(s)); }
long long ssp_aug_batch_table_bytes(int n) { return aug_batch_table_bytes(n); }
int ssp_aug_batch_plan(const ssp_aug_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* stage_dims) {
  return aug_batch_plan(items, n, out_w, out_h, resample, table_host, table_bytes, stage_dims);
}
int ssp_aug_batch_run(const void* table_dev, int n, const int* stage_dims, void* s) { return aug_batch_run(table_dev, n, stage_dims, ST(s)); }
long long ssp_augm_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) { return augm_work_bytes(in_w, in_h, out_w, out_h, resample); }
long long ssp_augm_table_bytes(int n) { return augm_table_bytes(n); }
int ssp_augm_plan_begin(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(0, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}
int ssp_augm_plan_attempt(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(1, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}
int ssp_augm_plan_finish(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(2, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}
int ssp_augm_run(const void* table_dev, int n, const int* stage_dims, void* s) { return augm_run(table_dev, n, stage_dims, ST(s)); }
long long ssp_aug_sample_work_bytes(int ow, int oh, int bw, int bh, int cw, int ch, int out_w, int out_h, int resample) {
  return aug_sample_work_bytes(ow, oh, bw, bh, cw, ch, out_w, out_h, resample);
}
int ssp_aug_sample(const void* img, const void* mask, int ow, int oh, const void* bg, int bw, int bh, const void* luts, int pleft, int ptop, int cw,
                   int ch, int out_w, int out_h, int resample, void* work, long long work_bytes, void* out_u8, float* out_chw, void* s) {
  return aug_sample((const uint8_t*)img, (const uint8_t*)mask, ow, oh, (const uint8_t*)bg, bw, bh, (const uint8_t*)luts, pleft, ptop, cw, ch, out_w, out_h,
                    resample, (uint8_t*)work, work_bytes, (uint8_t*)out_u8, out_chw, ST(s));
}
}
