// The parts of the extern "C" surface of libssp_b200.so (include/ssp_b200.h) that belong to no single kernel file: the error
// state, the layout helpers and the dispatchers over the convolution GEMMs.  Every other entry point is defined beside its kernels.
#include "ssp_common.cuh"
#include "gemm.cuh"
#include <stdio.h>

namespace ssp {
static thread_local char g_err[512] = "";
int fail_cuda(cudaError_t e, const char* file, int line) {
  snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s:%d", (int)e, cudaGetErrorString(e), file, line);
  return SSP_ERR_CUDA;
}
int fail_msg(int code, const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg); return code; }
}  // namespace ssp

using namespace ssp;
#define ST(s) ((cudaStream_t)(s))

extern "C" {
int ssp_version(void) { return 100; }
const char* ssp_last_error(void) { return g_err; }
long long ssp_flat_alloc_rows(int N, int H, int W) { return flat_alloc_rows(N, H, W); }
long long ssp_flat_row(int n, int h, int w, int H, int W) { Geom g{1, H, W}; return g.row(n, h, w); }

int ssp_conv_gemm(int impl, const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo,
                  int b_rows, int b_ld, int a_fmt, int b_fmt, int N, int H, int W, int taps, int cout, float* out, int out_ld,
                  long long out_rows, int epi, const float* bias, double* ssum, double* ssq, void* s) {
  if (epi == SSP_EPI_F16) {          // fp16 data-gradient planes: the operand-swapped kernel where eligible, the per-tap kernel otherwise
    if (impl != SSP_IMPL_BANDT && impl != SSP_IMPL_TC2) return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm: SSP_EPI_F16 needs SSP_IMPL_BANDT or SSP_IMPL_TC2");
    if (impl == SSP_IMPL_BANDT) {
      const int rc = conv_gemm_bandt(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s));
      if (rc != 1) return rc;
    }
    return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s), nullptr, nullptr);
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
  return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, a_fmt, b_fmt, N, H, W, taps, cout, out, out_ld, out_rows, epi, bias, ssum, ssq, ST(s), nullptr, nullptr);
}
int ssp_wgrad_gemm(int impl, const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt, const void* x, long long x_rows, int x_ld,
                   int cin, int x_fmt, int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, void* s) {
  if (impl == SSP_IMPL_SIMT) return wgrad_gemm_simt(dy, dy_rows, dy_ld, cout, dy_fmt, x, x_rows, x_ld, cin, x_fmt, N, H, W, taps, dw, dw_ld, cin_store, scale, ST(s));
  return wgrad_gemm_tc(dy, dy_rows, dy_ld, cout, dy_fmt, x, x_rows, x_ld, cin, x_fmt, N, H, W, taps, dw, dw_ld, cin_store, scale, ST(s));
}
}  // extern "C"
