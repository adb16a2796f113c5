// The convolution GEMM launchers behind ssp_conv_gemm / ssp_wgrad_gemm (abi.cu) and the inference entry points of conv_tc.cu.
// Operands as in include/ssp_b200.h; conv_gemm_band and conv_gemm_bandt return 1 when the layer is not eligible.
#pragma once
#include "ssp_common.cuh"

namespace ssp {

// forward and data gradient: out[m][n] = sum_tap sum_c A[m + shift(tap)][c] * B[n][tap*cin + c]
int conv_gemm_tc(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                 const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                 int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                 int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream, const FusedAct* fa,
                 const SplitK* sk);
int conv_gemm_band(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                   const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                   int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                   int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream);
int conv_gemm_bandt(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                    const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                    int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                    int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream);
int conv_gemm_simt(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                   const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                   int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                   int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream);

// weight gradient: dw[co][tap][ci] += scale * sum_m dy[m][co] * x[m + shift(tap)][ci]
int wgrad_gemm_tc(const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt,
                  const void* x, long long x_rows, int x_ld, int cin, int x_fmt,
                  int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, cudaStream_t stream);
int wgrad_gemm_simt(const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt,
                    const void* x, long long x_rows, int x_ld, int cin, int x_fmt,
                    int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, cudaStream_t stream);

}  // namespace ssp
