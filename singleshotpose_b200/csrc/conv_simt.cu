// fp32 CUDA-core versions of the two GEMM-shaped kernels (same operands, same outputs as conv_tc.cu /
// wgrad_tc.cu).  They are the on-device cross-check for the tensor-core kernels (SSP_IMPL_SIMT through the
// ABI); all arithmetic is fp32 FFMA on hi+lo reconstructed operands.
#include "ssp_common.cuh"
#include "gemm.cuh"

namespace ssp {

struct ConvSimtParams {
  const uint16_t *a_hi, *a_lo, *b_hi, *b_lo;
  long long a_rows, m_rows, store_rows;
  int a_ld, b_ld, cin, taps, cout, b_rows;
  int shifts[9];
  int Wp, HpWp, a_fmt, b_fmt;
  float* out; long long out_ld;
  const float* bias; double* stat_sum; double* stat_sq; int epi;
};

__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvSimtParams p) {
  __shared__ float sA[16][64 + 4];
  __shared__ float sB[16][64 + 4];
  __shared__ float sRed[2][16][64];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const long long m0 = (long long)blockIdx.x * 64;
  const int n0 = blockIdx.y * 64;
  float acc[4][4] = {};
  const int lr = threadIdx.x >> 2;          // 0..63 : tile row loaded by this thread
  const int lk = (threadIdx.x & 3) * 4;     // 0,4,8,12 : first of 4 k values
  for (int tap = 0; tap < p.taps; tap++) {
    const long long arow = m0 + lr + p.shifts[tap];
    const bool arow_ok = arow >= 0 && arow < p.a_rows;
    for (int k0 = 0; k0 < p.cin; k0 += 16) {
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c = k0 + lk + j;
        float a = 0.f, b = 0.f;
        if (arow_ok && c < p.cin) {
          a = cvt16_to_f32(p.a_hi[arow * p.a_ld + c], p.a_fmt);
          if (p.a_lo) a += cvt16_to_f32(p.a_lo[arow * p.a_ld + c], p.a_fmt);
        }
        const int n = n0 + lr;
        if (n < p.b_rows && c < p.cin) {
          const long long bi = (long long)n * p.b_ld + (long long)tap * p.cin + c;
          b = cvt16_to_f32(p.b_hi[bi], p.b_fmt);
          if (p.b_lo) b += cvt16_to_f32(p.b_lo[bi], p.b_fmt);
        }
        sA[lk + j][lr] = a;
        sB[lk + j][lr] = b;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 16; k++) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { a[i] = sA[k][ty * 4 + i]; b[i] = sB[k][tx * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  float cs[4] = {}, cq[4] = {};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const long long m = m0 + ty * 4 + i;
    bool valid = false;
    if (m < p.m_rows) { const int rem = (int)(m % p.HpWp); valid = (rem / p.Wp >= 1) && (rem % p.Wp >= 1); }
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = n0 + tx * 4 + j;
      float v = acc[i][j];
      if (n < p.cout) {
        if (p.epi == EPI_BIAS) v += p.bias[n];
        if (m < p.store_rows) p.out[m * p.out_ld + n] = v;
        if (valid) { cs[j] += v; cq[j] += v * v; }
      }
    }
  }
  if (p.epi == EPI_STATS) {
#pragma unroll
    for (int j = 0; j < 4; j++) { sRed[0][ty][tx * 4 + j] = cs[j]; sRed[1][ty][tx * 4 + j] = cq[j]; }
    __syncthreads();
    if (threadIdx.x < 128) {
      const int which = threadIdx.x >> 6, c = threadIdx.x & 63;
      double s = 0.0;
      for (int r = 0; r < 16; r++) s += (double)sRed[which][r][c];
      if (n0 + c < p.cout) atomicAdd((which ? p.stat_sq : p.stat_sum) + n0 + c, s);
    }
  }
}

int conv_gemm_simt(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                   const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                   int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                   int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream) {
  if (!a_hi || !b_hi || !out || (taps != 1 && taps != 9)) return fail_msg(SSP_ERR_ARG, "conv_gemm_simt: bad argument");
  ConvSimtParams p;
  Geom g{N, H, W};
  p.a_hi = (const uint16_t*)a_hi; p.a_lo = (const uint16_t*)a_lo; p.b_hi = (const uint16_t*)b_hi; p.b_lo = (const uint16_t*)b_lo;
  p.a_rows = a_rows; p.m_rows = g.m_rows(); p.store_rows = out_rows;
  p.a_ld = a_ld; p.b_ld = b_ld; p.cin = cin; p.taps = taps; p.cout = cout; p.b_rows = b_rows;
  for (int t = 0; t < 9; t++) p.shifts[t] = (taps == 9) ? ((t / 3) - 1) * g.Wp() + ((t % 3) - 1) : 0;
  p.Wp = g.Wp(); p.HpWp = g.HpWp(); p.a_fmt = a_fmt; p.b_fmt = b_fmt;
  p.out = out; p.out_ld = out_ld; p.bias = bias; p.stat_sum = stat_sum; p.stat_sq = stat_sq; p.epi = epi;
  dim3 grid((unsigned)((p.m_rows + 63) / 64), (unsigned)((cout + 63) / 64));
  conv_simt_kernel<<<grid, 256, 0, stream>>>(p);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

// ---------------------------------------------------------------------------------------------
struct WgradSimtParams {
  const uint16_t *dy, *x;
  long long dy_rows, x_rows, m_rows;
  int dy_ld, x_ld, cout, cin, taps, dy_fmt, x_fmt, splits;
  int shifts[9];
  float* dw; int dw_ld, cin_store; float scale;
};

__global__ void __launch_bounds__(256) wgrad_simt_kernel(const WgradSimtParams p) {
  __shared__ float sA[16][64 + 4];   // dY chunk: [k rows][co]
  __shared__ float sB[16][64 + 4];   // X chunk:  [k rows][ci]
  const int ci_tiles = (p.cin + 63) / 64;
  const int co0 = (blockIdx.x / ci_tiles) * 64, ci0 = (blockIdx.x % ci_tiles) * 64;
  const int tap = blockIdx.y;
  const long long per = ((p.m_rows + p.splits - 1) / p.splits + 15) / 16 * 16;
  const long long k_begin = (long long)blockIdx.z * per;
  long long k_end = k_begin + per; if (k_end > p.m_rows) k_end = p.m_rows;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lr = threadIdx.x >> 4;          // k row 0..15
  const int lc = (threadIdx.x & 15) * 4;    // channel 0..60
  float acc[4][4] = {};
  for (long long k0 = k_begin; k0 < k_end; k0 += 16) {
    const long long r = k0 + lr, rx = r + p.shifts[tap];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float a = 0.f, b = 0.f;
      if (r < k_end && r < p.dy_rows && co0 + lc + j < p.cout) a = cvt16_to_f32(p.dy[r * p.dy_ld + co0 + lc + j], p.dy_fmt);
      if (r < k_end && rx >= 0 && rx < p.x_rows && ci0 + lc + j < p.cin) b = cvt16_to_f32(p.x[rx * p.x_ld + ci0 + lc + j], p.x_fmt);
      sA[lr][lc + j] = a; sB[lr][lc + j] = b;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; k++) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { a[i] = sA[k][ty * 4 + i]; b[i] = sB[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int co = co0 + ty * 4 + i, ci = ci0 + tx * 4 + j;
      if (co < p.cout && ci < p.cin_store && acc[i][j] != 0.f)
        atomicAdd(p.dw + ((long long)co * p.taps + tap) * p.dw_ld + ci, acc[i][j] * p.scale);
    }
}

int wgrad_gemm_simt(const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt,
                    const void* x, long long x_rows, int x_ld, int cin, int x_fmt,
                    int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, cudaStream_t stream) {
  if (!dy || !x || !dw || (taps != 1 && taps != 9)) return fail_msg(SSP_ERR_ARG, "wgrad_gemm_simt: bad argument");
  WgradSimtParams p;
  Geom g{N, H, W};
  p.dy = (const uint16_t*)dy; p.x = (const uint16_t*)x; p.dy_rows = dy_rows; p.x_rows = x_rows; p.m_rows = g.m_rows();
  p.dy_ld = dy_ld; p.x_ld = x_ld; p.cout = cout; p.cin = cin; p.taps = taps; p.dy_fmt = dy_fmt; p.x_fmt = x_fmt;
  for (int t = 0; t < 9; t++) p.shifts[t] = (taps == 9) ? ((t / 3) - 1) * g.Wp() + ((t % 3) - 1) : 0;
  const int tiles = ((cout + 63) / 64) * ((cin + 63) / 64);
  int splits = (int)((p.m_rows + 4095) / 4096);
  const int want = (4 * ssp_sm_count() + tiles * taps - 1) / (tiles * taps);
  if (splits > want) splits = want;
  if (splits < 1) splits = 1;
  p.splits = splits; p.dw = dw; p.dw_ld = dw_ld; p.cin_store = cin_store; p.scale = scale;
  dim3 grid(tiles, taps, splits);
  wgrad_simt_kernel<<<grid, 256, 0, stream>>>(p);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

}  // namespace ssp
