// Implicit-GEMM 3x3 convolution for NARROW layers (few channels, huge images): "band" loads + resident weights (wgmma).
//
// conv_tc.cu issues one TMA tile per tap; with <= 64 channels every 128-B row request carries little work and the
// kernel is bound by the L2->SM request rate (~0.3 row requests / clk / SM, measured), not by the tensor pipe.
// Here, per kernel row kh, ONE band of 136 activation rows [m0 + (kh-1)(W+1) - 1, +136) is loaded and the three
// horizontal taps kw = 0,1,2 are read from it by starting the wgmma descriptor 0 / 128 / 256 bytes into the band
// (rows are 128-B lines; the 128-B swizzle phase follows the absolute shared-memory address, so a row offset keeps TMA's
// and the tensor core's swizzles consistent with the descriptor's base_offset field left 0).  The weight tiles of all taps are loaded ONCE per CTA and stay resident in
// shared memory (they fit because the layer is narrow).  Row requests per tile drop from 9*(256+2*BN) to 3*272.
// Same operands / epilogue / outputs as conv_tc.cu; replaces it for block-2-like layers and their data gradients.
#include "ssp_common.cuh"
#include "gemm.cuh"
#include "tmap.cuh"

namespace ssp {

struct ConvBandParams {
  CUtensorMap tmA[2];     // box {64, 136}
  CUtensorMap tmB[2];     // box {64, bn}
  long long m_rows, store_rows;
  int m_tiles;
  int kc_per_tap, cin;
  int Wp, HpWp;
  int cout, bn, n_terms;
  int fmt;
  int stages, stage_bytes, b_bytes, res_bytes, acc_cols;
  float* out; long long out_ld;
  const float* bias; double* stat_sum; double* stat_sq; int epi;
};

namespace {
constexpr int kBandRows = 136;
constexpr int kBandBytes = kBandRows * 128;      // 17408 = 17 swizzle atoms
constexpr int kMaxStagesB = 8;
constexpr int kThreadsB = 256;
}

// BN: N tile, BF: operand format (1 = bf16), NT: products per K step (3: split hi/lo planes, 1: single term), KS: K steps of 16 per
// 64-channel chunk (2 when cin <= 32: the rest of the chunk is TMA zero fill).  All compile-time, so that every wgmma of a unit sits in
// straight-line code.
template <int BN, int BF, int NT, int KS>
__global__ void __launch_bounds__(kThreadsB, 1) conv_band_kernel(const __grid_constant__ ConvBandParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* res_base = smem;                                      // resident weights: [(tap, kc)][plane][bn x 128 B]
  uint8_t* stage_base = smem + p.res_bytes;                      // ring of A bands: [plane][136 x 128 B]
  double* acc_sum = (double*)(stage_base + (size_t)p.stages * p.stage_bytes);
  double* acc_sq = acc_sum + p.acc_cols;
  float* stg = (float*)(acc_sq + p.acc_cols);
  uint64_t* full_bar = (uint64_t*)((uint8_t*)stg + kStageRowsBytes);
  uint64_t* empty_bar = full_bar + kMaxStagesB;
  uint64_t* res_bar = empty_bar + kMaxStagesB;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int planes = NT == 3 ? 2 : 1;
  const int units = 3 * p.kc_per_tap;                            // (kh, kc) per tile

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&p.tmA[0]); tma_prefetch_desc(&p.tmB[0]); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // empty: one arrive per consumer warp
    mbar_init(res_bar, 1);
    fence_barrier_init();
  }
  if (p.epi == EPI_STATS)
    for (int i = threadIdx.x; i < 2 * p.acc_cols; i += kThreadsB) acc_sum[i] = 0.0;
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // ---- weights: all 9 taps x kc tiles, once ----
      mbar_expect_tx(res_bar, (uint32_t)p.res_bytes);
      for (int tap = 0; tap < 9; tap++)
        for (int kc = 0; kc < p.kc_per_tap; kc++)
          for (int pl = 0; pl < planes; pl++)
            tma_load_2d(res_base + (size_t)((tap * p.kc_per_tap + kc) * planes + pl) * p.b_bytes, &p.tmB[pl], res_bar,
                        tap * p.cin + kc * 64, 0);
      // ---- activation bands ----
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = (uint32_t)planes * kBandBytes;
      for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x) {
        const int m0 = t * 128;
        for (int kh = 0; kh < 3; kh++) {
          const int arow = m0 + (kh - 1) * p.Wp - 1;
          for (int kc = 0; kc < p.kc_per_tap; kc++) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = stage_base + (size_t)stage * p.stage_bytes;
            mbar_expect_tx(&full_bar[stage], tx);
            tma_load_2d(sa, &p.tmA[0], &full_bar[stage], kc * 64, arow);
            if (planes == 2) tma_load_2d(sa + kBandBytes, &p.tmA[1], &full_bar[stage], kc * 64, arow);
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ---- consumer warpgroup: wgmma into registers, then the epilogue (thread et = tile row et) ----
    const int et = threadIdx.x - 128;
    mbar_wait(res_bar, 0);
    int stage = 0; uint32_t phase = 0;
    const uint32_t rb = smem_u32(res_base);
    float acc[2][BN / 2];
    for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x) {
      int prev = -1;
      for (int u = 0; u < units; u++) {
        const int kh = u / p.kc_per_tap, kc = u % p.kc_per_tap;
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(stage_base + (size_t)stage * p.stage_bytes);
        const uint32_t b0 = rb + (uint32_t)((kh * 3 * p.kc_per_tap + kc) * planes) * p.b_bytes;
        const uint32_t b_tap = (uint32_t)(p.kc_per_tap * planes) * p.b_bytes;
        wgmma_fence();
#pragma unroll
        for (int kw = 0; kw < 3; kw++) {
          const uint32_t a_hi = sa + kw * 128, a_lo = a_hi + kBandBytes;     // tap kw starts kw rows into the band
          const uint32_t b_hi = b0 + kw * b_tap, b_lo = b_hi + p.b_bytes;
#pragma unroll
          for (int k = 0; k < KS; k++) {
            const uint64_t dbh = gmma_desc_k_sw128(b_hi + k * 32);
            const int sd = (u > 0 || kw > 0 || k > 0) ? 1 : 0;
#pragma unroll
            for (int h = 0; h < 2; h++) {
              const uint64_t dah = gmma_desc_k_sw128(a_hi + h * 8192 + k * 32);
              if constexpr (NT == 3) {
                wgmma_f32<BN, 0, 0, BF>(acc[h], gmma_desc_k_sw128(a_lo + h * 8192 + k * 32), dbh, sd);
                wgmma_f32<BN, 0, 0, BF>(acc[h], dah, gmma_desc_k_sw128(b_lo + k * 32), 1);
                wgmma_f32<BN, 0, 0, BF>(acc[h], dah, dbh, 1);
              } else {
                wgmma_f32<BN, 0, 0, BF>(acc[h], dah, dbh, sd);
              }
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous unit's MMAs are done: release its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      const long long m = (long long)t * 128 + et;
      bool valid = false;
      if (m < p.m_rows) { const int rem = (int)(m % p.HpWp); valid = (rem / p.Wp >= 1) && (rem % p.Wp >= 1); }
      float* orow = p.out + m * p.out_ld;
      const bool can_store = m < p.store_rows;
#pragma unroll
      for (int ch = 0; ch < BN / 32; ch++) {
        float v[32];
        acc_rows_32<BN>(acc, ch, stg, et, v);
        const int c0 = ch * 32;
        if (p.epi == EPI_BIAS) {
#pragma unroll
          for (int j = 0; j < 32; j++) if (c0 + j < p.cout) v[j] += __ldg(p.bias + c0 + j);
        }
        if (can_store) {
          if (c0 + 32 <= p.cout) {
#pragma unroll
            for (int j = 0; j < 32; j += 4)
              *reinterpret_cast<float4*>(orow + c0 + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          } else {
#pragma unroll
            for (int j = 0; j < 32; j++) if (c0 + j < p.cout) orow[c0 + j] = v[j];
          }
        }
        if (p.epi == EPI_STATS) {
          float s1[32], s2[32];
#pragma unroll
          for (int j = 0; j < 32; j++) { const float x = valid ? v[j] : 0.f; s1[j] = x; s2[j] = x * x; }
          const float cs = warp_transpose_sum32(s1, lane);
          const float cq = warp_transpose_sum32(s2, lane);
          if (c0 + lane < p.cout) { atomicAdd(&acc_sum[c0 + lane], (double)cs); atomicAdd(&acc_sq[c0 + lane], (double)cq); }
        }
      }
    }
    if (p.epi == EPI_STATS) {
      epi_bar();
      for (int c = et; c < p.cout; c += 128) {
        const double a = acc_sum[c], b = acc_sq[c];
        if (a != 0.0 || b != 0.0) { atomicAdd(p.stat_sum + c, a); atomicAdd(p.stat_sq + c, b); }
      }
    }
  }
}

typedef void (*BandKernel)(ConvBandParams);
// [BN 32 | 64 | 128][fp16 split | fp16 single | bf16 single][KS 2 | 4]
#define SSP_BAND_ROW(BN) {{conv_band_kernel<BN, 0, 3, 2>, conv_band_kernel<BN, 0, 3, 4>}, {conv_band_kernel<BN, 0, 1, 2>, conv_band_kernel<BN, 0, 1, 4>}, \
                          {conv_band_kernel<BN, 1, 1, 2>, conv_band_kernel<BN, 1, 1, 4>}}
static const BandKernel band_kernels[3][3][2] = {SSP_BAND_ROW(32), SSP_BAND_ROW(64), SSP_BAND_ROW(128)};
#undef SSP_BAND_ROW

// returns SSP_OK, or 1 when the layer is not eligible (caller falls back to the per-tap kernel)
int conv_gemm_band(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                   const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                   int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                   int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream) {
  if (taps != 9 || cout > 128 || a_fmt != b_fmt || (a_lo && b_lo && a_fmt == FMT_BF16)) return 1;
  if (!a_hi || !b_hi || !out || (a_ld % 8) || (b_ld % 8) || (out_ld % 4)) return fail_msg(SSP_ERR_ARG, "conv_gemm_band: bad argument");
  ConvBandParams p;
  Geom g{N, H, W};
  p.n_terms = (a_lo && b_lo) ? 3 : 1;
  const int planes = p.n_terms == 3 ? 2 : 1;
  int bn = ((cout + 31) / 32) * 32;         // the whole layer is one N tile of at most 128 (the accumulator is in registers)
  if (bn > 64) bn = 128;
  p.bn = bn; p.b_bytes = bn * 128;
  p.kc_per_tap = (cin + 63) / 64; p.cin = cin;
  p.res_bytes = 9 * p.kc_per_tap * planes * p.b_bytes;
  p.stage_bytes = planes * kBandBytes;
  p.acc_cols = ((cout + 31) / 32) * 32;
  const int fixed = 2 * p.acc_cols * 8 + kStageRowsBytes + (2 * kMaxStagesB + 1) * 8 + 1024;
  int stages = (227 * 1024 - fixed - p.res_bytes) / p.stage_bytes;
  if (stages > kMaxStagesB) stages = kMaxStagesB;
  if (stages < 2) return 1;                       // weights do not fit next to two bands: not a narrow layer
  p.stages = stages;
  p.m_rows = g.m_rows(); p.store_rows = out_rows;
  p.m_tiles = (int)((p.m_rows + 127) / 128);
  p.Wp = g.Wp(); p.HpWp = g.HpWp(); p.cout = cout;
  p.fmt = a_fmt;
  p.out = out; p.out_ld = out_ld; p.bias = bias; p.stat_sum = stat_sum; p.stat_sq = stat_sq; p.epi = epi;
  if (epi == EPI_STATS && (!stat_sum || !stat_sq)) return fail_msg(SSP_ERR_ARG, "conv_gemm_band: statistics buffers missing");
  int rc = 0;
  rc |= tmap_2d_16bit(&p.tmA[0], a_hi, (uint64_t)cin, (uint64_t)a_rows, (uint64_t)a_ld, 64, kBandRows, a_fmt == FMT_BF16);
  rc |= tmap_2d_16bit(&p.tmB[0], b_hi, (uint64_t)9 * cin, (uint64_t)b_rows, (uint64_t)b_ld, 64, bn, b_fmt == FMT_BF16);
  if (planes == 2) {
    rc |= tmap_2d_16bit(&p.tmA[1], a_lo, (uint64_t)cin, (uint64_t)a_rows, (uint64_t)a_ld, 64, kBandRows, a_fmt == FMT_BF16);
    rc |= tmap_2d_16bit(&p.tmB[1], b_lo, (uint64_t)9 * cin, (uint64_t)b_rows, (uint64_t)b_ld, 64, bn, b_fmt == FMT_BF16);
  }
  if (rc) return fail_msg(SSP_ERR_DRIVER, "conv_gemm_band: cuTensorMapEncodeTiled failed");
  static int sms = 0, configured = 0;
  if (!sms) sms = ssp_sm_count();
  if (!configured) {
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 18 && e == cudaSuccess; i++)
      e = cudaFuncSetAttribute(band_kernels[i / 6][(i / 2) % 3][i % 2], cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  const int grid = p.m_tiles < sms ? p.m_tiles : sms;
  const int smem_bytes = p.res_bytes + stages * p.stage_bytes + fixed;
  const int variant = planes == 2 ? 0 : (a_fmt == FMT_BF16 ? 2 : 1);
  auto kern = band_kernels[bn == 32 ? 0 : (bn == 64 ? 1 : 2)][variant][cin <= 32 ? 0 : 1];
  kern<<<grid, kThreadsB, smem_bytes, stream>>>(p);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

}  // namespace ssp
