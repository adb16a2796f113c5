// Implicit-GEMM convolution for layers with FEW OUTPUT CHANNELS, operands swapped: the tensor cores compute the TRANSPOSED tile
//
//     D^T[n, m] = sum_tap sum_c  Wt[n, tap*cin + c] * X[m + shift(tap), c]          (n = output channel, m = pixel row)
//
// i.e. the weights are the M side (128 rows: two 64-row wgmma halves) and a band of 128 PIXELS is the N side of every wgmma.
// Why: with cout <= 64 the forward GEMM of conv_band.cu issues narrow 64 x 64 x 16 instructions; swapped, every instruction is
// 64 x 128 x 16 whatever the layer's width.  For the split-fp16 forward (x = hi + lo, three products) the unused half of
// the M side carries the second weight plane: rows 0-63 = W_hi, rows 64-127 = W_lo, so the MMAs against X_hi yield
// W_hi X_hi and W_lo X_hi, those against X_lo yield W_hi X_lo (and W_lo X_lo, 2^-22, harmless); row n and row n + 64 of the
// accumulator are held by the same thread and are added in registers.
//   * activations: per kernel row kh ONE band of np + 8 rows (conv_band.cu's trick): the three horizontal taps are the same band
//     read 0 / 128 / 256 bytes further in (the B descriptor's start address; the 128-B swizzle follows the absolute address);
//   * weights: all taps resident in shared memory, loaded once per CTA;
//   * epilogue: thread = output channel (accumulator row, through shared memory), 32 consecutive pixels per chunk; for every pixel the warp stores 32
//     consecutive channels = one 128-B line of the row-major output; BN statistics per thread (its channel) in fp64, pixel
//     validity (pad rows of the padded-flat layout) from a per-tile ballot mask.
// Same operands / outputs as conv_band.cu (drop-in behind ssp_conv_gemm, SSP_IMPL_BANDT); not eligible (returns 1): cout > 64 with
// split operands, cout > 128 single-term, bias epilogue, weights that do not fit next to two bands.
// Replaces nn.Conv2d of reference darknet.py:156-160 for the narrow blocks, and their data gradients (train.py:103).
#include "ssp_common.cuh"
#include "gemm.cuh"
#include "tmap.cuh"

namespace ssp {

struct ConvBandTParams {
  CUtensorMap tmX[2][2];   // [plane][part]: band boxes {64, rows0} and {64, rows1}
  CUtensorMap tmW[2];      // [plane]: weight box {64, wbox_rows}
  long long m_rows, store_rows;
  int m_tiles, np;         // pixels per tile = MMA N (128)
  int taps, nk;            // nk = 3 (3x3) or 1 (1x1)
  int kc_per_tap, cin;
  int Wp, HpWp;
  int cout, stacked;
  int ovl;                 // 32-channel 3x3 layer through the overlapping-row tensor map: a band row = [pixel | pixel + 1], K chunk 0 = taps kw 0,1, chunk 1 = tap kw 2
  int fmt;
  int stages, stage_bytes, plane_bytes, rows0, rows1;
  int w_tile_bytes, res_bytes;
  float* out; long long out_ld;
  double* stat_sum; double* stat_sq; int epi;
};

namespace {
constexpr int kMaxStagesT = 6;
constexpr int kThreadsT = 256;
constexpr int kNp = 128;                           // pixels per tile: the 128 x 128 accumulator is 128 registers per thread
}

// BF: operand format (1 = bf16); ST: stacked W_hi / W_lo planes (split fp16 forward); UP: rows 64-127 of the M side are multiplied
// (ST, or more than 64 output channels); NK: kernel rows (3: 3x3, 1: 1x1); OVL: overlapping-row band (32-channel 3x3 layers).
// All compile-time, so that every wgmma of a unit sits in straight-line code.
template <int BF, bool ST, bool UP, int NK, bool OVL>
__global__ void __launch_bounds__(kThreadsT, 1) conv_bandt_kernel(const __grid_constant__ ConvBandTParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* res_base = smem;                                       // resident weight tiles [(tap, kc)][w_tile_bytes]
  uint8_t* stage_base = smem + p.res_bytes;                       // ring of bands: [plane][(rows0 + rows1) x 128 B]
  float* stg = (float*)(stage_base + (size_t)p.stages * p.stage_bytes);
  uint32_t* vmask = (uint32_t*)((uint8_t*)stg + (p.stacked ? kStageRowsBytes / 2 : kStageRowsBytes));   // [2 x 8 words]
  uint64_t* full_bar = (uint64_t*)(vmask + 16);
  uint64_t* empty_bar = full_bar + kMaxStagesT;
  uint64_t* res_bar = empty_bar + kMaxStagesT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int planes = p.stacked ? 2 : 1;
  const int units = p.nk * p.kc_per_tap;                          // (kh, kc) per tile

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&p.tmX[0][0]); tma_prefetch_desc(&p.tmW[0]); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // empty: one arrive per consumer warp
    mbar_init(res_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // ---- weights: every (tap, kc) tile, once.  stacked: rows 0-63 <- W_hi, rows 64-127 <- W_lo of the same 16 KB tile ----
      const int wbox_rows = p.stacked ? 64 : p.w_tile_bytes / 128;
      mbar_expect_tx(res_bar, (uint32_t)((p.ovl ? 6 : p.taps * p.kc_per_tap) * planes * wbox_rows * 128));
      const int ntile = p.ovl ? 6 : p.taps * p.kc_per_tap;
      for (int ti = 0; ti < ntile; ti++) {
        // ovl: tile 2 kh = the 64 K columns of taps (kh, 0) and (kh, 1), tile 2 kh + 1 = tap (kh, 2) (its upper 32 columns are never multiplied)
        const int kcol = p.ovl ? (ti >> 1) * 3 * p.cin + (ti & 1) * 64 : (ti / p.kc_per_tap) * p.cin + (ti % p.kc_per_tap) * 64;
        uint8_t* wt = res_base + (size_t)ti * p.w_tile_bytes;
        tma_load_2d(wt, &p.tmW[0], res_bar, kcol, 0);
        if (p.stacked) tma_load_2d(wt + 64 * 128, &p.tmW[1], res_bar, kcol, 0);
      }
      // ---- activation bands ----
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = (uint32_t)planes * (uint32_t)p.plane_bytes;
      for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x) {
        const int m0 = t * p.np;
        for (int kh = 0; kh < p.nk; kh++) {
          const int arow = p.nk == 3 ? m0 + (kh - 1) * p.Wp - 1 : m0;
          for (int kc = 0; kc < p.kc_per_tap; kc++) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = stage_base + (size_t)stage * p.stage_bytes;
            mbar_expect_tx(&full_bar[stage], tx);
            for (int pl = 0; pl < planes; pl++) {
              tma_load_2d(sa + (size_t)pl * p.plane_bytes, &p.tmX[pl][0], &full_bar[stage], kc * 64, arow);
              if (p.rows1) tma_load_2d(sa + (size_t)pl * p.plane_bytes + (size_t)p.rows0 * 128, &p.tmX[pl][1], &full_bar[stage], kc * 64, arow + p.rows0);
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ---- consumer warpgroup: wgmma into registers, then the epilogue: thread et = weight row = output channel; columns = pixels ----
    const int et = threadIdx.x - 128;
    const bool stats = p.epi == EPI_STATS;
    const int n_own = et;                                          // output channel of this thread (stacked: rows 64-127 are folded into 0-63)
    const bool own = n_own < p.cout && (!ST || n_own < 64);
    double d1 = 0.0, d2 = 0.0;
    mbar_wait(res_bar, 0);
    int stage = 0; uint32_t phase = 0;
    const uint32_t rb = smem_u32(res_base);
    float acc[2][kNp / 2];
    int it = 0;
    for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x, it++) {
      const long long m0 = (long long)t * p.np;
      uint32_t* vmt = vmask + (it & 1) * 8;                        // a slower warp may still read the previous tile's words
      if (stats) {
        const long long m = m0 + et;
        bool valid = false;
        if (m < p.m_rows) { const int rem = (int)(m % p.HpWp); valid = (rem / p.Wp >= 1) && (rem % p.Wp >= 1); }
        const uint32_t b = __ballot_sync(0xffffffffu, valid);
        if (lane == 0) vmt[et >> 5] = b;                           // read after the staging barriers of the first chunk
      }
      int prev = -1;
      for (int u = 0; u < units; u++) {
        const int kh = u / p.kc_per_tap, kc = u % p.kc_per_tap;
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(stage_base + (size_t)stage * p.stage_bytes);
        constexpr int ngrp = OVL ? 2 : NK;
        wgmma_fence();
#pragma unroll
        for (int kw = 0; kw < ngrp; kw++) {
          // ovl: group 0 = taps kw 0,1 (64 K of a [pixel | pixel + 1] row), group 1 = tap kw 2 (32 K, band read two rows further in)
          const uint32_t wt = rb + (uint32_t)((OVL ? kh * 2 + kw : (kh * NK + kw) * p.kc_per_tap + kc) * p.w_tile_bytes);
          const uint32_t x_hi = sa + (OVL ? 2 * kw : kw) * 128, x_lo = x_hi + (uint32_t)p.plane_bytes;     // tap kw starts kw rows into the band
          // K steps of 16: all four (channels >= cin are TMA zero fill, so extra steps add exact zeros), except the overlapping-row
          // group 1 whose upper 32 columns are the next pixel's channels
          const int ks = (OVL && kw == 1) ? 2 : 4;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            if (k < ks) {
              const int sd = (u > 0 || kw > 0 || k > 0) ? 1 : 0;
              const uint64_t dxh = gmma_desc_k_sw128(x_hi + k * 32);
#pragma unroll
              for (int h = 0; h < 2; h++) {
                if (h == 1 && !UP) continue;
                const uint64_t da = gmma_desc_k_sw128(wt + h * 8192 + k * 32);
                if constexpr (ST) {
                  wgmma_f32<kNp, 0, 0, BF>(acc[h], da, gmma_desc_k_sw128(x_lo + k * 32), sd);   // small terms first
                  wgmma_f32<kNp, 0, 0, BF>(acc[h], da, dxh, 1);
                } else {
                  wgmma_f32<kNp, 0, 0, BF>(acc[h], da, dxh, sd);
                }
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
      if constexpr (ST) {
#pragma unroll
        for (int i = 0; i < kNp / 2; i++) acc[0][i] += acc[1][i];   // W_hi X + W_lo X: row n + 64 onto row n (same thread)
      }
      float ts1 = 0.f, ts2 = 0.f;
#pragma unroll
      for (int ch = 0; ch < kNp / 32; ch++) {
        float r[32];
        acc_rows_32<kNp, ST ? 1 : 2>(acc, ch, stg, et, r);            // stacked: only rows 0-63 carry output, half the staging buffer
        const uint32_t vm = stats ? vmt[ch] : 0u;
        if (own) {
          // branch-free inner loops: a predicated store per element compiles to a BSSY / BRA / BSYNC triple per column
          float* o = p.out + (m0 + ch * 32) * p.out_ld + n_own;
          if (p.epi == EPI_F16) {                  // fp16 data gradient: the warp writes 64 B of every pixel row
            uint16_t* o16 = reinterpret_cast<uint16_t*>(p.out) + (m0 + ch * 32) * p.out_ld + n_own;
            if (m0 + ch * 32 + 32 <= p.store_rows) {
#pragma unroll
              for (int j = 0; j < 32; j++) { *o16 = cvt_f32_to_16(r[j], FMT_F16); o16 += p.out_ld; }
            } else {
              for (int j = 0; j < 32; j++) if (m0 + ch * 32 + j < p.store_rows) o16[(long long)j * p.out_ld] = cvt_f32_to_16(r[j], FMT_F16);
            }
          } else if (m0 + ch * 32 + 32 <= p.store_rows) {
#pragma unroll
            for (int j = 0; j < 32; j++) { *o = r[j]; o += p.out_ld; }
          } else {
            for (int j = 0; j < 32; j++) if (m0 + ch * 32 + j < p.store_rows) o[(long long)j * p.out_ld] = r[j];
          }
          if (stats) {
#pragma unroll
            for (int j = 0; j < 32; j++) { const float v = ((vm >> j) & 1u) ? r[j] : 0.f; ts1 += v; ts2 = fmaf(v, v, ts2); }
          }
        }
      }
      d1 += (double)ts1; d2 += (double)ts2;
    }
    if (stats && own && (d1 != 0.0 || d2 != 0.0)) {
      atomicAdd(p.stat_sum + n_own, d1);
      atomicAdd(p.stat_sq + n_own, d2);
    }
  }
}

typedef void (*BandTKernel)(ConvBandTParams);
// [stacked fp16 | fp16 <= 64 ch | fp16 > 64 ch | bf16 <= 64 ch | bf16 > 64 ch][1x1 | 3x3 | 3x3 overlapping rows]
#define SSP_BANDT_ROW(BF, ST, UP) {conv_bandt_kernel<BF, ST, UP, 1, false>, conv_bandt_kernel<BF, ST, UP, 3, false>, conv_bandt_kernel<BF, ST, UP, 3, true>}
static const BandTKernel bandt_kernels[5][3] = {SSP_BANDT_ROW(0, true, true), SSP_BANDT_ROW(0, false, false), SSP_BANDT_ROW(0, false, true),
                                                SSP_BANDT_ROW(1, false, false), SSP_BANDT_ROW(1, false, true)};
#undef SSP_BANDT_ROW

static int g_bandt_launches = 0;

// returns SSP_OK, or 1 when the layer is not eligible (caller falls back to conv_band / the per-tap kernels)
int conv_gemm_bandt(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                    const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                    int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                    int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream) {
  (void)bias;
  if ((taps != 9 && taps != 1) || epi == EPI_BIAS || epi == EPI_BNACT) return 1;
  if (!a_hi || !b_hi || !out || (a_ld % 8) || (b_ld % 8)) return fail_msg(SSP_ERR_ARG, "conv_gemm_bandt: bad argument");
  ConvBandTParams p;
  Geom g{N, H, W};
  p.stacked = (a_lo && b_lo) ? 1 : 0;
  if (p.stacked ? cout > 64 : cout > 128) return 1;
  if (epi == EPI_F16 && p.stacked) return 1;
  if (a_fmt != b_fmt) return 1;
  const int planes = p.stacked ? 2 : 1;
  p.taps = taps; p.nk = taps == 9 ? 3 : 1;
  p.kc_per_tap = (cin + 63) / 64; p.cin = cin; p.cout = cout;
  // 32-channel 3x3 layer with a row pitch of exactly 32 channels: overlapping-row tensor map (a legal tensor map: rows may overlap) -- a band row
  // is [pixel | pixel + 1], dense 128 B instead of 64 B + zero fill, and the taps (kh, 0), (kh, 1) share one 64-wide K chunk: six resident
  // weight tiles instead of nine, which is what makes room for a third ring stage (block 2 forward: 477 us at 42 % tensor-active with two)
  p.ovl = (taps == 9 && cin == 32 && a_ld == 32) ? 1 : 0;
  const int mrows = p.stacked ? 128 : ((cout + 7) / 8) * 8;
  p.w_tile_bytes = mrows * 128;
  long long res = (long long)(p.ovl ? 6 : taps * p.kc_per_tap) * p.w_tile_bytes + (128 - mrows) * 128;      // every MMA reads 128 rows from its tile's start
  res = (res + 1023) / 1024 * 1024;
  const int fixed = (p.stacked ? kStageRowsBytes / 2 : kStageRowsBytes) + 64 + (2 * kMaxStagesT + 1) * 8 + 1024;
  const int np = kNp;
  const long long st = (227 * 1024 - fixed - res) / ((long long)planes * (taps == 9 ? np + 8 : np) * 128);
  if (res >= 200 * 1024 || st < 2) return 1;
  const int stages = (int)(st > kMaxStagesT ? kMaxStagesT : st);
  p.np = np; p.stages = stages; p.res_bytes = (int)res;
  if (taps == 9) { p.rows0 = np + 8; p.rows1 = 0; } else { p.rows0 = np; p.rows1 = 0; }
  p.plane_bytes = (p.rows0 + p.rows1) * 128;
  p.stage_bytes = planes * p.plane_bytes;
  p.m_rows = g.m_rows(); p.store_rows = out_rows;
  p.m_tiles = (int)((p.m_rows + np - 1) / np);
  p.Wp = g.Wp(); p.HpWp = g.HpWp();
  p.fmt = a_fmt;
  p.out = out; p.out_ld = out_ld; p.stat_sum = stat_sum; p.stat_sq = stat_sq; p.epi = epi;
  if (epi == EPI_STATS && (!stat_sum || !stat_sq)) return fail_msg(SSP_ERR_ARG, "conv_gemm_bandt: statistics buffers missing");
  int rc = 0;
  for (int pl = 0; pl < planes; pl++) {
    const void* xa = pl ? a_lo : a_hi; const void* wa = pl ? b_lo : b_hi;
    const uint64_t xin = p.ovl ? 64 : (uint64_t)cin, xrows = p.ovl ? (uint64_t)a_rows - 1 : (uint64_t)a_rows;
    rc |= tmap_2d_16bit(&p.tmX[pl][0], xa, xin, xrows, (uint64_t)a_ld, 64, p.rows0, a_fmt == FMT_BF16);
    if (p.rows1) rc |= tmap_2d_16bit(&p.tmX[pl][1], xa, xin, xrows, (uint64_t)a_ld, 64, p.rows1, a_fmt == FMT_BF16);
    rc |= tmap_2d_16bit(&p.tmW[pl], wa, (uint64_t)taps * cin, (uint64_t)b_rows, (uint64_t)b_ld, 64, p.stacked ? 64 : mrows, b_fmt == FMT_BF16);
  }
  if (rc) return fail_msg(SSP_ERR_DRIVER, "conv_gemm_bandt: cuTensorMapEncodeTiled failed");
  static int sms = 0, configured = 0;
  if (!sms) sms = ssp_sm_count();
  if (!configured) {
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 15 && e == cudaSuccess; i++)
      e = cudaFuncSetAttribute(bandt_kernels[i / 3][i % 3], cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  const int grid = p.m_tiles < sms ? p.m_tiles : sms;
  const int variant = p.stacked ? 0 : 1 + 2 * (a_fmt == FMT_BF16 ? 1 : 0) + (cout > 64 ? 1 : 0);
  bandt_kernels[variant][p.ovl ? 2 : (taps == 9 ? 1 : 0)]<<<grid, kThreadsT, p.res_bytes + stages * p.stage_bytes + fixed, stream>>>(p);
  SSP_CHECK_LAUNCH();
  g_bandt_launches++;
  return SSP_OK;
}

}  // namespace ssp

extern "C" {
int ssp_conv_bandt_launches(void) { return ssp::g_bandt_launches; }
}  // extern "C"
