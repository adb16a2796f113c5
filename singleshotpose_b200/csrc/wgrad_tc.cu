// Weight-gradient GEMM on the Hopper tensor cores (wgmma):   dW[co, tap, ci] += sum_m dY[m, co] * X[m + shift(tap), ci]
//
// The contraction runs over pixels (rows of the padded-flat matrices), so BOTH operands are "MN-major"
// for the tensor core (channels contiguous, K = rows): the TMA boxes [64 rows][64 channels] land in
// shared memory exactly in the canonical MN-major SWIZZLE_128B layout, no transposed copies needed.
// dY has zero pad rows, X has zero pad rows, so the shifted product never picks up wrap-around terms.
// Work item = (co tile of 128, ci tile of BN, tap); the 128 x BN fp32 accumulator lives in the registers of one warpgroup.
// Narrow layers have few items and very long K (all pixels of the batch), so K is split over the CTAs of a thread-block cluster
// (1, 2, 4 or 8 CTAs, rank r = K range r): rank 0 adds the other ranks' partial sums from their shared memory in rank order and
// is the only writer of its dW elements.  The result is the same bits on every run (no atomics, whose order would vary), and
// dW -- which the caller zeroes once per step -- receives exactly one `+=` per element and launch.  Output layout
// [co][tap][ci] is the layout the master weights are kept in (engine.py), i.e. the gradient of nn.Conv2d.weight seen through a
// permuted view.  Replaces the conv weight-gradient autograd computes for reference train.py:103.
#include "ssp_common.cuh"
#include "gemm.cuh"
#include "tmap.cuh"

namespace ssp {

struct WgradTcParams {
  CUtensorMap tmDy;     // [rows][cout]   box {64, 64}
  CUtensorMap tmX;      // [rows][cin]    box {64, 64}
  long long m_rows;
  int co_tiles, ci_tiles, taps, splits;   // splits = CTAs per cluster
  int kblocks_total;    // ceil(m_rows / 64)
  int shifts[9];
  int cout, cin, bn;
  int xbox0;            // index of the first X box inside a stage: 2 (two dY boxes), or 1 when cout <= 64
  int fmt;
  int stages, stage_bytes;
  float* dw;
  int dw_ld, cin_store;  // row pitch of dW per (co, tap) and number of real input channels
  float scale;          // applied to the reduced sums before they are added to dW (loss-scale undo)
};

static constexpr int kBox = 64 * 128;   // 64 rows x 64 ch x 2 B
static constexpr int kMaxStagesW = 8;
static constexpr int kThreadsW = 256;

// BN: N tile, BF: operand format (1 = bf16), TWO: cout > 64 -- both 64-row halves of the M side are multiplied (in a last tile with
// fewer than 65 channels the second half multiplies a stale slot and is never stored).  Compile-time, so that every wgmma of a
// k-block sits in straight-line code.
template <int BN, int BF, bool TWO>
__global__ void __launch_bounds__(kThreadsW, 1) wgrad_tc_kernel(const __grid_constant__ WgradTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  float* stg = (float*)(smem + (size_t)p.stages * p.stage_bytes);
  uint64_t* full_bar = (uint64_t*)((uint8_t*)stg + kStageRowsBytes);
  uint64_t* empty_bar = full_bar + kMaxStagesW;
  uint64_t* ready_bar = empty_bar + kMaxStagesW;    // rank 0: the other ranks' chunk is staged (count splits - 1)
  uint64_t* free_bar = ready_bar + 1;               // rank r > 0: rank 0 has read the staged chunk (count 1)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int cid = blockIdx.x / p.splits, ncl = gridDim.x / p.splits;
  const int tiles = p.co_tiles * p.ci_tiles * p.taps;
  constexpr int nb = BN / 64;                       // X boxes per stage
  const int kb_per_split = (p.kblocks_total + p.splits - 1) / p.splits;
  const int kb0 = (int)rank * kb_per_split;
  const int kb1 = kb0 + kb_per_split < p.kblocks_total ? kb0 + kb_per_split : p.kblocks_total;

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&p.tmDy); tma_prefetch_desc(&p.tmX); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // empty: one arrive per consumer warp
    mbar_init(ready_bar, p.splits > 1 ? p.splits - 1 : 1);
    mbar_init(free_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();                               // every rank's barriers are initialised before any remote arrive

  // tile -> (tap, ci tile, co tile); co fastest so that concurrently running clusters share X tiles in L2
  auto decode = [&](int t, int& co_t, int& ci_t, int& tap) {
    co_t = t % p.co_tiles; t /= p.co_tiles;
    ci_t = t % p.ci_tiles; t /= p.ci_tiles;
    tap = t;
  };

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = cid; t < tiles; t += ncl) {
        int co_t, ci_t, tap; decode(t, co_t, ci_t, tap);
        const bool two_dy = co_t * 128 + 64 < p.cout;
        const uint32_t tx = (uint32_t)((two_dy ? 2 : 1) + nb) * kBox;
        for (int kb = kb0; kb < kb1; kb++) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* s = smem + (size_t)stage * p.stage_bytes;
          mbar_expect_tx(&full_bar[stage], tx);
          const int row = kb * 64;
          tma_load_2d(s, &p.tmDy, &full_bar[stage], co_t * 128, row);
          if (two_dy) tma_load_2d(s + kBox, &p.tmDy, &full_bar[stage], co_t * 128 + 64, row);
          for (int j = 0; j < nb; j++)
            tma_load_2d(s + (p.xbox0 + j) * kBox, &p.tmX, &full_bar[stage], ci_t * BN + j * 64, row + p.shifts[tap]);
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // consumer warpgroup: wgmma into registers, then the cluster reduction and the dW update (thread et = output channel co_t * 128 + et)
    const int et = threadIdx.x - 128;
    int stage = 0; uint32_t phase = 0;
    uint32_t xphase = 0;                            // phase of ready_bar (rank 0) / free_bar (other ranks)
    float acc[2][BN / 2];
    for (int t = cid; t < tiles; t += ncl) {
      int co_t, ci_t, tap; decode(t, co_t, ci_t, tap);
      if (kb1 <= kb0) {                              // empty K range (tiny layers): this rank contributes zeros
#pragma unroll
        for (int i = 0; i < BN / 2; i++) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
      }
      int prev = -1;
      for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t s = smem_u32(smem + (size_t)stage * p.stage_bytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) {   // 16 K rows per MMA = 2 swizzle groups of 8 rows = 2048 B
          const uint64_t db = gmma_desc_sw128(s + p.xbox0 * kBox + k * 2048, kBox, 1024);
          const int sd = (kb > kb0 || k > 0) ? 1 : 0;
          wgmma_f32<BN, 1, 1, BF>(acc[0], gmma_desc_sw128(s + k * 2048, kBox, 1024), db, sd);
          if constexpr (TWO) wgmma_f32<BN, 1, 1, BF>(acc[1], gmma_desc_sw128(s + kBox + k * 2048, kBox, 1024), db, sd);
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous k-block's MMAs are done: release its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      const int co = co_t * 128 + et;
      float* drow = p.dw + ((long long)co * p.taps + tap) * p.dw_ld;
#pragma unroll
      for (int ch = 0; ch < BN / 32; ch++) {
        if (rank != 0) {
          // stage this rank's chunk, publish it to rank 0 and wait until rank 0 has read it (the buffer is reused next chunk)
          acc_stage_32<BN>(acc, ch, stg, et);
          fence_cluster();
          epi_bar();
          if (et == 0) mbar_arrive_remote(ready_bar, 0);
          mbar_wait_cluster(free_bar, xphase); xphase ^= 1;
          continue;
        }
        float v[32];
        acc_rows_32<BN>(acc, ch, stg, et, v);
        if (p.splits > 1) {
          mbar_wait_cluster(ready_bar, xphase); xphase ^= 1;
          for (int r = 1; r < p.splits; r++) {        // fixed order: rank 0 + rank 1 + ... (the same bits on every run)
#pragma unroll
            for (int j = 0; j < 32; j++) v[j] += ld_remote_f32(stg + et * 33 + j, (uint32_t)r);
          }
          epi_bar();                                   // every row has been read from every rank
          if (et == 0) for (int r = 1; r < p.splits; r++) mbar_arrive_remote(free_bar, (uint32_t)r);
        }
        const int c0 = ci_t * BN + ch * 32;
        if (co < p.cout) {
#pragma unroll
          for (int j = 0; j < 32; j++)
            if (c0 + j < p.cin_store) drow[c0 + j] += v[j] * p.scale;
        }
      }
    }
  }
}

static int g_num_sms_w = 0;

int wgrad_gemm_tc(const void* dy, long long dy_rows, int dy_ld, int cout, int dy_fmt,
                  const void* x, long long x_rows, int x_ld, int cin, int x_fmt,
                  int N, int H, int W, int taps, float* dw, int dw_ld, int cin_store, float scale, cudaStream_t stream) {
  if (!dy || !x || !dw || (taps != 1 && taps != 9)) return fail_msg(SSP_ERR_ARG, "wgrad_gemm_tc: bad argument");
  if ((dy_ld % 8) || (x_ld % 8)) return fail_msg(SSP_ERR_ARG, "wgrad_gemm_tc: leading dimensions must be multiples of 8");
  if (dy_fmt != x_fmt) return fail_msg(SSP_ERR_ARG, "wgrad_gemm_tc: both operands must have the same 16-bit format");
  if (!g_num_sms_w) {
    g_num_sms_w = ssp_sm_count();
  }
  WgradTcParams p;
  Geom g{N, H, W};
  // N tile over input channels: 64 (narrow layers; TMA zero-fills channels past cin) or 128 -- the 128 x BN accumulator is BN
  // registers per thread of the consumer warpgroup
  const int bn = cin <= 64 ? 64 : 128;
  p.bn = bn;
  p.m_rows = g.m_rows();
  p.kblocks_total = (int)((p.m_rows + 63) / 64);
  p.co_tiles = (cout + 127) / 128;
  p.ci_tiles = (cin + bn - 1) / bn;
  p.taps = taps;
  for (int t = 0; t < 9; t++) p.shifts[t] = (taps == 9) ? ((t / 3) - 1) * g.Wp() + ((t % 3) - 1) : 0;
  p.cout = cout; p.cin = cin;
  const int tiles = p.co_tiles * p.ci_tiles * taps;
  // K split = cluster size: doubled (up to 8, the portable cluster size) while the chip is not yet covered and every split keeps
  // at least 32 k-blocks (2048 pixel rows)
  int splits = 1;
  while (splits < 8 && tiles * splits < g_num_sms_w && p.kblocks_total / (2 * splits) >= 32) splits *= 2;
  p.splits = splits;
  p.fmt = dy_fmt;
  p.xbox0 = cout > 64 ? 2 : 1;
  p.stage_bytes = (p.xbox0 + bn / 64) * kBox;
  const int fixed = kStageRowsBytes + (2 * kMaxStagesW + 2) * 8 + 1024;
  int stages = (227 * 1024 - fixed) / p.stage_bytes;
  if (stages > kMaxStagesW) stages = kMaxStagesW;
  p.stages = stages;
  p.dw = dw; p.dw_ld = dw_ld; p.cin_store = cin_store; p.scale = scale;
  int rc = 0;
  rc |= tmap_2d_16bit(&p.tmDy, dy, (uint64_t)cout, (uint64_t)dy_rows, (uint64_t)dy_ld, 64, 64, dy_fmt == FMT_BF16);
  rc |= tmap_2d_16bit(&p.tmX, x, (uint64_t)cin, (uint64_t)x_rows, (uint64_t)x_ld, 64, 64, x_fmt == FMT_BF16);
  if (rc) return fail_msg(SSP_ERR_DRIVER, "wgrad_gemm_tc: cuTensorMapEncodeTiled failed");
  static int configured = 0;
  if (!configured) {
    cudaError_t e = cudaSuccess;
    for (auto k : {wgrad_tc_kernel<64, 0, false>, wgrad_tc_kernel<128, 0, false>, wgrad_tc_kernel<64, 1, false>, wgrad_tc_kernel<128, 1, false>,
                   wgrad_tc_kernel<64, 0, true>, wgrad_tc_kernel<128, 0, true>, wgrad_tc_kernel<64, 1, true>, wgrad_tc_kernel<128, 1, true>})
      if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  int clusters = g_num_sms_w / splits;
  if (clusters > tiles) clusters = tiles;
  if (clusters < 1) clusters = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(clusters * splits)); cfg.blockDim = dim3(kThreadsW);
  cfg.dynamicSmemBytes = (size_t)stages * p.stage_bytes + fixed; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)splits; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  const bool bf = dy_fmt == FMT_BF16;
  auto kern = cout > 64
      ? (bn == 64 ? (bf ? wgrad_tc_kernel<64, 1, true> : wgrad_tc_kernel<64, 0, true>) : (bf ? wgrad_tc_kernel<128, 1, true> : wgrad_tc_kernel<128, 0, true>))
      : (bn == 64 ? (bf ? wgrad_tc_kernel<64, 1, false> : wgrad_tc_kernel<64, 0, false>) : (bf ? wgrad_tc_kernel<128, 1, false> : wgrad_tc_kernel<128, 0, false>));
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, p);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

}  // namespace ssp
