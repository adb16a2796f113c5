// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, fp32 accumulators in registers, TMA-fed).
//
//   out[m, n] = sum_{tap} sum_{c} A[m + shift(tap), c] * B[n, tap*cin + c]
//
// A  = activation matrix in the padded-flat NHWC layout (ssp_common.cuh), 16-bit, optionally as a hi/lo
//      pair (x = hi + lo) so that three MMAs  Ahi*Bhi + Alo*Bhi + Ahi*Blo  reproduce an fp32 product to
//      ~2^-22: the yolo-pose stack amplifies operand rounding ~50x, a single fp16/tf32 pass misses the
//      reference's logits by 3e-2 (DESIGN.md, "numerics").
// B  = weights [cout][taps*cin] (K contiguous), same hi/lo convention.
// Every tap is one plain 2-D TMA tile at a shifted row coordinate (negative / past-the-end rows are
// zero-filled by TMA), so 3x3 convs need no im2col buffer; 1x1 convs are the taps==1 case.  Replaces nn.Conv2d in reference darknet.py:156-160 (forward) and, with re-packed
// weights, its data gradient (train.py:103 autograd).
//
// CTA = 8 warps, persistent over (m-tile, n-tile) pairs:
//   warp 0   TMA producer (one lane)       smem ring of `stages` x {A_hi, A_lo, B_hi, B_lo}
//   warps 4-7 one consumer warpgroup       wgmma 2 x (64 x BN x 16) per K step into registers, then the epilogue:
//                                          accumulators -> shared memory -> one row per thread -> (bias | BN statistics |
//                                          fp16 data gradient) -> global
#include "ssp_common.cuh"
#include "gemm.cuh"
#include "tmap.cuh"

namespace ssp {

struct ConvTcParams {
  CUtensorMap tmA[2];
  CUtensorMap tmB[2];
  long long m_rows;       // rows of the output matrix that exist (N*(H+1)*(W+1))
  long long store_rows;   // rows that may be written (allocation bound)
  int m_tiles, n_tiles;
  int kc_per_tap, cin, taps;
  int shifts[9];
  int Wp, HpWp;
  int cout, bn, n_terms;
  int fmt;                // FMT_F16 | FMT_BF16, both operands
  int stages, stage_bytes, b_bytes;
  float* out;
  long long out_ld;
  const float* bias;
  double* stat_sum;
  double* stat_sq;
  int epi;
  FusedAct fa;            // EPI_BNACT only
  int splits;             // SPLIT only: K slices per output tile; slice s writes its raw accumulators to out + s * slab_elems
  long long slab_elems;
};

static constexpr int kABytes = 128 * 128;     // 128 rows x 64 x 2 B
static constexpr int kMaxStages = 8;
static constexpr int kAccCols = 1024;         // per-CTA statistics accumulators (channels)
static constexpr int kThreads = 256;
// split-K rule (ssp_conv_splitk_count): S = min(SMs / tiles, k-blocks / kSplitMinKblocks), 1 when that is below 2.  A slice
// shorter than this spends more of its time filling the TMA pipeline and storing its partial tile than in MMAs.
static constexpr int kSplitMinKblocks = 8;

// FUSED: the inference epilogue (EPI_BNACT) -- a separate instantiation keeps the training kernel's code unchanged.  BN = N tile (wgmma N),
// BF = operand format (1 = bf16), NT = products per K step (3: split hi/lo operands, 1: single term).  All compile-time, so that
// every wgmma of a k-block sits in straight-line code.
// SPLIT: split-K inference instantiation (ssp_conv_gemm_splitk) -- the persistent loop walks (tile, split) work items, split s
// covers k-blocks [s*kb/S, (s+1)*kb/S) of the taps x kc_per_tap sequence and stores its fp32 accumulator tile unmodified
// into slab s of the caller's workspace (plain stores, no atomics); ssp_bn_apply_splitk sums the slabs in a fixed order.
template <bool FUSED, int BN, int BF, int NT, bool SPLIT = false>
__global__ void __launch_bounds__(kThreads, 1) conv_tc_kernel(const __grid_constant__ ConvTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem base is only guaranteed 16-B aligned: round up to 1024 (swizzle-128B atoms)
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* stage_base = smem;
  double* acc_sum = (double*)(smem + (size_t)p.stages * p.stage_bytes);
  double* acc_sq = acc_sum + kAccCols;
  float* stg = (float*)(acc_sq + kAccCols);
  uint64_t* full_bar = (uint64_t*)((uint8_t*)stg + kStageRowsBytes);
  uint64_t* empty_bar = full_bar + kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.m_tiles * p.n_tiles;
  const int kblocks = p.taps * p.kc_per_tap;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmA[0]);
    tma_prefetch_desc(&p.tmB[0]);
    if (p.n_terms == 3) { tma_prefetch_desc(&p.tmA[1]); tma_prefetch_desc(&p.tmB[1]); }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // empty: one arrive per consumer warp
    fence_barrier_init();
  }
  if (p.epi == EPI_STATS)
    for (int i = threadIdx.x; i < 2 * kAccCols; i += kThreads) acc_sum[i] = 0.0;
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = (uint32_t)(p.n_terms == 3 ? 2 : 1) * (uint32_t)(kABytes + p.b_bytes);
      if constexpr (SPLIT) {
        // (tile, split) work items; the k-block sequence is the one of the loop below, cut at s*kb/S
        for (int t = blockIdx.x; t < total_tiles * p.splits; t += gridDim.x) {
          const int tile = t / p.splits, sp = t % p.splits;
          const int m0 = (tile / p.n_tiles) * 128, n0 = (tile % p.n_tiles) * p.bn;
          const int kb1 = (int)((long long)(sp + 1) * kblocks / p.splits);
          for (int kb = (int)((long long)sp * kblocks / p.splits); kb < kb1; kb++) {
            const int tap = kb / p.kc_per_tap, kc = kb - tap * p.kc_per_tap;
            const int arow = m0 + p.shifts[tap];
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = stage_base + (size_t)stage * p.stage_bytes;
            mbar_expect_tx(&full_bar[stage], tx);
            const int kcol_b = tap * p.cin + kc * 64;
            tma_load_2d(sa, &p.tmA[0], &full_bar[stage], kc * 64, arow);
            if (p.n_terms == 3) {
              tma_load_2d(sa + kABytes, &p.tmA[1], &full_bar[stage], kc * 64, arow);
              tma_load_2d(sa + 2 * kABytes, &p.tmB[0], &full_bar[stage], kcol_b, n0);
              tma_load_2d(sa + 2 * kABytes + p.b_bytes, &p.tmB[1], &full_bar[stage], kcol_b, n0);
            } else {
              tma_load_2d(sa + kABytes, &p.tmB[0], &full_bar[stage], kcol_b, n0);
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      } else {
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int mt = t / p.n_tiles, nt = t % p.n_tiles;
        const int m0 = mt * 128, n0 = nt * p.bn;
        for (int tap = 0; tap < p.taps; tap++) {
          const int arow = m0 + p.shifts[tap];
          for (int kc = 0; kc < p.kc_per_tap; kc++) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = stage_base + (size_t)stage * p.stage_bytes;
            mbar_expect_tx(&full_bar[stage], tx);
            const int kcol_b = tap * p.cin + kc * 64;
            tma_load_2d(sa, &p.tmA[0], &full_bar[stage], kc * 64, arow);
            if (p.n_terms == 3) {
              tma_load_2d(sa + kABytes, &p.tmA[1], &full_bar[stage], kc * 64, arow);
              tma_load_2d(sa + 2 * kABytes, &p.tmB[0], &full_bar[stage], kcol_b, n0);
              tma_load_2d(sa + 2 * kABytes + p.b_bytes, &p.tmB[1], &full_bar[stage], kcol_b, n0);
            } else {
              tma_load_2d(sa + kABytes, &p.tmB[0], &full_bar[stage], kcol_b, n0);
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumer warpgroup: MMA, then epilogue (thread et = tile row et)
    const int et = threadIdx.x - 128;
    int stage = 0; uint32_t phase = 0;
    float acc[2][BN / 2];
    const int items = SPLIT ? total_tiles * p.splits : total_tiles;
    for (int t = blockIdx.x; t < items; t += gridDim.x) {
      int tile = t, sp = 0, kb0 = 0, kb1 = kblocks;
      if constexpr (SPLIT) {
        tile = t / p.splits; sp = t % p.splits;
        kb0 = (int)((long long)sp * kblocks / p.splits); kb1 = (int)((long long)(sp + 1) * kblocks / p.splits);
      }
      const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
      int prev = -1;
      for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(stage_base + (size_t)stage * p.stage_bytes);
        const uint32_t a_hi = sa, a_lo = sa + kABytes;
        const uint32_t b_hi = (NT == 3) ? sa + 2 * kABytes : sa + kABytes;
        const uint32_t b_lo = b_hi + p.b_bytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) {     // 4 x K(16) = 64 K elements; +32 B inside the swizzle atom
          const uint64_t dbh = gmma_desc_k_sw128(b_hi + k * 32);
#pragma unroll
          for (int h = 0; h < 2; h++) {   // rows h * 64 .. h * 64 + 63 of the tile
            const uint64_t dah = gmma_desc_k_sw128(a_hi + h * 8192 + k * 32);
            const int sd = (kb > kb0 || k > 0) ? 1 : 0;
            if constexpr (NT == 3) {
              wgmma_f32<BN, 0, 0, BF>(acc[h], gmma_desc_k_sw128(a_lo + h * 8192 + k * 32), dbh, sd);   // small cross terms first
              wgmma_f32<BN, 0, 0, BF>(acc[h], dah, gmma_desc_k_sw128(b_lo + k * 32), 1);
              wgmma_f32<BN, 0, 0, BF>(acc[h], dah, dbh, 1);
            } else {
              wgmma_f32<BN, 0, 0, BF>(acc[h], dah, dbh, sd);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous k-block's MMAs are done: release its slot
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      const long long m = (long long)mt * 128 + et;
      const int n0 = nt * p.bn;
      bool valid = false;
      if (m < p.m_rows) {
        const int rem = (int)(m % p.HpWp);
        valid = (rem / p.Wp >= 1) && (rem % p.Wp >= 1);
      }
      float* orow = (p.out && p.epi != EPI_F16) ? p.out + m * p.out_ld : nullptr;
      const bool can_store = m < p.store_rows;
#pragma unroll
      for (int ch = 0; ch < BN / 32; ch++) {
        float v[32];
        acc_rows_32<BN>(acc, ch, stg, et, v);
        const int c0 = n0 + ch * 32;
        if constexpr (SPLIT) {
          // raw partial sums of this K slice; the reduction reads valid rows only
          if (can_store) {
            float* o = p.out + sp * p.slab_elems + m * p.out_ld;
            if (c0 + 32 <= p.cout) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(o + c0 + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++) if (c0 + j < p.cout) o[c0 + j] = v[j];
            }
          }
          continue;
        }
        if constexpr (FUSED) {
          // folded BatchNorm (running statistics) + LeakyReLU in the epilogue; only valid rows are written so that the
          // consumer's pad rows stay zero; the fp32 Y tensor is never materialised in this mode
          if (valid && c0 + 32 <= p.cout) {
            uint32_t ph[16], pl[16];
#pragma unroll
            for (int j = 0; j < 32; j += 2) {
              float z0 = fmaf(v[j], __ldg(p.fa.scale + c0 + j), __ldg(p.fa.shift + c0 + j));
              float z1 = fmaf(v[j + 1], __ldg(p.fa.scale + c0 + j + 1), __ldg(p.fa.shift + c0 + j + 1));
              z0 = z0 > 0.f ? z0 : z0 * p.fa.slope; z1 = z1 > 0.f ? z1 : z1 * p.fa.slope;
              split_f16x2(z0, z1, ph[j >> 1], pl[j >> 1]);
            }
            uint4* dh = reinterpret_cast<uint4*>(p.fa.d_hi + m * p.fa.d_ld + p.fa.d_c0 + c0);
            uint4* dl = reinterpret_cast<uint4*>(p.fa.d_lo + m * p.fa.d_ld + p.fa.d_c0 + c0);
#pragma unroll
            for (int j = 0; j < 4; j++) {
              dh[j] = make_uint4(ph[4 * j], ph[4 * j + 1], ph[4 * j + 2], ph[4 * j + 3]);
              dl[j] = make_uint4(pl[4 * j], pl[4 * j + 1], pl[4 * j + 2], pl[4 * j + 3]);
            }
          }
          continue;
        }
        if (p.epi == EPI_BIAS) {
#pragma unroll
          for (int j = 0; j < 32; j++) if (c0 + j < p.cout) v[j] += __ldg(p.bias + c0 + j);
        }
        if (p.epi == EPI_F16) {                     // data gradient kept in fp16 (the BN backward reads it twice): 64 B per row chunk
          if (can_store) {
            uint16_t* o16 = reinterpret_cast<uint16_t*>(p.out) + m * p.out_ld + c0;
            if (c0 + 32 <= p.cout) {
              uint32_t pk[16];
#pragma unroll
              for (int j = 0; j < 16; j++) pk[j] = cvt_f32_to_16(v[2 * j], FMT_F16) | ((uint32_t)cvt_f32_to_16(v[2 * j + 1], FMT_F16) << 16);
#pragma unroll
              for (int j = 0; j < 4; j++) reinterpret_cast<uint4*>(o16)[j] = make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++) if (c0 + j < p.cout) o16[j] = cvt_f32_to_16(v[j], FMT_F16);
            }
          }
        } else if (can_store && p.epi != 3) {     // epi 3: diagnostic mode without the global store
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
          if (c0 + lane < p.cout) {
            atomicAdd(&acc_sum[c0 + lane], (double)cs);
            atomicAdd(&acc_sq[c0 + lane], (double)cq);
          }
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

template <bool FUSED, int BF, int NT, bool SPLIT = false>
static int launch_conv_tc(const ConvTcParams& p, int grid, int smem_bytes, cudaStream_t stream) {
  static int configured = 0;
  if (!configured) {
    cudaError_t e = cudaSuccess;
    for (auto k : {conv_tc_kernel<FUSED, 32, BF, NT, SPLIT>, conv_tc_kernel<FUSED, 64, BF, NT, SPLIT>, conv_tc_kernel<FUSED, 128, BF, NT, SPLIT>})
      if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  if (p.bn == 32) conv_tc_kernel<FUSED, 32, BF, NT, SPLIT><<<grid, kThreads, smem_bytes, stream>>>(p);
  else if (p.bn == 64) conv_tc_kernel<FUSED, 64, BF, NT, SPLIT><<<grid, kThreads, smem_bytes, stream>>>(p);
  else conv_tc_kernel<FUSED, 128, BF, NT, SPLIT><<<grid, kThreads, smem_bytes, stream>>>(p);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

static int g_num_sms = 0;

// output tiles of the per-tap kernel and the k-blocks each of them walks (the N tile rule of conv_gemm_tc)
static void tile_geometry(int N, int H, int W, int taps, int cin, int cout, long long* tiles, int* kblocks) {
  const int bn = cout > 64 ? 128 : ((cout + 31) / 32) * 32;
  *tiles = ((Geom{N, H, W}.m_rows() + 127) / 128) * (long long)((cout + bn - 1) / bn);
  *kblocks = taps * ((cin + 63) / 64);
}

int conv_gemm_tc(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin,
                 const void* b_hi, const void* b_lo, int b_rows, int b_ld, int a_fmt, int b_fmt,
                 int N, int H, int W, int taps, int cout, float* out, int out_ld, long long out_rows,
                 int epi, const float* bias, double* stat_sum, double* stat_sq, cudaStream_t stream, const FusedAct* fa,
                 const SplitK* sk) {
  if (sk) {
    long long tiles; int kblocks;
    tile_geometry(N, H, W, taps, cin, cout, &tiles, &kblocks);
    if (fa || epi != EPI_F32) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: split-K stores plain fp32 partial sums");
    if (sk->splits < 1 || (cin > 0 && (taps == 1 || taps == 9) && sk->splits > kblocks))
      return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm_splitk: splits must be in [1, k-blocks] (taps * ceil(cin / 64))");
    if (!out || ((uintptr_t)out % 16) || (out_ld % 4) || out_ld < cout || (sk->slab_elems % 4))
      return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm_splitk: workspace must be non-null and 16-B aligned, partial_ld % 4 == 0 and >= cout, slab_elems % 4 == 0");
    if (sk->slab_elems < flat_alloc_rows(N, H, W) * (long long)out_ld)
      return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm_splitk: a slab must hold ssp_flat_alloc_rows(N, H, W) * partial_ld elements");
    out_rows = flat_alloc_rows(N, H, W);
  }
  if (fa) {
    if (!fa->scale || !fa->shift || !fa->d_hi || !fa->d_lo || (cout % 32) || (fa->d_ld % 8) || (fa->d_c0 % 8) || fa->d_c0 < 0 ||
        ((uintptr_t)fa->d_hi % 16) || ((uintptr_t)fa->d_lo % 16) || fa->d_ld < fa->d_c0 + cout)
      return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: fused BN+activation epilogue needs cout % 32 == 0, 16-B aligned destination planes and "
                                   "rows (d_ld % 8 == 0, d_c0 % 8 == 0) and d_ld >= d_c0 + cout");
    epi = EPI_BNACT;
  }
  if (!a_hi || !b_hi || (!out && !fa) || (taps != 1 && taps != 9) || cin <= 0 || cout <= 0) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: bad argument");
  if ((a_ld % 8) || (b_ld % 8)) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: leading dimensions must be multiples of 8 elements (16 B)");
  if (epi == EPI_STATS && (cout > kAccCols || !stat_sum || !stat_sq)) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: statistics need cout <= 1024 and buffers");
  if (epi == EPI_BIAS && !bias) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: bias missing");
  if (!fa && epi != EPI_F16 && ((out_ld % 4) || ((uintptr_t)out % 16))) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: output must be 16-B aligned with ld % 4 == 0");
  if (epi == EPI_F16 && ((out_ld % 8) || ((uintptr_t)out % 16))) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: fp16 output must be 16-B aligned with ld % 8 == 0");
  if (a_fmt != b_fmt) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: both operands must have the same 16-bit format");
  if (!g_num_sms) {
    g_num_sms = ssp_sm_count();
  }
  ConvTcParams p;
  Geom g{N, H, W};
  p.n_terms = (a_lo && b_lo) ? 3 : 1;
  // N tile: 32, 64 or 128 channels.  The 128 x BN fp32 accumulator lives in the registers of one warpgroup (BN per thread), so
  // 128 is the widest tile that leaves registers for the epilogue.
  int bn = ((cout + 31) / 32) * 32;
  if (bn > 64) bn = 128;
  p.bn = bn;
  p.b_bytes = bn * 128;
  p.m_rows = g.m_rows();
  p.store_rows = out_rows;
  p.m_tiles = (int)((p.m_rows + 127) / 128);
  p.n_tiles = (cout + bn - 1) / bn;
  p.kc_per_tap = (cin + 63) / 64;
  p.cin = cin;
  p.taps = taps;
  for (int t = 0; t < 9; t++) p.shifts[t] = (taps == 9) ? ((t / 3) - 1) * g.Wp() + ((t % 3) - 1) : 0;
  p.Wp = g.Wp(); p.HpWp = g.HpWp();
  p.cout = cout;
  p.fmt = a_fmt;
  p.stage_bytes = (p.n_terms == 3 ? 2 : 1) * (kABytes + p.b_bytes);
  const int fixed = 2 * kAccCols * 8 + kStageRowsBytes + 2 * kMaxStages * 8 + 1024;
  int stages = (227 * 1024 - fixed) / p.stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: tile does not fit shared memory");
  p.stages = stages;
  p.out = out; p.out_ld = out_ld; p.bias = bias; p.stat_sum = stat_sum; p.stat_sq = stat_sq; p.epi = epi;
  if (fa) p.fa = *fa; else p.fa = FusedAct{nullptr, nullptr, 1.f, nullptr, nullptr, 0, 0};
  p.splits = sk ? sk->splits : 1;
  p.slab_elems = sk ? sk->slab_elems : 0;
  int rc = 0;
  rc |= tmap_2d_16bit(&p.tmA[0], a_hi, (uint64_t)cin, (uint64_t)a_rows, (uint64_t)a_ld, 64, 128, a_fmt == FMT_BF16);
  rc |= tmap_2d_16bit(&p.tmB[0], b_hi, (uint64_t)taps * cin, (uint64_t)b_rows, (uint64_t)b_ld, 64, bn, b_fmt == FMT_BF16);
  if (p.n_terms == 3) {
    rc |= tmap_2d_16bit(&p.tmA[1], a_lo, (uint64_t)cin, (uint64_t)a_rows, (uint64_t)a_ld, 64, 128, a_fmt == FMT_BF16);
    rc |= tmap_2d_16bit(&p.tmB[1], b_lo, (uint64_t)taps * cin, (uint64_t)b_rows, (uint64_t)b_ld, 64, bn, b_fmt == FMT_BF16);
  }
  if (rc) return fail_msg(SSP_ERR_DRIVER, "conv_gemm_tc: cuTensorMapEncodeTiled failed (no driver, or misaligned operand)");
  const int smem_bytes = stages * p.stage_bytes + fixed;
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < g_num_sms ? total : g_num_sms;
  // split hi/lo operands are fp16 planes; the fused epilogue (ssp_conv_gemm_bnact) is fp16 only
  if (p.n_terms == 3 && p.fmt == FMT_BF16) return fail_msg(SSP_ERR_ARG, "conv_gemm_tc: split (hi/lo) operands must be fp16");
  if (sk) {
    const long long items = (long long)total * sk->splits;
    const int sgrid = items < g_num_sms ? (int)items : g_num_sms;
    return p.n_terms == 3 ? launch_conv_tc<false, 0, 3, true>(p, sgrid, smem_bytes, stream) : launch_conv_tc<false, 0, 1, true>(p, sgrid, smem_bytes, stream);
  }
  if (fa) return p.n_terms == 3 ? launch_conv_tc<true, 0, 3>(p, grid, smem_bytes, stream) : launch_conv_tc<true, 0, 1>(p, grid, smem_bytes, stream);
  if (p.n_terms == 3) return launch_conv_tc<false, 0, 3>(p, grid, smem_bytes, stream);
  return p.fmt == FMT_BF16 ? launch_conv_tc<false, 1, 1>(p, grid, smem_bytes, stream) : launch_conv_tc<false, 0, 1>(p, grid, smem_bytes, stream);
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_conv_gemm_bnact(int impl, const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo,
                        int b_rows, int b_ld, int N, int H, int W, int taps, int cout, const float* scale, const float* shift, float slope,
                        void* d_hi, void* d_lo, int d_ld, int d_c0, void* stream) {
  FusedAct fa{scale, shift, slope, (uint16_t*)d_hi, (uint16_t*)d_lo, d_ld, d_c0};
  if (impl == SSP_IMPL_TC || impl == SSP_IMPL_TC2 || impl == SSP_IMPL_BAND)
    return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, SSP_FMT_F16, SSP_FMT_F16, N, H, W, taps, cout, nullptr, 0, 0, EPI_BNACT,
                        nullptr, nullptr, nullptr, (cudaStream_t)stream, &fa, nullptr);
  return fail_msg(SSP_ERR_ARG, "ssp_conv_gemm_bnact: tensor-core implementations only");
}

int ssp_conv_gemm_splitk(const void* a_hi, const void* a_lo, long long a_rows, int a_ld, int cin, const void* b_hi, const void* b_lo, int b_rows,
                         int b_ld, int N, int H, int W, int taps, int cout, int splits, float* partial, long long slab_elems, int partial_ld,
                         void* stream) {
  const SplitK sk{splits, slab_elems};
  return conv_gemm_tc(a_hi, a_lo, a_rows, a_ld, cin, b_hi, b_lo, b_rows, b_ld, SSP_FMT_F16, SSP_FMT_F16, N, H, W, taps, cout, partial, partial_ld, 0,
                      EPI_F32, nullptr, nullptr, nullptr, (cudaStream_t)stream, nullptr, &sk);
}

int ssp_conv_splitk_count(int N, int H, int W, int taps, int cin, int cout, int num_sms) {
  if (N <= 0 || H <= 0 || W <= 0 || (taps != 1 && taps != 9) || cin <= 0 || cout <= 0 || num_sms <= 0)
    return fail_msg(SSP_ERR_ARG, "ssp_conv_splitk_count: bad argument");
  long long tiles; int kblocks;
  tile_geometry(N, H, W, taps, cin, cout, &tiles, &kblocks);
  long long s = num_sms / tiles;
  if (s > kblocks / kSplitMinKblocks) s = kblocks / kSplitMinKblocks;
  return s < 2 ? 1 : (int)s;
}
}  // extern "C"
