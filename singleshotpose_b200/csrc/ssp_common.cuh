// Shared device/host helpers for the sm_90a kernels of the singleshotpose hot path.
//
// Data layout ("padded-flat NHWC"): a feature map (N, C, H, W) is stored as a row-major matrix
// [rows, C] whose row index is
//     row(n, h, w) = n*(H+1)*(W+1) + (h+1)*(W+1) + (w+1)
// i.e. every image row is preceded by ONE zero pad pixel (which is also the right pad of the previous
// row) and every image by ONE zero pad row (also the bottom pad of the previous image).  A 3x3 / pad 1
// convolution then is, for every tap (kh, kw), the SAME matrix shifted by the constant row offset
// (kh-1)*(W+1) + (kw-1): each tap of the implicit GEMM is a plain 2-D TMA tile load, no im2col.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/ssp_b200.h"   // SSP_OK / SSP_ERR_* / SSP_* enums shared with the C ABI

#define SSP_CHECK_LAUNCH()                                   \
  do {                                                       \
    cudaError_t e__ = cudaGetLastError();                    \
    if (e__ != cudaSuccess) return ssp::fail_cuda(e__, __FILE__, __LINE__); \
  } while (0)

namespace ssp {

int fail_cuda(cudaError_t e, const char* file, int line);   // abi.cu: records message, returns SSP_ERR_CUDA
int fail_msg(int code, const char* msg);

// SMs the persistent kernels size their grids for.  SSP_SM_LIMIT=n (even, < the device's count) leaves SMs free, e.g. for NCCL's kernels in
// the data-parallel step: a collective cannot co-reside with a 227-KB GEMM CTA, it needs SMs of its own to overlap with the backward pass.
inline int ssp_sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    const char* e = getenv("SSP_SM_LIMIT");
    if (e) { const int l = atoi(e) & ~1; if (l >= 2 && l < n) n = l; }
  }
  return n;
}
enum Fmt16 { FMT_F16 = 0, FMT_BF16 = 1 };
// GEMM epilogues: plain fp32 store | store + per-channel sum / sum-of-squares over valid pixels | + bias
enum { EPI_F32 = 0, EPI_STATS = 1, EPI_BIAS = 2, EPI_BNACT = 4, EPI_F16 = 8 };
// inference-mode fusion: z = leaky(acc*scale[c] + shift[c]) written straight into the consumer's fp16 hi/lo operand planes
struct FusedAct {
  const float* scale; const float* shift; float slope;
  uint16_t* d_hi; uint16_t* d_lo; long long d_ld; int d_c0;
};
// inference split-K (ssp_conv_gemm_splitk): `splits` K slices per output tile, slice s stores into out + s * slab_elems
struct SplitK { int splits; long long slab_elems; };
struct Geom {
  int N, H, W;
  __host__ __device__ int Wp() const { return W + 1; }
  __host__ __device__ int HpWp() const { return (H + 1) * (W + 1); }
  __host__ __device__ long long m_rows() const { return (long long)N * (H + 1) * (W + 1); }
  __host__ __device__ long long row(int n, int h, int w) const {
    return (long long)n * HpWp() + (long long)(h + 1) * Wp() + (w + 1);
  }
};

__host__ __device__ inline long long flat_alloc_rows(int N, int H, int W) {
  long long m = (long long)N * (H + 1) * (W + 1) + (W + 1) + 2;
  return ((m + 127) / 128) * 128 + 128;
}

// ---------------------------------------------------------------------------------------------
// 16-bit conversions with runtime format
__device__ __forceinline__ float cvt16_to_f32(uint16_t v, int fmt) {
  return fmt == FMT_F16 ? __half2float(__ushort_as_half(v)) : __bfloat162float(__ushort_as_bfloat16(v));
}
// fp16(clamp(f, +-65504)), round to nearest even: a conversion that would overflow gives the largest finite fp16 instead of an
// infinity, NaN stays NaN (PTX cvt .satfinite: one instruction, like the plain conversion)
__device__ __forceinline__ uint16_t f16_satfinite(float f) {
  uint16_t h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(f));
  return h;
}
// the single-term 16-bit store of the backward's planes (loss-scaled gradients, dgrad weights): fp16 saturates like f16_satfinite
// instead of overflowing to inf, and a NaN stays NaN (a clamp through fmaxf would return its finite argument, -65504, for NaN)
__device__ __forceinline__ uint16_t cvt_f32_to_16(float f, int fmt) {
  return fmt == FMT_F16 ? f16_satfinite(f) : __bfloat16_as_ushort(__float2bfloat16_rn(f));
}
// split an fp32 value into fp16 hi + fp16 lo (hi + lo carries ~22 mantissa bits).  Saturating: hi = fp16(clamp(f, +-65504)) and
// lo = fp16(clamp(f - hi, +-65504)), so a finite f never yields an infinite part (an unclamped hi of +-inf for |f| >= 65520
// would make lo = -+inf and hi + lo NaN).  f is represented to ~2^-11 relative up to |f| = 131008 and saturates beyond; for
// |f| < 65520 both parts are the unclamped ones bit for bit.
__device__ __forceinline__ void split_f16(float f, uint16_t& hi, uint16_t& lo) {
  hi = f16_satfinite(f);
  lo = f16_satfinite(f - __half2float(__ushort_as_half(hi)));
}
// split_f16 of two values at once, packed (a in the low half): one paired conversion per plane, as the stores want them
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi2, uint32_t& lo2) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi2) : "f"(b), "f"(a));      // the first source goes to the upper half
  const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi2));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo2) : "f"(b - h.y), "f"(a - h.x));
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers (mbarrier, TMA, wgmma)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (cudaErrorLaunchFailure), never as a hang.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) { __trap(); }
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// named barrier of the 128 threads of the consumer warpgroup (warps 4-7)
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// Shared-memory matrix descriptor for wgmma, SWIZZLE_128B (sm_90 encoding: layout type 1 at bits 62-63, base offset 0).
//   K-major tile  [rows][64 x 16-bit] (one 128-byte swizzled line per row): LBO unused (16), SBO = 8 rows = 1024 B.
//   MN-major tile [k rows][64 x 16-bit]: LBO = byte distance between 64-element MN groups, SBO = 8 k-rows = 1024 B.
// The swizzle phase follows the absolute shared-memory address, so a start address 32 B (one K step) or 128 B (one row) into a
// 1024-B atom addresses the same bytes TMA wrote there.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) { return gmma_desc_sw128(smem_addr, 16, 1024); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N] from shared memory, fp32 accumulators in registers of the whole warpgroup (issued by all
// 128 threads).  TA / TB = 1: that operand is MN-major.  sd = 0 overwrites D.  Fragment of thread t (warp w = t / 32, lane l):
//   d[i] = D[w * 16 + l / 4 + 8 * ((i / 2) % 2)][(i / 4) * 8 + (l % 4) * 2 + i % 2]
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16_f16(float (&d)[16], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16_bf16(float (&d)[16], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t da, uint64_t db, int sd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(sd), "n"(TA), "n"(TB));
}

// BF16: both operands bf16 (else fp16).  A compile-time choice: a runtime format switch puts every wgmma in a divergent path,
// and ptxas then serialises them (warpgroup.arrive inserted around each one).
template <int N, int TA, int TB, int BF16>
__device__ __forceinline__ void wgmma_f32(float (&d)[N / 2], uint64_t da, uint64_t db, int sd) {
  if constexpr (N == 32) { if constexpr (BF16) wgmma_m64n32k16_bf16<TA, TB>(d, da, db, sd); else wgmma_m64n32k16_f16<TA, TB>(d, da, db, sd); }
  else if constexpr (N == 64) { if constexpr (BF16) wgmma_m64n64k16_bf16<TA, TB>(d, da, db, sd); else wgmma_m64n64k16_f16<TA, TB>(d, da, db, sd); }
  else { static_assert(N == 128, "N in {32, 64, 128}"); if constexpr (BF16) wgmma_m64n128k16_bf16<TA, TB>(d, da, db, sd); else wgmma_m64n128k16_f16<TA, TB>(d, da, db, sd); }
}

// The 128 x N accumulator of a warpgroup (two m64 halves: rows h * 64 + ...) seen as "thread t owns row t": columns
// [32 ch, 32 ch + 32) of every row go through `stg` (HALVES * 64 x 33 floats of shared memory) and thread t receives row t
// (HALVES = 1: only the first half, threads 64-127 receive nothing).  Every thread of the warpgroup must call it with the same ch.
static constexpr int kStageRowsBytes = 128 * 33 * 4;
template <int N, int HALVES = 2>
__device__ __forceinline__ void acc_stage_32(const float (&acc)[2][N / 2], int ch, float* stg, int t) {
  const int w = t >> 5, l = t & 31;
  epi_bar();                                  // the previous chunk has been read
#pragma unroll
  for (int c = 0; c < N / 32; c++) {
    if (c == ch) {
#pragma unroll
      for (int h = 0; h < HALVES; h++)
#pragma unroll
        for (int j = 0; j < 16; j++) {
          const int i = 16 * c + j;
          const int row = h * 64 + w * 16 + (l >> 2) + 8 * ((i >> 1) & 1);
          const int col = ((i >> 2) & 3) * 8 + (l & 3) * 2 + (i & 1);
          stg[row * 33 + col] = acc[h][i];
        }
    }
  }
  epi_bar();
}
template <int N, int HALVES = 2>
__device__ __forceinline__ void acc_rows_32(const float (&acc)[2][N / 2], int ch, float* stg, int t, float (&v)[32]) {
  acc_stage_32<N, HALVES>(acc, ch, stg, t);
  if (t < HALVES * 64) {
#pragma unroll
    for (int j = 0; j < 32; j++) v[j] = stg[t * 33 + j];
  }
}

// ---------------------------------------------------------------------------------------------
// thread-block clusters: rank, cluster-wide barrier, mbarrier arrive / shared-memory load in another CTA of the cluster
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void fence_cluster() { asm volatile("fence.acq_rel.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tmbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
               ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}
__device__ __forceinline__ float ld_remote_f32(const float* p, uint32_t rank) {
  float v;
  asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %1, %2;\n\tld.shared::cluster.f32 %0, [ra];\n\t}"
               : "=f"(v) : "r"(smem_u32(p)), "r"(rank) : "memory");
  return v;
}
// wait for a phase of a barrier that threads of OTHER CTAs of the cluster arrive on (acquire at cluster scope), bounded like mbar_wait
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (ok) return;
    if (++spins > (1u << 26)) { __trap(); }
  }
}

// optim.SGD(momentum, dampening = 0, weight_decay), train.py:388:  g += wd*p ; v = mu*v + g ; p -= lr*v  (torch's first step,
// v = g, is the same with v0 = 0).  Explicit FMAs: every kernel that applies the update produces the same bits.
__device__ __forceinline__ void sgd_update(float& p, float g, float& v, float lr, float mu, float wd, float gscale) {
  const float vn = fmaf(mu, v, fmaf(wd, p, g * gscale));
  v = vn;
  p = fmaf(-lr, vn, p);
}

// Sum over the 32 lanes of v[j], delivered to lane j (31 shuffles instead of 32*5).  One level per template instance, so every
// index is a compile-time constant and v stays in registers.
template <int OFF>
__device__ __forceinline__ void warp_transpose_level(float (&v)[32], int lane) {
  const bool up = (lane & OFF) != 0;
#pragma unroll
  for (int i = 0; i < OFF; i++) {
    const float send = up ? v[i] : v[i + OFF];
    const float keep = up ? v[i + OFF] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
  if constexpr (OFF > 1) warp_transpose_level<OFF / 2>(v, lane);
}
__device__ __forceinline__ float warp_transpose_sum32(float (&v)[32], int lane) {
  warp_transpose_level<16>(v, lane);
  return v[0];
}

}  // namespace ssp
