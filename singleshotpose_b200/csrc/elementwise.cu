// HBM-bound kernels of the conv stack: layout packing, BatchNorm (train statistics, apply + LeakyReLU fused
// with 2x2 max-pool / reorg / concat placement), BatchNorm+LeakyReLU+pool backward, weight re-packing, SGD.
// They replace nn.BatchNorm2d / nn.LeakyReLU / nn.MaxPool2d / Reorg / torch.cat of reference
// darknet.py:16-35,96-106,156-176 and their autograd, and optim.SGD of train.py:388.
// All activations live in the padded-flat NHWC layout (ssp_common.cuh); 4 channels per thread (16-B fp32 /
// 8-B fp16 vectors), consecutive threads on consecutive channels -> fully coalesced rows.
#include "ssp_common.cuh"

// Occupancy of the HBM-bound BN kernels: uncapped they use 97-118 registers -> 2 blocks/SM, 23 % warps active, 47-63 % of DRAM
// peak under ncu (round 1).  Capped at 85 registers for a third resident block (a few spilled bytes per thread): same-box A/B
// of the batch-64 step in round 2: 18.35 -> 17.92 ms (a fourth block, 64 registers, spills too much: 18.86 ms).
constexpr int kBnMinBlocks = 3;
#define SSP_BN_BOUNDS __launch_bounds__(256, kBnMinBlocks)

namespace ssp {

// ------------------------------------------------------------------------------------------------
// generic NCHW fp32 -> padded-flat rows (hi/lo fp16, or a single 16-bit plane in `fmt` when lo == nullptr)
__global__ void pack_nchw_kernel(const float* __restrict__ x, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                 int N, int C, int H, int W, int ld, int c0, int fmt, float scale) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * H * W * C;
  if (idx >= total) return;
  const int c = (int)(idx % C);
  long long pix = idx / C;
  const int w = (int)(pix % W); pix /= W;
  const int h = (int)(pix % H);
  const int n = (int)(pix / H);
  const float v = __ldg(x + (((long long)n * C + c) * H + h) * W + w) * scale;
  Geom g{N, H, W};
  const long long o = g.row(n, h, w) * ld + c0 + c;
  if (lo) { uint16_t a, b; split_f16(v, a, b); hi[o] = a; lo[o] = b; }
  else hi[o] = cvt_f32_to_16(v, fmt);
}

// padded-flat fp32 rows -> NCHW fp32 (network output / tests)
__global__ void unpack_nchw_kernel(const float* __restrict__ y, float* __restrict__ out, int N, int C, int H, int W, int ld, int c0) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * C * H * W;
  if (idx >= total) return;
  const int w = (int)(idx % W);
  long long r = idx / W;
  const int h = (int)(r % H); r /= H;
  const int c = (int)(r % C);
  const int n = (int)(r / C);
  Geom g{N, H, W};
  out[idx] = y[g.row(n, h, w) * ld + c0 + c];
}

// padded-flat 16-bit plane(s) -> NCHW fp32 (tests: read activations back)
__global__ void unpack16_nchw_kernel(const uint16_t* __restrict__ hi, const uint16_t* __restrict__ lo, float* __restrict__ out,
                                     int N, int C, int H, int W, int ld, int c0, int fmt) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * C * H * W;
  if (idx >= total) return;
  const int w = (int)(idx % W);
  long long r = idx / W;
  const int h = (int)(r % H); r /= H;
  const int c = (int)(r % C);
  const int n = (int)(r / C);
  Geom g{N, H, W};
  const long long o = g.row(n, h, w) * ld + c0 + c;
  float v = cvt16_to_f32(hi[o], fmt);
  if (lo) v += cvt16_to_f32(lo[o], fmt);
  out[idx] = v;
}

// ------------------------------------------------------------------------------------------------
// BatchNorm statistics -> per-channel affine.  train: batch statistics from the conv epilogue's fp64 sums
// (biased variance for normalisation, unbiased for running_var, momentum, eps as nn.BatchNorm2d(eps=1e-4),
// darknet.py:157); eval: running statistics.  Zeroes the sum buffers for the next step.
__global__ void bn_finalize_kernel(double* __restrict__ ssum, double* __restrict__ ssq, double count,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float momentum, float eps, int train,
                                   float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                   float* __restrict__ scale_out, float* __restrict__ shift_out, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mean, invstd;
  if (train) {
    const double m = ssum[c] / count;
    double var = ssq[c] / count - m * m;
    if (var < 0.0) var = 0.0;
    mean = (float)m;
    invstd = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean) {
      const double unb = count > 1.0 ? var * count / (count - 1.0) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    }
    ssum[c] = 0.0; ssq[c] = 0.0;
  } else {
    mean = running_mean[c];
    invstd = 1.f / sqrtf(running_var[c] + eps);
  }
  const float sc = gamma[c] * invstd;
  mean_out[c] = mean; invstd_out[c] = invstd;
  scale_out[c] = sc; shift_out[c] = beta[c] - mean * sc;
}

// ------------------------------------------------------------------------------------------------
// z = leaky(y*scale + shift) written to up to two destinations.
enum { DST_NONE = 0, DST_DIRECT = 1, DST_POOL = 2, DST_REORG = 3 };
struct ActDst {
  uint16_t* hi; uint16_t* lo;   // lo may be null (single plane in fmt)
  int ld, c0, kind;
};
struct BnApplyParams {
  const float* y; int y_ld;
  const float* scale; const float* shift;
  int N, C, H, W;
  float slope;          // 0.1 leaky, 1.0 linear
  ActDst dst[2];
  float* ypool; int ypool_ld;   // POOLED only, optional: conv output y at the arg-max position of every 2x2 window (fp32, pooled geometry)
  int splits; long long slab;   // SPLIT only: y = sum of the slabs y + s * slab, s = 0 .. splits-1 in this order
};

__device__ __forceinline__ float leaky(float v, float slope) { return v > 0.f ? v : v * slope; }

__device__ __forceinline__ void store4(const ActDst& d, long long row, int c, const float (&z)[4]) {
  const long long o = row * d.ld + d.c0 + c;
  uint32_t h01, l01, h23, l23;
  split_f16x2(z[0], z[1], h01, l01);
  split_f16x2(z[2], z[3], h23, l23);
  *reinterpret_cast<uint2*>(d.hi + o) = make_uint2(h01, h23);
  if (d.lo) *reinterpret_cast<uint2*>(d.lo + o) = make_uint2(l01, l23);
}

// Thread layout shared by the BN kernels: channel group cgi = tid % CG (4 channels each, consecutive threads on
// consecutive channels => 16-B vectors of one pixel row are contiguous), pixel lane pl = tid / CG.  A block owns a
// contiguous range of "units" (pixels, or 2x2 windows when a pooled route is involved) and every thread walks it with
// stride PL, so the per-channel constants are loaded once per thread and several independent loads are in flight.
struct UnitWalk {
  int c, pl, PL; long long begin, end; bool active;
  __device__ UnitWalk(int C, long long nunits, int per_thread) {
    const int cgs = C >> 2;
    const int CG = cgs < 256 ? cgs : 256;
    PL = 256 / CG;
    const int cblocks = (cgs + CG - 1) / CG;
    const int cb = blockIdx.x % cblocks;
    const long long pb = blockIdx.x / cblocks;
    const int cgi = threadIdx.x % CG;
    pl = threadIdx.x / CG;
    c = (cb * CG + cgi) * 4;
    const long long per = (long long)PL * per_thread;
    begin = pb * per; end = begin + per; if (end > nunits) end = nunits;
    active = c < C && pl < PL;
  }
};
static inline unsigned unit_grid(int C, long long nunits, int per_thread) {
  const int cgs = C / 4, CG = cgs < 256 ? cgs : 256, PL = 256 / CG;
  const int cblocks = (cgs + CG - 1) / CG;
  const long long per = (long long)PL * per_thread;
  return (unsigned)(((nunits + per - 1) / per) * cblocks);
}
constexpr int kBnUnitsPerThread = 8;          // BN units (channel quad x pixel or 2x2 window) per thread, chosen by a measured sweep

// POOLED = true : unit = one 2x2 window (needed when any destination is DST_POOL)
// SPLIT = true  : y is the sum of the split-K partial slabs of ssp_conv_gemm_splitk (inference, no arg-max plane)
template <bool POOLED, bool SPLIT = false>
__global__ void SSP_BN_BOUNDS bn_apply_kernel(const BnApplyParams p) {
  const int Hs = POOLED ? p.H / 2 : p.H, Ws = POOLED ? p.W / 2 : p.W;
  UnitWalk wk(p.C, (long long)p.N * Hs * Ws, kBnUnitsPerThread);
  if (!wk.active) return;
  const int c = wk.c;
  const float4 sc = *reinterpret_cast<const float4*>(p.scale + c);
  const float4 sh = *reinterpret_cast<const float4*>(p.shift + c);
  Geom g{p.N, p.H, p.W};
  Geom gh{p.N, p.H / 2, p.W / 2};
  constexpr int NP = POOLED ? 4 : 1;
  // 8 / 4 independent 16-B loads in flight per thread; the split-K sum keeps one unit's slabs in flight (no spills under the
  // register cap of SSP_BN_BOUNDS)
  constexpr int UNR = SPLIT ? 1 : (POOLED ? 2 : 4);
  for (long long u0 = wk.begin + wk.pl; u0 < wk.end; u0 += (long long)UNR * wk.PL) {
    float4 yv[UNR][NP]; long long rows[UNR][NP]; int nn[UNR], hh[UNR], ww[UNR]; bool ok[UNR];
#pragma unroll
    for (int t = 0; t < UNR; t++) {
      const long long u = u0 + (long long)t * wk.PL;
      ok[t] = u < wk.end;
      const unsigned uu = (unsigned)(ok[t] ? u : wk.begin);          // 32-bit index math: 64-bit div/mod is ~10x the cost
      const unsigned tq = uu / (unsigned)Ws;
      ww[t] = (int)(uu - tq * (unsigned)Ws); nn[t] = (int)(tq / (unsigned)Hs); hh[t] = (int)(tq - (unsigned)nn[t] * (unsigned)Hs);
#pragma unroll
      for (int q = 0; q < NP; q++) {
        const int h = POOLED ? hh[t] * 2 + (q >> 1) : hh[t], w = POOLED ? ww[t] * 2 + (q & 1) : ww[t];
        rows[t][q] = g.row(nn[t], h, w);
        yv[t][q] = *reinterpret_cast<const float4*>(p.y + rows[t][q] * p.y_ld + c);
        if constexpr (SPLIT) {
          for (int s = 1; s < p.splits; s++) {
            const float4 b = *reinterpret_cast<const float4*>(p.y + s * p.slab + rows[t][q] * p.y_ld + c);
            yv[t][q].x += b.x; yv[t][q].y += b.y; yv[t][q].z += b.z; yv[t][q].w += b.w;
          }
        }
      }
    }
#pragma unroll
    for (int t = 0; t < UNR; t++) {
      if (!ok[t]) continue;
      float zmax[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
      float ybest[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int q = 0; q < NP; q++) {
        const int h = POOLED ? hh[t] * 2 + (q >> 1) : hh[t], w = POOLED ? ww[t] * 2 + (q & 1) : ww[t];
        const float4 v = yv[t][q];
        float z[4] = {leaky(fmaf(v.x, sc.x, sh.x), p.slope), leaky(fmaf(v.y, sc.y, sh.y), p.slope),
                      leaky(fmaf(v.z, sc.z, sh.z), p.slope), leaky(fmaf(v.w, sc.w, sh.w), p.slope)};
        if (POOLED) {
          // the first maximum of the ACTIVATED values in (h, w) scan order wins -- the rule of bn_bwd's arg-max (max_pool2d semantics)
          const float yq[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int j = 0; j < 4; j++) if (z[j] > zmax[j]) { zmax[j] = z[j]; ybest[j] = yq[j]; }
        }
#pragma unroll
        for (int d = 0; d < 2; d++) {
          if (p.dst[d].kind == DST_DIRECT) store4(p.dst[d], rows[t][q], c, z);
          else if (p.dst[d].kind == DST_REORG)     // marvis ordering, darknet.py:31-34: ch = ((h%2)*2 + w%2)*C + c
            store4(p.dst[d], gh.row(nn[t], h >> 1, w >> 1), ((h & 1) * 2 + (w & 1)) * p.C + c, z);
        }
      }
      if (POOLED) {
#pragma unroll
        for (int d = 0; d < 2; d++)
          if (p.dst[d].kind == DST_POOL) store4(p.dst[d], gh.row(nn[t], hh[t], ww[t]), c, zmax);
        if (p.ypool)
          *reinterpret_cast<float4*>(p.ypool + gh.row(nn[t], hh[t], ww[t]) * p.ypool_ld + c) = make_float4(ybest[0], ybest[1], ybest[2], ybest[3]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward of (BN -> leaky -> {direct | 2x2 max-pool | reorg} consumers).  Upstream gradients are fp32
// matrices in the consumers' geometries; dz = (sum of routed grads) * leaky'(z).
//   pass 1 (reduce): per-channel  S1 = sum dz,  S2 = sum dz * xhat          (fp64 atomics, one per block/channel)
//   pass 2 (apply):  dY = gamma*invstd * (dz - S1/cnt - xhat*S2/cnt)  -> 16-bit plane (operand of dgrad/wgrad)
enum { SRC_NONE = 0, SRC_DIRECT = 1, SRC_POOL = 2, SRC_REORG = 3 };
struct GradSrc { const float* g; int ld, c0, kind, f16; };   // f16: the plane holds fp16 (written by a GEMM with EPI_F16), ld / c0 in elements
__device__ __forceinline__ float4 load_grad4(const GradSrc& gs, long long elem) {
  if (gs.f16) {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(gs.g) + elem);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return *reinterpret_cast<const float4*>(gs.g + elem);
}
struct BnBwdParams {
  const float* y; int y_ld;
  const float* scale; const float* shift; const float* mean; const float* invstd; const float* gamma;
  int N, C, H, W; float slope; int has_bn;
  GradSrc src[2];
  double* s1; double* s2; double count;
  uint16_t* dy; int dy_ld, dy_fmt; float dy_scale;
};

struct BwdConsts { float4 sc, sh, mu, is; };
__device__ __forceinline__ BwdConsts bwd_consts(const BnBwdParams& p, int c) {
  BwdConsts k;
  k.sc = make_float4(1, 1, 1, 1); k.sh = make_float4(0, 0, 0, 0); k.mu = k.sh; k.is = k.sc;
  if (p.has_bn) {
    k.sc = *reinterpret_cast<const float4*>(p.scale + c); k.sh = *reinterpret_cast<const float4*>(p.shift + c);
    k.mu = *reinterpret_cast<const float4*>(p.mean + c); k.is = *reinterpret_cast<const float4*>(p.invstd + c);
  }
  return k;
}

// one unit (pixel or 2x2 window) of the backward pass: all global loads first, arithmetic afterwards
template <int K0, int K1>
struct BwdUnit {
  static constexpr bool POOLED = (K0 == SRC_POOL || K1 == SRC_POOL);
  static constexpr int NP = POOLED ? 4 : 1;
  float4 y[NP], gd[2][NP], gp[2];
  long long rows[NP];
  bool ok;
  __device__ __forceinline__ void load(const BnBwdParams& p, long long u, long long ubegin, long long uend, int Hs, int Ws, int c) {
    ok = u < uend;
    const unsigned uu = (unsigned)(ok ? u : ubegin);                 // 32-bit index math (units < 2^31)
    const unsigned tq = uu / (unsigned)Ws;
    const int ws = (int)(uu - tq * (unsigned)Ws), n = (int)(tq / (unsigned)Hs), hs = (int)(tq - (unsigned)n * (unsigned)Hs);
    Geom g{p.N, p.H, p.W};
    Geom gh{p.N, p.H / 2, p.W / 2};
#pragma unroll
    for (int q = 0; q < NP; q++) {
      const int h = POOLED ? hs * 2 + (q >> 1) : hs, w = POOLED ? ws * 2 + (q & 1) : ws;
      rows[q] = g.row(n, h, w);
      y[q] = *reinterpret_cast<const float4*>(p.y + rows[q] * p.y_ld + c);
#pragma unroll
      for (int s = 0; s < 2; s++) {
        const GradSrc& gs = p.src[s];
        const int kind = s == 0 ? K0 : K1;                 // compile-time: unused sources cost no registers
        gd[s][q] = make_float4(0, 0, 0, 0);
        if (kind == SRC_DIRECT) gd[s][q] = load_grad4(gs, rows[q] * gs.ld + gs.c0 + c);
        else if (kind == SRC_REORG)
          gd[s][q] = load_grad4(gs, gh.row(n, h >> 1, w >> 1) * gs.ld + gs.c0 + ((h & 1) * 2 + (w & 1)) * p.C + c);
      }
    }
#pragma unroll
    for (int s = 0; s < 2; s++) {
      const int kind = s == 0 ? K0 : K1;
      gp[s] = make_float4(0, 0, 0, 0);
      if (kind == SRC_POOL)
        gp[s] = load_grad4(p.src[s], gh.row(n, hs, ws) * p.src[s].ld + p.src[s].c0 + c);
    }
  }
  // dz = (routed upstream gradient) * leaky'(z);  xh = normalised conv output
  __device__ __forceinline__ void compute(const BnBwdParams& p, const BwdConsts& k, float (&dz)[NP][4], float (&xh)[NP][4]) const {
    float z[NP][4];
#pragma unroll
    for (int q = 0; q < NP; q++) {
      const float4 yv = y[q];
      z[q][0] = fmaf(yv.x, k.sc.x, k.sh.x); z[q][1] = fmaf(yv.y, k.sc.y, k.sh.y);
      z[q][2] = fmaf(yv.z, k.sc.z, k.sh.z); z[q][3] = fmaf(yv.w, k.sc.w, k.sh.w);
      xh[q][0] = (yv.x - k.mu.x) * k.is.x; xh[q][1] = (yv.y - k.mu.y) * k.is.y;
      xh[q][2] = (yv.z - k.mu.z) * k.is.z; xh[q][3] = (yv.w - k.mu.w) * k.is.w;
      dz[q][0] = gd[0][q].x + gd[1][q].x; dz[q][1] = gd[0][q].y + gd[1][q].y;
      dz[q][2] = gd[0][q].z + gd[1][q].z; dz[q][3] = gd[0][q].w + gd[1][q].w;
    }
    if (POOLED) {
      const float gv[4] = {gp[0].x + gp[1].x, gp[0].y + gp[1].y, gp[0].z + gp[1].z, gp[0].w + gp[1].w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        // arg-max of the ACTIVATED values; the first maximum in (h, w) scan order wins (max_pool2d semantics)
        int best = 0; float bv = leaky(z[0][j], p.slope);
#pragma unroll
        for (int q = 1; q < NP; q++) { const float a = leaky(z[q][j], p.slope); if (a > bv) { bv = a; best = q; } }
#pragma unroll
        for (int q = 0; q < NP; q++) if (q == best) dz[q][j] += gv[j];
      }
    }
#pragma unroll
    for (int q = 0; q < NP; q++)
#pragma unroll
      for (int j = 0; j < 4; j++) dz[q][j] *= (z[q][j] > 0.f ? 1.f : p.slope);
  }
};

constexpr int kBwdReduceUnitsPerThread = 32;  // the same for the BN-backward reduction, chosen by a measured sweep

template <int K0, int K1>
__global__ void SSP_BN_BOUNDS bn_bwd_reduce_kernel(const BnBwdParams p) {
  extern __shared__ float red[];           // [2][PL][CG*4]
  constexpr bool POOLED = BwdUnit<K0, K1>::POOLED;
  const int Hs = POOLED ? p.H / 2 : p.H, Ws = POOLED ? p.W / 2 : p.W;
  UnitWalk wk(p.C, (long long)p.N * Hs * Ws, kBwdReduceUnitsPerThread);
  constexpr int NP = POOLED ? 4 : 1;
  constexpr int UNR = POOLED ? 1 : 4;
  const int c = wk.c;
  float a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
  if (wk.active) {
    const BwdConsts k = bwd_consts(p, c);
    for (long long u0 = wk.begin + wk.pl; u0 < wk.end; u0 += (long long)UNR * wk.PL) {
      BwdUnit<K0, K1> un[UNR];
#pragma unroll
      for (int t = 0; t < UNR; t++) un[t].load(p, u0 + (long long)t * wk.PL, wk.begin, wk.end, Hs, Ws, c);
#pragma unroll
      for (int t = 0; t < UNR; t++) {
        if (!un[t].ok) continue;
        float dz[NP][4], xh[NP][4];
        un[t].compute(p, k, dz, xh);
#pragma unroll
        for (int q = 0; q < NP; q++)
#pragma unroll
          for (int j = 0; j < 4; j++) { a1[j] += dz[q][j]; a2[j] = fmaf(dz[q][j], xh[q][j], a2[j]); }
      }
    }
  }
  const int cgs = p.C >> 2, CG = cgs < 256 ? cgs : 256, PL = 256 / CG, CW = CG * 4;
  const int cgi = threadIdx.x % CG, pl = threadIdx.x / CG;
  const int cblocks = (cgs + CG - 1) / CG, cb = blockIdx.x % cblocks;
  if (pl < PL) {
#pragma unroll
    for (int j = 0; j < 4; j++) { red[(0 * PL + pl) * CW + cgi * 4 + j] = a1[j]; red[(1 * PL + pl) * CW + cgi * 4 + j] = a2[j]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * CW; i += 256) {
    const int which = i / CW, cc = i % CW;
    double sacc = 0.0;
    for (int r = 0; r < PL; r++) sacc += (double)red[(which * PL + r) * CW + cc];
    const int ch = cb * CW + cc;
    if (ch < p.C) atomicAdd((which ? p.s2 : p.s1) + ch, sacc);
  }
}

template <int K0, int K1>
__global__ void SSP_BN_BOUNDS bn_bwd_apply_kernel(const BnBwdParams p) {
  constexpr bool POOLED = BwdUnit<K0, K1>::POOLED;
  const int Hs = POOLED ? p.H / 2 : p.H, Ws = POOLED ? p.W / 2 : p.W;
  UnitWalk wk(p.C, (long long)p.N * Hs * Ws, kBnUnitsPerThread);
  if (!wk.active) return;
  constexpr int NP = POOLED ? 4 : 1;
  constexpr int UNR = POOLED ? 1 : 4;
  const int c = wk.c;
  const BwdConsts k = bwd_consts(p, c);
  float k1[4] = {0, 0, 0, 0}, k2[4] = {0, 0, 0, 0}, gsc[4] = {1, 1, 1, 1};
  if (p.has_bn) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      k1[j] = (float)(p.s1[c + j] / p.count); k2[j] = (float)(p.s2[c + j] / p.count);
      gsc[j] = p.gamma[c + j] * p.invstd[c + j] * p.dy_scale;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; j++) gsc[j] = p.dy_scale;
  }
  for (long long u0 = wk.begin + wk.pl; u0 < wk.end; u0 += (long long)UNR * wk.PL) {
    BwdUnit<K0, K1> un[UNR];
#pragma unroll
    for (int t = 0; t < UNR; t++) un[t].load(p, u0 + (long long)t * wk.PL, wk.begin, wk.end, Hs, Ws, c);
#pragma unroll
    for (int t = 0; t < UNR; t++) {
      if (!un[t].ok) continue;
      float dz[NP][4], xh[NP][4];
      un[t].compute(p, k, dz, xh);
#pragma unroll
      for (int q = 0; q < NP; q++) {
        uint16_t o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) o[j] = cvt_f32_to_16(gsc[j] * (dz[q][j] - k1[j] - xh[q][j] * k2[j]), p.dy_fmt);
        *reinterpret_cast<uint2*>(p.dy + un[t].rows[q] * p.dy_ld + c) = make_uint2(o[0] | ((uint32_t)o[1] << 16), o[2] | ((uint32_t)o[3] << 16));
      }
    }
  }
}

// dgamma = S2, dbeta = S1 (accumulate into the gradient buffers), then clear S1/S2.  Launch AFTER bn_bwd_apply.
__global__ void bn_bwd_finalize_kernel(double* __restrict__ s1, double* __restrict__ s2, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int C, int accumulate, float scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float a = (float)(s2[c] * (double)scale), b = (float)(s1[c] * (double)scale);
  if (accumulate) { dgamma[c] += a; dbeta[c] += b; }
  else { dgamma[c] = a; dbeta[c] = b; }
  s1[c] = 0.0; s2[c] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// column sums of an NCHW fp32 tensor over (n, h, w): bias gradient of the linear head (conv 30)
__global__ void bias_grad_nchw_kernel(const float* __restrict__ g, float* __restrict__ db, int N, int C, int HW, int accumulate, float scale) {
  const int c = blockIdx.x;
  double s = 0.0;
  for (int i = threadIdx.x; i < N * HW; i += blockDim.x) s += (double)g[((long long)(i / HW) * C + c) * HW + (i % HW)];
  __shared__ double sm[256];
  sm[threadIdx.x] = s; __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) { const float v = (float)(sm[0] * (double)scale); if (accumulate) db[c] += v; else db[c] = v; }
}

// ------------------------------------------------------------------------------------------------
// Weight re-packing.  Master weights: fp32 [cout][taps][cin] (the memory behind the permuted nn.Conv2d.weight view).
//   fwd  : hi/lo fp16 [cout][ld_f]      k = tap*cin + ci                 (B operand of the forward GEMM)
//   dgrad: 16-bit     [cin][ld_d]       k = tap'*cout + co, tap' = taps-1-tap   (B operand of the data-gradient GEMM)
// A 64(co) x 64(ci) tile of one tap per block moves through shared memory so that BOTH the forward planes and the transposed
// data-gradient plane are written in 128-B rows (a one-thread-per-weight kernel would write the transposed plane with row-strided
// 2-byte stores).
__global__ void __launch_bounds__(256) pack_weights_tiled_kernel(const float* __restrict__ w, int cout, int taps, int cin,
                                                                 uint16_t* __restrict__ f_hi, uint16_t* __restrict__ f_lo, int ld_f,
                                                                 uint16_t* __restrict__ d, int ld_d, int d_fmt) {
  __shared__ uint16_t tile[64][66];                 // [ci][co], +2 pad: 33-word row pitch, conflict-free both ways
  const int ci0 = blockIdx.x * 64, co0 = blockIdx.y * 64, tap = blockIdx.z;
  const int lane64 = threadIdx.x & 63, grp = threadIdx.x >> 6;      // 4 groups of 64 threads
#pragma unroll 4
  for (int r = 0; r < 16; r++) {
    const int co = co0 + r * 4 + grp, ci = ci0 + lane64;            // consecutive threads -> consecutive ci (coalesced fp32 reads)
    uint16_t t = 0;
    if (co < cout && ci < cin) {
      const float v = w[((long long)co * taps + tap) * cin + ci];
      if (f_hi) {
        uint16_t a, b; split_f16(v, a, b);
        const long long o = (long long)co * ld_f + tap * cin + ci;
        f_hi[o] = a; if (f_lo) f_lo[o] = b;
      }
      t = cvt_f32_to_16(v, d_fmt);
    }
    tile[lane64][r * 4 + grp] = t;
  }
  if (!d) return;
  __syncthreads();
#pragma unroll 4
  for (int r = 0; r < 16; r++) {
    const int ci = ci0 + r * 4 + grp, co = co0 + lane64;            // consecutive threads -> consecutive co (coalesced 16-bit writes)
    if (ci < cin && co < cout) d[(long long)ci * ld_d + (long long)(taps - 1 - tap) * cout + co] = tile[r * 4 + grp][lane64];
  }
}


// ------------------------------------------------------------------------------------------------
// optim.SGD(momentum, dampening=0, weight_decay) over one flat buffer (train.py:388):
//   g += wd*p ; v = mu*v + g ; p -= lr*v      (first step of torch: v = g, identical with v0 = 0)
__global__ void sgd_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v, long long n,
                                float lr, float mu, float wd, float gscale) {
  const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 + 3 < n) {
    float4 pp = *reinterpret_cast<float4*>(p + i4);
    const float4 gg = *reinterpret_cast<const float4*>(g + i4);
    float4 vv = *reinterpret_cast<float4*>(v + i4);
    sgd_update(pp.x, gg.x, vv.x, lr, mu, wd, gscale); sgd_update(pp.y, gg.y, vv.y, lr, mu, wd, gscale);
    sgd_update(pp.z, gg.z, vv.z, lr, mu, wd, gscale); sgd_update(pp.w, gg.w, vv.w, lr, mu, wd, gscale);
    *reinterpret_cast<float4*>(v + i4) = vv;
    *reinterpret_cast<float4*>(p + i4) = pp;
  } else {
    for (long long i = i4; i < n; i++) {
      float pv = p[i], vv = v[i];
      sgd_update(pv, g[i], vv, lr, mu, wd, gscale);
      v[i] = vv; p[i] = pv;
    }
  }
}

// ================================================================================================ host launchers
static inline unsigned nblk(long long total, int bs) { return (unsigned)((total + bs - 1) / bs); }
static inline bool aligned(const void* p, int bytes) { return ((uintptr_t)p % bytes) == 0; }

// Layout rules of the 4-channel vectors of the BN kernels, checked before any launch: a misaligned vector access would fault.
// The fp32 conv output y is read in 16-B vectors at row * y_ld + c.
static bool y_layout_ok(const float* y, int y_ld, int C) { return aligned(y, 16) && y_ld % 4 == 0 && y_ld >= C; }
// A 16-bit destination (8-B stores) or an upstream gradient plane (8-B fp16 / 16-B fp32 loads) at row * ld + c0 + channel, with
// channels [c0, c0 + C), or [c0, c0 + 4C) behind a reorg.
static bool plane_layout_ok(const void* base, int elem_bytes, int ld, int c0, int route, int C) {
  return aligned(base, 4 * elem_bytes) && ld % 4 == 0 && c0 % 4 == 0 && c0 >= 0 && ld >= c0 + (route == SSP_ROUTE_REORG ? 4 * C : C);
}

// ssp_bn_apply and ssp_bn_apply_splitk.  splits == 1 launches the plain kernel (the ssp_bn_apply path); splits > 1 the instantiation
// that sums the partial slabs first
static int bn_apply_splitk(const float* y, int splits, long long slab, int y_ld, const float* scale, const float* shift, int N, int C, int H, int W,
                           float slope, void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_kind, void* d1_hi, void* d1_lo, int d1_ld, int d1_c0,
                           int d1_kind, cudaStream_t s, float* ypool, int ypool_ld) {
  if (!y || !scale || !shift || (C % 4)) return fail_msg(SSP_ERR_ARG, "bn_apply: bad argument (C must be a multiple of 4)");
  if (splits < 1 || (splits > 1 && (((uintptr_t)y % 16) || (y_ld % 4) || y_ld < C || (slab % 4) || slab < (long long)y_ld * flat_alloc_rows(N, H, W))))
    return fail_msg(SSP_ERR_ARG, "bn_apply_splitk: splits >= 1; partial slabs 16-B aligned, partial_ld % 4 == 0 and >= C, slab_elems % 4 == 0 and "
                                 ">= ssp_flat_alloc_rows(N, H, W) * partial_ld");
  if (!y_layout_ok(y, y_ld, C)) return fail_msg(SSP_ERR_ARG, "bn_apply: y must be 16-B aligned with y_ld % 4 == 0 and y_ld >= C");
  if (ypool && !y_layout_ok(ypool, ypool_ld, C)) return fail_msg(SSP_ERR_ARG, "bn_apply: arg-max plane must be 16-B aligned with ld % 4 == 0 and ld >= C");
  const struct { void* hi; void* lo; int ld, c0, kind; } dsts[2] = {{d0_hi, d0_lo, d0_ld, d0_c0, d0_kind}, {d1_hi, d1_lo, d1_ld, d1_c0, d1_kind}};
  for (const auto& d : dsts)
    if (d.hi && d.kind != DST_NONE && !(plane_layout_ok(d.hi, 2, d.ld, d.c0, d.kind, C) && (!d.lo || aligned(d.lo, 8))))
      return fail_msg(SSP_ERR_ARG, "bn_apply: destination planes must be 8-B aligned with ld % 4 == 0, c0 % 4 == 0 and ld >= c0 + C "
                                   "(c0 + 4C for a reorg)");
  BnApplyParams p;
  p.y = y; p.y_ld = y_ld; p.scale = scale; p.shift = shift; p.N = N; p.C = C; p.H = H; p.W = W; p.slope = slope;
  p.dst[0] = ActDst{(uint16_t*)d0_hi, (uint16_t*)d0_lo, d0_ld, d0_c0, d0_hi ? d0_kind : DST_NONE};
  p.dst[1] = ActDst{(uint16_t*)d1_hi, (uint16_t*)d1_lo, d1_ld, d1_c0, d1_hi ? d1_kind : DST_NONE};
  const bool pooled = p.dst[0].kind == DST_POOL || p.dst[1].kind == DST_POOL;
  if (ypool && !pooled) return fail_msg(SSP_ERR_ARG, "bn_apply: the arg-max plane belongs to a max-pool destination");
  p.ypool = ypool; p.ypool_ld = ypool_ld;
  p.splits = splits; p.slab = slab;
  const bool halves = pooled || p.dst[0].kind == DST_REORG || p.dst[1].kind == DST_REORG;
  if (halves && ((H | W) & 1)) return fail_msg(SSP_ERR_ARG, "bn_apply: pool/reorg need even H and W");
  const unsigned grid = pooled ? unit_grid(C, (long long)N * (H / 2) * (W / 2), kBnUnitsPerThread) : unit_grid(C, (long long)N * H * W, kBnUnitsPerThread);
  if (splits > 1) {
    if (pooled) bn_apply_kernel<true, true><<<grid, 256, 0, s>>>(p);
    else bn_apply_kernel<false, true><<<grid, 256, 0, s>>>(p);
  } else if (pooled) bn_apply_kernel<true><<<grid, 256, 0, s>>>(p);
  else bn_apply_kernel<false><<<grid, 256, 0, s>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

static int fill_bwd(BnBwdParams& p, const float* y, int y_ld, const float* scale, const float* shift, const float* mean,
                    const float* invstd, const float* gamma, int N, int C, int H, int W, float slope,
                    const float* g0, int g0_ld, int g0_c0, int g0_kind, const float* g1, int g1_ld, int g1_c0, int g1_kind,
                    double* s1, double* s2) {
  if (!y || (C % 4) || !g0) return SSP_ERR_ARG;
  p.y = y; p.y_ld = y_ld; p.scale = scale; p.shift = shift; p.mean = mean; p.invstd = invstd; p.gamma = gamma;
  p.has_bn = (scale && shift && mean && invstd && gamma) ? 1 : 0;
  p.N = N; p.C = C; p.H = H; p.W = W; p.slope = slope;
  p.src[0] = GradSrc{g0, g0_ld, g0_c0, g0_kind & 15, (g0_kind & SSP_ROUTE_F16) ? 1 : 0};
  p.src[1] = GradSrc{g1, g1_ld, g1_c0, g1 ? (g1_kind & 15) : SRC_NONE, (g1_kind & SSP_ROUTE_F16) ? 1 : 0};
  p.s1 = s1; p.s2 = s2; p.count = (double)N * H * W;
  p.dy = nullptr; p.dy_ld = 0; p.dy_fmt = 0; p.dy_scale = 1.f;
  return SSP_OK;
}
// layout rules of y and of the upstream gradient planes, after fill_bwd has accepted the arguments
static int check_bwd_layout(const BnBwdParams& p) {
  if (!y_layout_ok(p.y, p.y_ld, p.C)) return fail_msg(SSP_ERR_ARG, "bn_bwd: y must be 16-B aligned with y_ld % 4 == 0 and y_ld >= C");
  for (const GradSrc& gs : p.src)
    if (gs.kind != SRC_NONE && !plane_layout_ok(gs.g, gs.f16 ? 2 : 4, gs.ld, gs.c0, gs.kind, p.C))
      return fail_msg(SSP_ERR_ARG, "bn_bwd: gradient planes must be 16-B (fp32) / 8-B (fp16) aligned with ld % 4 == 0, c0 % 4 == 0 "
                                   "and ld >= c0 + C (c0 + 4C for a reorg)");
  return SSP_OK;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_pack_nchw(const float* x, void* hi, void* lo, int N, int C, int H, int W, int ld, int c0, int fmt, float scale, void* stream) {
  if (!x || !hi) return fail_msg(SSP_ERR_ARG, "pack_nchw: null pointer");
  const long long total = (long long)N * C * H * W;
  pack_nchw_kernel<<<nblk(total, 256), 256, 0, (cudaStream_t)stream>>>(x, (uint16_t*)hi, (uint16_t*)lo, N, C, H, W, ld, c0, fmt, scale);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_unpack_nchw(const float* y, float* out, int N, int C, int H, int W, int ld, int c0, void* stream) {
  if (!y || !out) return fail_msg(SSP_ERR_ARG, "unpack_nchw: null pointer");
  const long long total = (long long)N * C * H * W;
  unpack_nchw_kernel<<<nblk(total, 256), 256, 0, (cudaStream_t)stream>>>(y, out, N, C, H, W, ld, c0);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_unpack16_nchw(const void* hi, const void* lo, float* out, int N, int C, int H, int W, int ld, int c0, int fmt, void* stream) {
  if (!hi || !out) return fail_msg(SSP_ERR_ARG, "unpack16_nchw: null pointer");
  const long long total = (long long)N * C * H * W;
  unpack16_nchw_kernel<<<nblk(total, 256), 256, 0, (cudaStream_t)stream>>>((const uint16_t*)hi, (const uint16_t*)lo, out, N, C, H, W, ld, c0, fmt);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_bn_finalize(double* ssum, double* ssq, double count, const float* gamma, const float* beta, float* rm, float* rv,
                    float momentum, float eps, int train, float* mean, float* invstd, float* scale, float* shift, int C, void* stream) {
  if (!gamma || !beta || !mean || !invstd || !scale || !shift || (train && (!ssum || !ssq)) || (!train && (!rm || !rv)))
    return fail_msg(SSP_ERR_ARG, "bn_finalize: null pointer");
  bn_finalize_kernel<<<nblk(C, 128), 128, 0, (cudaStream_t)stream>>>(ssum, ssq, count, gamma, beta, rm, rv, momentum, eps, train, mean, invstd,
                                                                     scale, shift, C);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_bn_apply(const float* y, int y_ld, const float* scale, const float* shift, int N, int C, int H, int W, float slope,
                 void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_kind,
                 void* d1_hi, void* d1_lo, int d1_ld, int d1_c0, int d1_kind, float* ypool, int ypool_ld, void* stream) {
  return bn_apply_splitk(y, 1, 0, y_ld, scale, shift, N, C, H, W, slope, d0_hi, d0_lo, d0_ld, d0_c0, d0_kind, d1_hi, d1_lo, d1_ld, d1_c0, d1_kind,
                         (cudaStream_t)stream, ypool, ypool_ld);
}
int ssp_bn_apply_splitk(const float* partial, int splits, long long slab_elems, int partial_ld, const float* scale, const float* shift, int N, int C,
                        int H, int W, float slope, void* d0_hi, void* d0_lo, int d0_ld, int d0_c0, int d0_kind, void* d1_hi, void* d1_lo, int d1_ld,
                        int d1_c0, int d1_kind, void* stream) {
  return bn_apply_splitk(partial, splits, slab_elems, partial_ld, scale, shift, N, C, H, W, slope, d0_hi, d0_lo, d0_ld, d0_c0, d0_kind, d1_hi, d1_lo,
                         d1_ld, d1_c0, d1_kind, (cudaStream_t)stream, nullptr, 0);
}
int ssp_bn_bwd_reduce(const float* y, int y_ld, const float* scale, const float* shift, const float* mean, const float* invstd,
                      const float* gamma, int N, int C, int H, int W, float slope,
                      const float* g0, int g0_ld, int g0_c0, int g0_kind, const float* g1, int g1_ld, int g1_c0, int g1_kind,
                      double* s1, double* s2, void* stream) {
  BnBwdParams p;
  if (fill_bwd(p, y, y_ld, scale, shift, mean, invstd, gamma, N, C, H, W, slope, g0, g0_ld, g0_c0, g0_kind, g1, g1_ld, g1_c0, g1_kind, s1, s2) || !s1 || !s2 || !p.has_bn)
    return fail_msg(SSP_ERR_ARG, "bn_bwd_reduce: bad argument");
  if (const int rc = check_bwd_layout(p)) return rc;
  const bool pooled = p.src[0].kind == SRC_POOL || p.src[1].kind == SRC_POOL;
  const int cgs = C / 4, CG = cgs < 256 ? cgs : 256, PL = 256 / CG;
  const long long nunits = (long long)N * (pooled ? H / 2 : H) * (pooled ? W / 2 : W);
  const size_t sm = (size_t)2 * PL * CG * 4 * sizeof(float);
  const unsigned grid = unit_grid(C, nunits, kBwdReduceUnitsPerThread);
#define SSP_BWD_DISPATCH(KERN, ...)                                                                                  \
  do {                                                                                                              \
    const int k0 = p.src[0].kind, k1 = p.src[1].kind;                                                               \
    if (k0 == SRC_DIRECT && k1 == SRC_NONE) KERN<SRC_DIRECT, SRC_NONE><<<__VA_ARGS__>>>(p);                         \
    else if (k0 == SRC_POOL && k1 == SRC_NONE) KERN<SRC_POOL, SRC_NONE><<<__VA_ARGS__>>>(p);                        \
    else if (k0 == SRC_REORG && k1 == SRC_NONE) KERN<SRC_REORG, SRC_NONE><<<__VA_ARGS__>>>(p);                      \
    else if (k0 == SRC_POOL && k1 == SRC_DIRECT) KERN<SRC_POOL, SRC_DIRECT><<<__VA_ARGS__>>>(p);                    \
    else if (k0 == SRC_DIRECT && k1 == SRC_POOL) KERN<SRC_DIRECT, SRC_POOL><<<__VA_ARGS__>>>(p);                    \
    else if (k0 == SRC_DIRECT && k1 == SRC_DIRECT) KERN<SRC_DIRECT, SRC_DIRECT><<<__VA_ARGS__>>>(p);                \
    else if (k0 == SRC_DIRECT && k1 == SRC_REORG) KERN<SRC_DIRECT, SRC_REORG><<<__VA_ARGS__>>>(p);                  \
    else if (k0 == SRC_REORG && k1 == SRC_DIRECT) KERN<SRC_REORG, SRC_DIRECT><<<__VA_ARGS__>>>(p);                  \
    else return fail_msg(SSP_ERR_ARG, "bn_bwd: unsupported combination of gradient routes");                         \
  } while (0)
  SSP_BWD_DISPATCH(bn_bwd_reduce_kernel, grid, 256, sm, (cudaStream_t)stream);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_bn_bwd_apply(const float* y, int y_ld, const float* scale, const float* shift, const float* mean, const float* invstd,
                     const float* gamma, int N, int C, int H, int W, float slope,
                     const float* g0, int g0_ld, int g0_c0, int g0_kind, const float* g1, int g1_ld, int g1_c0, int g1_kind,
                     double* s1, double* s2, void* dy, int dy_ld, int dy_fmt, float dy_scale, void* stream) {
  BnBwdParams p;
  if (fill_bwd(p, y, y_ld, scale, shift, mean, invstd, gamma, N, C, H, W, slope, g0, g0_ld, g0_c0, g0_kind, g1, g1_ld, g1_c0, g1_kind, s1, s2) || !dy)
    return fail_msg(SSP_ERR_ARG, "bn_bwd_apply: bad argument");
  if (p.has_bn && (!s1 || !s2)) return fail_msg(SSP_ERR_ARG, "bn_bwd_apply: statistics buffers missing");
  if (const int rc = check_bwd_layout(p)) return rc;
  if (!aligned(dy, 8) || (dy_ld % 4) || dy_ld < C) return fail_msg(SSP_ERR_ARG, "bn_bwd_apply: dY must be 8-B aligned with dy_ld % 4 == 0 and dy_ld >= C");
  p.dy = (uint16_t*)dy; p.dy_ld = dy_ld; p.dy_fmt = dy_fmt; p.dy_scale = dy_scale;
  const bool pooled = p.src[0].kind == SRC_POOL || p.src[1].kind == SRC_POOL;
  const long long nunits = (long long)N * (pooled ? H / 2 : H) * (pooled ? W / 2 : W);
  const unsigned grid = unit_grid(C, nunits, kBnUnitsPerThread);
  SSP_BWD_DISPATCH(bn_bwd_apply_kernel, grid, 256, 0, (cudaStream_t)stream);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_bn_bwd_finalize(double* s1, double* s2, float* dgamma, float* dbeta, int C, int accumulate, float scale, void* stream) {
  if (!s1 || !s2 || !dgamma || !dbeta) return fail_msg(SSP_ERR_ARG, "bn_bwd_finalize: null pointer");
  bn_bwd_finalize_kernel<<<nblk(C, 128), 128, 0, (cudaStream_t)stream>>>(s1, s2, dgamma, dbeta, C, accumulate, scale);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_bias_grad_nchw(const float* g, float* db, int N, int C, int HW, int accumulate, float scale, void* stream) {
  if (!g || !db) return fail_msg(SSP_ERR_ARG, "bias_grad_nchw: null pointer");
  bias_grad_nchw_kernel<<<C, 256, 0, (cudaStream_t)stream>>>(g, db, N, C, HW, accumulate, scale);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_pack_weights(const float* w, int cout, int taps, int cin, void* f_hi, void* f_lo, int ld_f, void* d, int ld_d, int d_fmt, void* stream) {
  if (!w || cout <= 0 || taps <= 0 || cin <= 0 || taps > 65535) return fail_msg(SSP_ERR_ARG, "pack_weights: bad argument");
  dim3 grid((cin + 63) / 64, (cout + 63) / 64, taps);
  if (grid.y > 65535) return fail_msg(SSP_ERR_ARG, "pack_weights: cout too large");
  pack_weights_tiled_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, cout, taps, cin, (uint16_t*)f_hi, (uint16_t*)f_lo, ld_f, (uint16_t*)d, ld_d, d_fmt);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
int ssp_sgd_step_flat(float* p, const float* g, float* v, long long n, float lr, float mu, float wd, float gscale, void* stream) {
  if (!p || !g || !v) return fail_msg(SSP_ERR_ARG, "sgd_step_flat: null pointer");
  sgd_flat_kernel<<<nblk((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(p, g, v, n, lr, mu, wd, gscale);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
