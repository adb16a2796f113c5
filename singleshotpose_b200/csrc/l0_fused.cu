// First layer (3 -> 32 channels, 3x3, K = 27) followed by BatchNorm + LeakyReLU + 2x2 max-pool, WITHOUT ever materialising the
// 416x416x32 conv output: at batch 64 that tensor is 1.42 GB of fp32, and round 1/2 wrote it once and read it three times
// (bn_apply, bn_bwd_apply, plus a 0.7 GB fp16 dY plane and a 0.7 GB im2col plane for the weight gradient): 2.5 ms of a 16.5 ms
// step for 0.07 % of the FLOPs.  Everything the training step needs from layer 0 is a function of the image patches
// p(px) in R^27, the 864 weights and a few per-channel sums, because y = W p is LINEAR in p:
//
//   forward   sum_px y_c     = w_c . (sum_px p)                 -> colsum  (27 numbers per batch)
//             sum_px y_c^2   = w_c^T (sum_px p p^T) w_c         -> Gram matrix G (27 x 27 per batch)
//             => BN batch statistics without a pass over y; then ONE kernel: conv + BN + leaky + pool -> the consumer's fp16 hi/lo
//             operand planes and a 1-byte code per pooled cell (arg-max position, sign of the pre-activation).
//   backward  dz is non-zero only at the arg-max of every window:  dz = dX_pool * leaky'(z_argmax)
//             S1_c = sum dz,   T_c = sum dz * p(argmax)  (27-vector),   sum dz*y = w_c . T_c,   S2_c = invstd (w_c . T_c - mean S1)
//             dY = gamma invstd (dz - S1/n - xhat S2/n) is never formed:  dW_c = sum_px p dY
//                 = gamma invstd [ T_c - (S1/n) colsum - (S2/n) invstd (G w_c - mean colsum) ]
//             => one kernel over the POOLED gradient (quarter resolution) + the image, and a 32-thread epilogue.
// The algebra is exact; only the summation order differs from autograd (fp64 across threads, fp32 inside a thread).
// Replaces nn.Conv2d(3,32,3,1,1) + BatchNorm2d + LeakyReLU + MaxPool2d(2,2) of reference darknet.py:154-167 (blocks 0-1 of
// cfg/yolo-pose.cfg) and their autograd (train.py:103).
#include "ssp_common.cuh"

namespace ssp {

namespace {
constexpr int kC0 = 32;               // output channels
constexpr int kTH = 16, kTW = 32;     // pixel tile of one block iteration
constexpr int kInW = 37;              // smem row pitch of the halo tile (odd)
constexpr int kG = 28;                // 27 patch entries + the constant 1 (its Gram row is colsum, G[27][27] = pixel count)

struct Tile { int n, h0, w0; };
__device__ __forceinline__ Tile tile_of(int tile, int tiles_h, int tiles_w) {
  Tile t; t.w0 = (tile % tiles_w) * kTW; t.h0 = ((tile / tiles_w) % tiles_h) * kTH; t.n = tile / (tiles_w * tiles_h); return t;
}
// Halo tile (3 x 18 x 34) of image n around (h0, w0), zero outside the image (the convolution's padding), staged through registers:
// halo_fetch() issues the global loads of a tile (element i = tid + 256 k, k < 8), halo_store() writes them to shared memory one
// tile later -- the loads of tile t+1 are in flight while tile t is computed (round 2, ncu: with a plain load-sync-compute loop
// 25-50 % of the samples of these kernels sat on the STS waiting for its LDG, one resident block per SM had nothing to overlap).
// (c, rr, cc) walk incrementally: 256 = 7 * 34 + 18.
constexpr int kHaloElems = 3 * (kTH + 2) * (kTW + 2);
constexpr int kHaloPer = (kHaloElems + 255) / 256;
__device__ __forceinline__ void halo_fetch(float (&pre)[kHaloPer], const float* __restrict__ x, const Tile& t, int H, int W) {
  const long long HW = (long long)H * W;
  const float* xi = x + (long long)t.n * 3 * HW;
  int cc = threadIdx.x % (kTW + 2), rr = threadIdx.x / (kTW + 2), c = 0;       // tid < 256 < 18 * 34: c = 0
#pragma unroll
  for (int k = 0; k < kHaloPer; k++) {
    const int hh = t.h0 + rr - 1, ww = t.w0 + cc - 1;
    const bool ok = (c < 3) && hh >= 0 && hh < H && ww >= 0 && ww < W;
    pre[k] = ok ? __ldg(xi + c * HW + (long long)hh * W + ww) : 0.f;
    cc += 256 % (kTW + 2); rr += 256 / (kTW + 2);
    if (cc >= kTW + 2) { cc -= kTW + 2; rr++; }
    if (rr >= kTH + 2) { rr -= kTH + 2; c++; }
  }
}
__device__ __forceinline__ void halo_store(float (*sin)[kTH + 2][kInW], const float (&pre)[kHaloPer]) {
  int cc = threadIdx.x % (kTW + 2), rr = threadIdx.x / (kTW + 2), c = 0;
#pragma unroll
  for (int k = 0; k < kHaloPer; k++) {
    if (c < 3) sin[c][rr][cc] = pre[k];
    cc += 256 % (kTW + 2); rr += 256 / (kTW + 2);
    if (cc >= kTW + 2) { cc -= kTW + 2; rr++; }
    if (rr >= kTH + 2) { rr -= kTH + 2; c++; }
  }
}
}  // namespace

// ------------------------------------------------------------------------------------------------ Gram matrix of the patches
// gram[a][b] (a <= b, fp64, accumulated) = sum over all pixels of q[a] q[b], q = (patch[27], 1); patch index k = (kh*3+kw)*3 + c.
// Warp role r owns the Gram rows [RA, RB) (~100 accumulators per lane, static indices); the two warps of a role split the tile's pixels.
template <int RA, int RB>
__device__ __forceinline__ void gram_rows(const float (*sin)[kTH + 2][kInW], int lane, const Tile& t, int H, int W,
                                          float* acc /*[sum over rows of (28 - a)]*/) {
#pragma unroll 1
  for (int it = 0; it < (kTH * kTW) / 32; it++) {            // one tile row of 32 pixels per iteration
    const int pr = it, pc = lane;
    const bool ok = (t.h0 + pr < H) && (t.w0 + pc < W);
    float q[kG];
#pragma unroll
    for (int k = RA; k < 27; k++) {
      const int c = k % 3, kw = (k / 3) % 3, kh = k / 9;
      q[k] = ok ? sin[c][pr + kh][pc + kw] : 0.f;
    }
    q[27] = ok ? 1.f : 0.f;
    int idx = 0;
#pragma unroll
    for (int a = RA; a < RB; a++)
#pragma unroll
      for (int b = a; b < kG; b++) { acc[idx] = fmaf(q[a], q[b], acc[idx]); idx++; }
  }
}
template <int RA, int RB>
__device__ __forceinline__ void gram_flush(const float* acc, int lane, double* gram) {
  int idx = 0;
#pragma unroll
  for (int a = RA; a < RB; a++)
#pragma unroll
    for (int b = a; b < kG; b++) {
      float v = acc[idx++];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0 && v != 0.f) atomicAdd(gram + a * kG + b, (double)v);
    }
}

// Warp w owns the Gram rows of role w (43 ... 57 accumulators per lane, static indices) and walks all 512 pixels of every tile.
#define SSP_GRAM_ROLES(F)                                                                                                   \
  switch (warp) {                                                                                                           \
    case 0: F(0, 2); break; case 1: F(2, 4); break; case 2: F(4, 6); break; case 3: F(6, 8); break;                         \
    case 4: F(8, 11); break; case 5: F(11, 14); break; case 6: F(14, 18); break; default: F(18, 28); break;                 \
  }

__global__ void __launch_bounds__(256, 2) l0_gram_kernel(const float* __restrict__ x, double* __restrict__ gram, int N, int H, int W) {
  __shared__ float sin[3][kTH + 2][kInW];
  const int tiles_w = (W + kTW - 1) / kTW, tiles_h = (H + kTH - 1) / kTH;
  const int ntiles = N * tiles_h * tiles_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[57];
#pragma unroll
  for (int i = 0; i < 57; i++) acc[i] = 0.f;
  float pre[kHaloPer];
  if ((int)blockIdx.x < ntiles) halo_fetch(pre, x, tile_of(blockIdx.x, tiles_h, tiles_w), H, W);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const Tile t = tile_of(tile, tiles_h, tiles_w);
    __syncthreads();
    halo_store(sin, pre);
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) halo_fetch(pre, x, tile_of(tile + gridDim.x, tiles_h, tiles_w), H, W);
#define SSP_GRAM_RUN(A, B) gram_rows<A, B>(sin, lane, t, H, W, acc)
    SSP_GRAM_ROLES(SSP_GRAM_RUN)
  }
#define SSP_GRAM_FLUSH(A, B) gram_flush<A, B>(acc, lane, gram)
  SSP_GRAM_ROLES(SSP_GRAM_FLUSH)
}

// ------------------------------------------------------------------------------------------------ Gram matrix through shift correlations
// The brute-force kernel above forms all 406 products of every pixel's 28-vector.  But patch entry (kh, kw, c) of output pixel p is the
// image value x_c(u), u = p + (kh-1, kw-1), so
//     G[(t,c),(t',c')] = sum over u in (image minus the rows / columns that tap t cannot reach) of x_c(u) * x~_c'(u + D),   D = t' - t,
// (x~ = zero outside the image) = C[c,c',D] - Row[..] - Col[..] + Corner[..] with
//     C[c,c',D] = sum over ALL image pixels u of x_c(u) x~_c'(u + D)      -- 25 shifts x 9 channel pairs, C[c,c',D] = C[c',c,-D]: 117 numbers
// and the corrections sums of the same products over the first / last row and column (tap kh = 0 never reaches the last image row,
// kh = 2 never the first; likewise kw).  l0_corr_kernel: 117 FMAs per pixel instead of 406, four pixels per lane share one 3 x 8 x 3
// window (72 shared-memory loads per 468 FMAs); l0_border_kernel: the 8 border sets by brute force (2(H+W) pixels per image);
// l0_gram_assemble_kernel: the 28 x 28 matrix (column 27 = sums of x, entry [27][27] = pixel count).  Round 2: 467 -> ~100 us.
namespace {
constexpr int kCorrN = 13 * 9 + 3;          // 13 shifts D >= 0 (lexicographic) x c x c', then the three channel sums
constexpr int kGramScratch = 784;           // scratch behind the 28 x 28 matrix: C (117) | E[8][25][9] | T1[3] | ES1[8][3]
constexpr int kOffC = kGramScratch, kOffE = kOffC + 117, kOffT1 = kOffE + 8 * 225, kOffES1 = kOffT1 + 3, kGramDoubles = kOffES1 + 24;
constexpr int kCT = 32;                     // correlation tile: 32 x 32 pixels, halo 2 rows below, 2 columns left / right
constexpr int kCW = kCT + 4, kCH = kCT + 2, kCP = 37;
__device__ __forceinline__ int shift_index(int dh, int dw) { return dh == 0 ? dw : 3 + (dh - 1) * 5 + (dw + 2); }      // D >= 0 only
}

__global__ void __launch_bounds__(256, 1) l0_corr_kernel(const float* __restrict__ x, double* __restrict__ gram, int N, int H, int W) {
  __shared__ float sx[3][kCH][kCP];
  __shared__ double sacc[kCorrN];
  for (int i = threadIdx.x; i < kCorrN; i += 256) sacc[i] = 0.0;
  const int tiles_w = (W + kCT - 1) / kCT, tiles_h = (H + kCT - 1) / kCT;
  const int ntiles = N * tiles_h * tiles_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = 4 * warp + (lane >> 3), c0 = 4 * (lane & 7);        // this lane's 4 consecutive pixels inside the tile
  const long long HW = (long long)H * W;
  float acc[kCorrN];
#pragma unroll
  for (int i = 0; i < kCorrN; i++) acc[i] = 0.f;
  constexpr int kPer = (3 * kCH * kCW + 255) / 256;                  // halo elements per thread (15), staged one tile ahead
  float pre[kPer];
  auto fetch = [&](int tile) {
    const int w0 = (tile % tiles_w) * kCT, h0 = ((tile / tiles_w) % tiles_h) * kCT, n = tile / (tiles_w * tiles_h);
    const float* xi = x + (long long)n * 3 * HW;
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const int i = threadIdx.x + 256 * k;
      const int cc = i % kCW, rr = (i / kCW) % kCH, c = i / (kCW * kCH);
      const int hh = h0 + rr, ww = w0 + cc - 2;
      pre[k] = (c < 3 && hh < H && ww >= 0 && ww < W) ? __ldg(xi + c * HW + (long long)hh * W + ww) : 0.f;
    }
  };
  if ((int)blockIdx.x < ntiles) fetch(blockIdx.x);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const int i = threadIdx.x + 256 * k;
      const int cc = i % kCW, rr = (i / kCW) % kCH, c = i / (kCW * kCH);
      if (c < 3) sx[c][rr][cc] = pre[k];
    }
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) fetch(tile + gridDim.x);
    float win[3][3][8];                                              // [channel][row r0 + dh][column c0 - 2 ... c0 + 5]
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int dh = 0; dh < 3; dh++)
#pragma unroll
        for (int j = 0; j < 8; j++) win[c][dh][j] = sx[c][r0 + dh][c0 + j];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float xv = win[c][0][2 + i];                           // zero for pixels of the tile that lie outside the image
        acc[117 + c] += xv;
#pragma unroll
        for (int dh = 0; dh < 3; dh++)
#pragma unroll
          for (int dw = -2; dw <= 2; dw++) {
            if (dh == 0 && dw < 0) continue;
#pragma unroll
            for (int c2 = 0; c2 < 3; c2++) {
              const int a = shift_index(dh, dw) * 9 + c * 3 + c2;
              acc[a] = fmaf(xv, win[c2][dh][2 + i + dw], acc[a]);
            }
          }
      }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kCorrN; i++) {
    float v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) atomicAdd(&sacc[i], (double)v);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kCorrN; i += 256) if (sacc[i] != 0.0) atomicAdd(gram + (i < 117 ? kOffC + i : kOffT1 + (i - 117)), sacc[i]);
}

// border sets: 0 = first row, 1 = last row, 2 = first column, 3 = last column, 4..7 = corners (0,0) (0,L) (L,0) (L,L)
__global__ void __launch_bounds__(256) l0_border_kernel(const float* __restrict__ x, double* __restrict__ gram, int N, int H, int W, int chunks) {
  // block = (image, set, chunk of 16 border pixels); thread j < 225 = (shift D, c, c'), threads 225..227 = the plain sums of x_c.
  // (One block per (image, set) walking all 416 pixels serially took 250 us at batch 64: a latency chain of dependent loads.)
  constexpr int kChunk = 16;
  const int chunk = blockIdx.x % chunks, set = (blockIdx.x / chunks) % 8, n = blockIdx.x / (chunks * 8), j = threadIdx.x;
  if (j >= 228) return;
  const long long HW = (long long)H * W;
  const float* xi = x + (long long)n * 3 * HW;
  const int npx = set < 2 ? W : (set < 4 ? H : 1);
  const int k0 = chunk * kChunk, k1 = k0 + kChunk < npx ? k0 + kChunk : npx;
  if (k0 >= npx) return;
  const int di = j / 9, c = j < 225 ? (j % 9) / 3 : j - 225, c2 = j % 3;
  const int dh = di / 5 - 2, dw = di % 5 - 2;
  double a = 0.0;
  for (int k = k0; k < k1; k++) {
    int h, w;
    if (set == 0) { h = 0; w = k; } else if (set == 1) { h = H - 1; w = k; } else if (set == 2) { h = k; w = 0; } else if (set == 3) { h = k; w = W - 1; }
    else { h = (set & 2) ? H - 1 : 0; w = (set & 1) ? W - 1 : 0; }
    const float xv = __ldg(xi + c * HW + (long long)h * W + w);
    if (j >= 225) { a += (double)xv; continue; }
    const int h2 = h + dh, w2 = w + dw;
    if (h2 >= 0 && h2 < H && w2 >= 0 && w2 < W) a += (double)xv * (double)__ldg(xi + c2 * HW + (long long)h2 * W + w2);
  }
  if (a != 0.0) atomicAdd(gram + (j < 225 ? kOffE + set * 225 + j : kOffES1 + set * 3 + (j - 225)), a);
}

__global__ void l0_gram_assemble_kernel(double* __restrict__ gram, double count) {
  for (int i = threadIdx.x; i < kG * kG; i += blockDim.x) {
    const int a = i / kG, b = i % kG;
    if (a > b) continue;
    double v;
    if (a == 27) v = count;
    else {
      const int ta = a / 3, c = a % 3, kh = ta / 3, kw = ta % 3;
      const int eh = kh == 0 ? 1 : (kh == 2 ? 0 : -1), ew = kw == 0 ? 3 : (kw == 2 ? 2 : -1);      // the row / column set tap (kh, kw) never reaches
      const int ec = (eh >= 0 && ew >= 0) ? 4 + (eh == 1 ? 2 : 0) + (ew == 3 ? 1 : 0) : -1;
      if (b == 27) {
        v = gram[kOffT1 + c];
        if (eh >= 0) v -= gram[kOffES1 + eh * 3 + c];
        if (ew >= 0) v -= gram[kOffES1 + ew * 3 + c];
        if (ec >= 0) v += gram[kOffES1 + ec * 3 + c];
      } else {
        const int tb = b / 3, c2 = b % 3, dh = tb / 3 - kh, dw = tb % 3 - kw;
        const bool pos = dh > 0 || (dh == 0 && dw >= 0);
        v = pos ? gram[kOffC + shift_index(dh, dw) * 9 + c * 3 + c2] : gram[kOffC + shift_index(-dh, -dw) * 9 + c2 * 3 + c];
        const int e = ((dh + 2) * 5 + (dw + 2)) * 9 + c * 3 + c2;
        if (eh >= 0) v -= gram[kOffE + eh * 225 + e];
        if (ew >= 0) v -= gram[kOffE + ew * 225 + e];
        if (ec >= 0) v += gram[kOffE + ec * 225 + e];
      }
    }
    gram[i] = v;
  }
}

__device__ __forceinline__ double gram_at(const double* g, int a, int b) { return a <= b ? g[a * kG + b] : g[b * kG + a]; }

// per-channel sum / sum of squares of the (never materialised) conv output from the Gram matrix: the inputs of bn_finalize.
// warp = output channel, lane = Gram row (one 27-term dot product per lane, shuffle reductions; a serial 27 x 27 fp64 loop per thread
// took 35 us of pure latency)
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__global__ void __launch_bounds__(1024) l0_stats_kernel(const double* __restrict__ gram, const float* __restrict__ wgt /*[32][27]*/,
                                                        double* __restrict__ ssum, double* __restrict__ ssq) {
  const int c = threadIdx.x >> 5, a = threadIdx.x & 31;
  double s = 0.0, q = 0.0;
  if (a < 27) {
    const double wa = (double)wgt[c * 27 + a];
    double r = 0.0;
    for (int b = 0; b < 27; b++) r += gram_at(gram, a, b) * (double)wgt[c * 27 + b];
    s = wa * gram_at(gram, a, 27); q = wa * r;
  }
  s = warp_sum_d(s); q = warp_sum_d(q);
  if (a == 0) { ssum[c] = s; ssq[c] = q; }
}

// ------------------------------------------------------------------------------------------------ conv + BN + leaky + 2x2 max-pool
// thread = one 2x2 pixel window x 16 output channels (64 accumulators); channel ownership 8q + 4*half + j, so the two threads of a
// window fill 16 contiguous bytes of every destination row chunk.  One resident block per SM leaves the kernel the whole register
// file (two cap it at 128 registers, with a few spills).
__global__ void __launch_bounds__(256, 1) l0_fused_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wgt /*[32][27]*/,
                                                              const float* __restrict__ scale, const float* __restrict__ shift, float slope,
                                                              int N, int H, int W, uint16_t* __restrict__ d_hi, uint16_t* __restrict__ d_lo,
                                                              int d_ld, int d_c0, uint8_t* __restrict__ code /*[pooled rows][32] or null*/) {
  __shared__ __align__(16) float sw[27][kC0];            // [k][co]
  __shared__ float sin[3][kTH + 2][kInW];
  for (int i = threadIdx.x; i < 27 * kC0; i += 256) sw[i / kC0][i % kC0] = wgt[(i % kC0) * 27 + (i / kC0)];
  const int tiles_w = (W + kTW - 1) / kTW, tiles_h = (H + kTH - 1) / kTH;
  const int ntiles = N * tiles_h * tiles_w;
  const int half = threadIdx.x & 1, wg = threadIdx.x >> 1;
  const int wrow = wg >> 4, wcol = wg & 15;                          // window inside the 8 x 16 window tile
  __shared__ float ssc[kC0], ssh[kC0];                               // BN scale / shift (smem: the 64 accumulators own the registers)
  if (threadIdx.x < kC0) { ssc[threadIdx.x] = scale[threadIdx.x]; ssh[threadIdx.x] = shift[threadIdx.x]; }
  Geom gh{N, H / 2, W / 2};
  float pre[kHaloPer];
  if ((int)blockIdx.x < ntiles) halo_fetch(pre, x, tile_of(blockIdx.x, tiles_h, tiles_w), H, W);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const Tile t = tile_of(tile, tiles_h, tiles_w);
    __syncthreads();
    halo_store(sin, pre);
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) halo_fetch(pre, x, tile_of(tile + gridDim.x, tiles_h, tiles_w), H, W);
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; p++)
#pragma unroll
      for (int j = 0; j < 16; j++) acc[p][j] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      float in[4][4];
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int i = 0; i < 4; i++) in[r][i] = sin[c][2 * wrow + r][2 * wcol + i];
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++) {
          const float* wr = &sw[(dy * 3 + dx) * 3 + c][4 * half];
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const float4 v = *reinterpret_cast<const float4*>(wr + 8 * q);
#pragma unroll
            for (int p = 0; p < 4; p++) {
              const float a = in[(p >> 1) + dy][(p & 1) + dx];
              acc[p][4 * q] = fmaf(a, v.x, acc[p][4 * q]); acc[p][4 * q + 1] = fmaf(a, v.y, acc[p][4 * q + 1]);
              acc[p][4 * q + 2] = fmaf(a, v.z, acc[p][4 * q + 2]); acc[p][4 * q + 3] = fmaf(a, v.w, acc[p][4 * q + 3]);
            }
          }
        }
    }
    const int hs = (t.h0 >> 1) + wrow, ws = (t.w0 >> 1) + wcol;
    if (2 * hs + 1 < H && 2 * ws + 1 < W) {
      const long long row = gh.row(t.n, hs, ws);
      uint32_t cd[4];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        uint16_t hh[4], ll[4];
        uint32_t cq = 0;
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          const int j = 4 * q + jj;
          const float scj = ssc[8 * q + 4 * half + jj], shj = ssh[8 * q + 4 * half + jj];
          // the first maximum of the ACTIVATED values in (h, w) scan order wins (max_pool2d semantics, as bn_apply / bn_bwd)
          float zb = -INFINITY; int best = 0; bool pos = false;
#pragma unroll
          for (int p = 0; p < 4; p++) {
            const float zp = fmaf(acc[p][j], scj, shj);
            const float z = zp > 0.f ? zp : zp * slope;
            if (z > zb) { zb = z; best = p; pos = zp > 0.f; }
          }
          split_f16(zb, hh[jj], ll[jj]);
          cq |= (uint32_t)(best | (pos ? 4 : 0)) << (8 * jj);
        }
        cd[q] = cq;
        const long long o = row * d_ld + d_c0 + 8 * q + 4 * half;
        *reinterpret_cast<uint2*>(d_hi + o) = make_uint2(hh[0] | ((uint32_t)hh[1] << 16), hh[2] | ((uint32_t)hh[3] << 16));
        *reinterpret_cast<uint2*>(d_lo + o) = make_uint2(ll[0] | ((uint32_t)ll[1] << 16), ll[2] | ((uint32_t)ll[3] << 16));
      }
      if (code) {
#pragma unroll
        for (int q = 0; q < 4; q++) *reinterpret_cast<uint32_t*>(code + row * kC0 + 8 * q + 4 * half) = cd[q];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward over the pooled gradient
// t1[k][c] (k < 27) += sum_windows dz * patch(argmax)[k],  t1[27][c] += sum dz      (fp64 accumulators, zeroed by the launcher)
// lane = channel; a warp walks the 16 windows of one window row of the tile.
template <bool G16>      // the pooled gradient plane holds fp16 (SSP_EPI_F16) or fp32 -- compile-time, so that the 16 loads of a window row stay batched
__global__ void __launch_bounds__(256, 2) l0_bwd_kernel(const float* __restrict__ x, const void* __restrict__ g, int g_ld, int g_c0,
                                                        const uint8_t* __restrict__ code, float slope, int N, int H, int W,
                                                        double* __restrict__ t1) {
  __shared__ float sin[3][kTH + 2][kInW];
  __shared__ float sred[8][kG][kC0];
  const int tiles_w = (W + kTW - 1) / kTW, tiles_h = (H + kTH - 1) / kTH;
  const int ntiles = N * tiles_h * tiles_w;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  Geom gh{N, H / 2, W / 2};
  float acc[kG];
#pragma unroll
  for (int k = 0; k < kG; k++) acc[k] = 0.f;
  float pre[kHaloPer];
  if ((int)blockIdx.x < ntiles) halo_fetch(pre, x, tile_of(blockIdx.x, tiles_h, tiles_w), H, W);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const Tile t = tile_of(tile, tiles_h, tiles_w);
    // this warp's window row: all 16 gradient rows (128 B each) and code rows (32 B) are requested before anything waits on them
    const int hs = (t.h0 >> 1) + warp;
    const bool row_ok = 2 * hs + 1 < H;
    float gv[kTW / 2]; int cd[kTW / 2];
    {
      // the 16 pooled cells of a window row are consecutive rows of the pooled plane: one 64-bit row index, then pointer increments
      const int ws0 = t.w0 >> 1;
      const int nw = row_ok ? ((W >> 1) - ws0 < kTW / 2 ? (W >> 1) - ws0 : kTW / 2) : 0;      // windows of this row inside the image
      const long long row0 = row_ok ? gh.row(t.n, hs, ws0) : 0;
      const uint8_t* cp = code + row0 * kC0 + lane;
      const __half* gp16 = reinterpret_cast<const __half*>(g) + row0 * g_ld + g_c0 + lane;
      const float* gp32 = reinterpret_cast<const float*>(g) + row0 * g_ld + g_c0 + lane;
#pragma unroll
      for (int wc = 0; wc < kTW / 2; wc++) {
        const bool ok = wc < nw;                                          // out-of-image windows contribute dz = 0
        if (G16) gv[wc] = ok ? __half2float(__ldg(gp16 + (long long)wc * g_ld)) : 0.f;
        else gv[wc] = ok ? __ldg(gp32 + (long long)wc * g_ld) : 0.f;
        cd[wc] = ok ? (int)__ldg(cp + wc * kC0) : 0;
      }
    }
    __syncthreads();
    halo_store(sin, pre);
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) halo_fetch(pre, x, tile_of(tile + gridDim.x, tiles_h, tiles_w), H, W);
#pragma unroll 4
    for (int wc = 0; wc < kTW / 2; wc++) {
      const float dz = gv[wc] * ((cd[wc] & 4) ? 1.f : slope);
      const int pr = 2 * warp + ((cd[wc] >> 1) & 1), pc = 2 * wc + (cd[wc] & 1);      // arg-max pixel in tile coordinates
#pragma unroll
      for (int k = 0; k < 27; k++) {
        const int c = k % 3, kw = (k / 3) % 3, kh = k / 9;
        acc[k] = fmaf(dz, sin[c][pr + kh][pc + kw], acc[k]);
      }
      acc[27] += dz;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kG; k++) sred[warp][k][lane] = acc[k];
  __syncthreads();
  for (int i = threadIdx.x; i < kG * kC0; i += 256) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++) s += (double)sred[w][i / kC0][i % kC0];
    if (s != 0.0) atomicAdd(t1 + i, s);
  }
}

// dW0, dgamma, dbeta from the sums (header comment); grads are written (not accumulated), `gscale` undoes the loss scale.
// warp = output channel, lane = patch entry k.
__global__ void __launch_bounds__(1024) l0_bwd_finalize_kernel(const double* __restrict__ t1, const double* __restrict__ gram, const float* __restrict__ wgt,
                                                               const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ invstd,
                                                               double count, float gscale, float* __restrict__ dW /*[32][27]*/, float* __restrict__ dgamma,
                                                               float* __restrict__ dbeta) {
  const int c = threadIdx.x >> 5, k = threadIdx.x & 31;
  const double mu = (double)mean[c], is = (double)invstd[c], ga = (double)gamma[c];
  const double S1 = t1[27 * kC0 + c];
  double tk = 0.0, gw = 0.0, cs = 0.0, part = 0.0;
  if (k < 27) {
    tk = t1[k * kC0 + c];
    for (int b = 0; b < 27; b++) gw += gram_at(gram, k, b) * (double)wgt[c * 27 + b];
    cs = gram_at(gram, k, 27);
    part = (double)wgt[c * 27 + k] * tk;
  }
  const double dzy = warp_sum_d(part);
  const double S2 = is * (dzy - mu * S1);
  const double k1 = S1 / count, k2 = S2 / count;
  if (k < 27) dW[c * 27 + k] = (float)(ga * is * (tk - k1 * cs - k2 * is * (gw - mu * cs)) * (double)gscale);
  if (k == 0) { dgamma[c] = (float)(S2 * (double)gscale); dbeta[c] = (float)(S1 * (double)gscale); }
}

// ================================================================================================ host launchers
static int l0_grid(long long ntiles, int per_sm) {
  static int sms = 0;
  if (!sms) sms = ssp_sm_count();
  long long g = (long long)sms * per_sm;
  return (int)(g < ntiles ? g : ntiles);
}
static long long l0_tiles(int N, int H, int W) { return (long long)N * ((H + kTH - 1) / kTH) * ((W + kTW - 1) / kTW); }

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_l0_gram(const float* x, int N, int H, int W, double* gram, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!x || !gram || N <= 0 || H <= 0 || W <= 0) return fail_msg(SSP_ERR_ARG, "l0_gram: bad argument");
  const long long nt = l0_tiles(N, H, W);
  if (nt > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "l0_gram: bad shape");
  cudaError_t e = cudaMemsetAsync(gram, 0, sizeof(double) * kGramDoubles, s);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  if (H < 2 || W < 2) {
    l0_gram_kernel<<<l0_grid(nt, 2), 256, 0, s>>>(x, gram, N, H, W);
    SSP_CHECK_LAUNCH(); return SSP_OK;
  }
  const long long nct = (long long)N * ((H + kCT - 1) / kCT) * ((W + kCT - 1) / kCT);
  l0_corr_kernel<<<l0_grid(nct, 1), 256, 0, s>>>(x, gram, N, H, W);
  const int chunks = ((H > W ? H : W) + 15) / 16;
  l0_border_kernel<<<(unsigned)(8 * N * chunks), 256, 0, s>>>(x, gram, N, H, W, chunks);
  l0_gram_assemble_kernel<<<1, 256, 0, s>>>(gram, (double)N * H * W);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_l0_stats(const double* gram, const float* w, double* ssum, double* ssq, void* stream) {
  if (!gram || !w || !ssum || !ssq) return fail_msg(SSP_ERR_ARG, "l0_stats: bad argument");
  l0_stats_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(gram, w, ssum, ssq);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_l0_fused_fwd(const float* x, const float* w, const float* scale, const float* shift, float slope, int N, int H, int W,
                     void* d_hi, void* d_lo, int d_ld, int d_c0, uint8_t* code, void* stream) {
  if (!x || !w || !scale || !shift || !d_hi || !d_lo || (H & 1) || (W & 1) || (d_ld % 4) || (d_c0 % 4) || d_ld < d_c0 + kC0)
    return fail_msg(SSP_ERR_ARG, "l0_fused_fwd: bad argument (even H / W, destination rows 8-B aligned)");
  const long long nt = l0_tiles(N, H, W);
  if (nt <= 0 || nt > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "l0_fused_fwd: bad shape");
  l0_fused_fwd_kernel<<<l0_grid(nt, 1), 256, 0, (cudaStream_t)stream>>>(x, w, scale, shift, slope, N, H, W, (uint16_t*)d_hi, (uint16_t*)d_lo, d_ld, d_c0, code);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_l0_bwd(const float* x, const void* g, int g_f16, int g_ld, int g_c0, const uint8_t* code, float slope, int N, int H, int W, double* t1,
               void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!x || !g || !code || !t1 || (H & 1) || (W & 1)) return fail_msg(SSP_ERR_ARG, "l0_bwd: bad argument");
  const long long nt = l0_tiles(N, H, W);
  if (nt <= 0 || nt > 0x7fffffffLL) return fail_msg(SSP_ERR_ARG, "l0_bwd: bad shape");
  cudaError_t e = cudaMemsetAsync(t1, 0, sizeof(double) * kG * kC0, s);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  if (g_f16) l0_bwd_kernel<true><<<l0_grid(nt, 2), 256, 0, s>>>(x, g, g_ld, g_c0, code, slope, N, H, W, t1);
  else l0_bwd_kernel<false><<<l0_grid(nt, 2), 256, 0, s>>>(x, g, g_ld, g_c0, code, slope, N, H, W, t1);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_l0_bwd_finalize(const double* t1, const double* gram, const float* w, const float* gamma, const float* mean, const float* invstd,
                        double count, float gscale, float* dW, float* dgamma, float* dbeta, void* stream) {
  if (!t1 || !gram || !w || !gamma || !mean || !invstd || !dW || !dgamma || !dbeta || !(count > 0))
    return fail_msg(SSP_ERR_ARG, "l0_bwd_finalize: bad argument");
  l0_bwd_finalize_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(t1, gram, w, gamma, mean, invstd, count, gscale, dW, dgamma, dbeta);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
