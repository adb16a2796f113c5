// optim.SGD(momentum, dampening=0, weight_decay) of train.py:388 over the flat parameter buffer AND the re-pack of the conv
// weights into the GEMM operand planes, in one pass: the optimiser already touches every weight, so the fp16 forward planes
// (W_hi, W_lo: [cout][tap*cin + ci]) and the transposed, tap-flipped data-gradient plane (W_d: [cin][tap'*cout + co]) are written
// while the updated value is still in a register -- the separate pack_weights launches (23 per step, 0.53 ms, row-strided
// 2-byte stores) disappear.  HBM-bound: 20 B (p, g, v read; p, v written) + 6 B of operand planes per weight.
//
// Work list: a device table of segments, one per parameter tensor in flat-buffer order (ssp_sgd_segment, include/ssp_b200.h).
//   conv weight [cout][taps][cin]  -> blocks of 64(co) x 64(ci) for one tap: fp32 rows of 64 ci are read coalesced, the forward
//                                     planes written in the same order, W_d through a shared-memory transpose (128-B rows both ways)
//   any other tensor (taps == 0)   -> blocks of 1024 consecutive elements
// A launch covers blocks [block_begin, block_end) so that the multi-GPU path can update one gradient bucket at a time as soon as
// its all-reduce has finished.
#include "ssp_common.cuh"

namespace ssp {

struct SgdScalars { float lr, mu, wd, gscale; };

__device__ __forceinline__ float sgd_update(float& p, float g, float& v, const SgdScalars& k) {
  sgd_update(p, g, v, k.lr, k.mu, k.wd, k.gscale);          // ssp_common.cuh: the same FMAs as sgd_flat_kernel
  return p;
}

__global__ void __launch_bounds__(256) sgd_pack_kernel(const ssp_sgd_segment* __restrict__ segs, int n_seg, int block_begin,
                                                       float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v,
                                                       const SgdScalars k) {
  __shared__ uint16_t tile[64][66];                 // [ci][co], 33-word pitch: conflict-free for both access directions
  const int blk = block_begin + (int)blockIdx.x;
  int lo = 0, hi = n_seg - 1;                       // last segment with block0 <= blk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].block0 <= blk) lo = mid; else hi = mid - 1;
  }
  const ssp_sgd_segment sg = segs[lo];
  const int local = blk - sg.block0;
  if (sg.taps == 0) {                               // plain tensor: 4 elements per thread
    const long long i4 = (long long)local * 1024 + threadIdx.x * 4;
    if (i4 >= sg.n) return;
    const long long o = sg.off + i4;
    if (i4 + 3 < sg.n && (o & 3) == 0) {
      float4 pp = *reinterpret_cast<float4*>(p + o);
      const float4 gg = *reinterpret_cast<const float4*>(g + o);
      float4 vv = *reinterpret_cast<float4*>(v + o);
      sgd_update(pp.x, gg.x, vv.x, k); sgd_update(pp.y, gg.y, vv.y, k); sgd_update(pp.z, gg.z, vv.z, k); sgd_update(pp.w, gg.w, vv.w, k);
      *reinterpret_cast<float4*>(v + o) = vv; *reinterpret_cast<float4*>(p + o) = pp;
    } else {
      for (long long i = i4; i < sg.n && i < i4 + 4; i++) { float pv = p[sg.off + i], vv = v[sg.off + i]; sgd_update(pv, g[sg.off + i], vv, k); p[sg.off + i] = pv; v[sg.off + i] = vv; }
    }
    return;
  }
  const int cin = sg.cin, cout = sg.cout, taps = sg.taps;
  const int nci = (cin + 63) >> 6, nco = (cout + 63) >> 6;
  const int cib = local % nci, cob = (local / nci) % nco, tap = local / (nci * nco);
  const int ci0 = cib * 64, co0 = cob * 64;
  const int lane64 = threadIdx.x & 63, grp = threadIdx.x >> 6;      // 4 groups of 64 threads
  uint16_t* f_hi = (uint16_t*)sg.f_hi; uint16_t* f_lo = (uint16_t*)sg.f_lo; uint16_t* d = (uint16_t*)sg.d;
  if ((cin & 3) == 0 && (sg.off & 3) == 0) {
    // vector path: thread = 4 consecutive ci of one (co, tap) row (16-B loads / stores of p, g, v; 8-B stores of the forward planes);
    // 16 threads cover the 64 ci of a row, 16 rows per pass, 4 passes.  (Round 2: the scalar path below moved 1.3 GB in 0.45 ms =
    // 2.9 TB/s; every access was a 4-byte load or a 2-byte store.)
    const int q = threadIdx.x & 15, rr = threadIdx.x >> 4;
    const int ci = ci0 + 4 * q;
    float4 pv[4], gv[4], vv[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int co = co0 + r * 16 + rr;
      pv[r] = gv[r] = vv[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (co < cout && ci < cin) {
        const long long o = sg.off + ((long long)co * taps + tap) * cin + ci;
        pv[r] = *reinterpret_cast<const float4*>(p + o); gv[r] = *reinterpret_cast<const float4*>(g + o); vv[r] = *reinterpret_cast<const float4*>(v + o);
      }
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int co = co0 + r * 16 + rr;
      uint16_t t[4] = {0, 0, 0, 0};
      if (co < cout && ci < cin) {
        const long long o = sg.off + ((long long)co * taps + tap) * cin + ci;
        sgd_update(pv[r].x, gv[r].x, vv[r].x, k); sgd_update(pv[r].y, gv[r].y, vv[r].y, k);
        sgd_update(pv[r].z, gv[r].z, vv[r].z, k); sgd_update(pv[r].w, gv[r].w, vv[r].w, k);
        *reinterpret_cast<float4*>(p + o) = pv[r]; *reinterpret_cast<float4*>(v + o) = vv[r];
        const float w[4] = {pv[r].x, pv[r].y, pv[r].z, pv[r].w};
        if (f_hi) {
          uint16_t a[4], b[4];
#pragma unroll
          for (int j = 0; j < 4; j++) split_f16(w[j], a[j], b[j]);
          const long long of = (long long)co * sg.ld_f + tap * cin + ci;
          if ((of & 3) == 0) {
            *reinterpret_cast<uint2*>(f_hi + of) = make_uint2(a[0] | ((uint32_t)a[1] << 16), a[2] | ((uint32_t)a[3] << 16));
            if (f_lo) *reinterpret_cast<uint2*>(f_lo + of) = make_uint2(b[0] | ((uint32_t)b[1] << 16), b[2] | ((uint32_t)b[3] << 16));
          } else {
#pragma unroll
            for (int j = 0; j < 4; j++) { f_hi[of + j] = a[j]; if (f_lo) f_lo[of + j] = b[j]; }
          }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) t[j] = cvt_f32_to_16(w[j], sg.d_fmt);
      }
#pragma unroll
      for (int j = 0; j < 4; j++) tile[4 * q + j][r * 16 + rr] = t[j];
    }
  } else {
  float pv[16], gv[16], vv[16];
  const int ci = ci0 + lane64;
#pragma unroll
  for (int r = 0; r < 16; r++) {                     // all loads first: 48 independent 4-B loads per thread in flight
    const int co = co0 + r * 4 + grp;
    pv[r] = gv[r] = vv[r] = 0.f;
    if (co < cout && ci < cin) {
      const long long o = sg.off + ((long long)co * taps + tap) * cin + ci;
      pv[r] = p[o]; gv[r] = g[o]; vv[r] = v[o];
    }
  }
#pragma unroll
  for (int r = 0; r < 16; r++) {
    const int co = co0 + r * 4 + grp;
    uint16_t t = 0;
    if (co < cout && ci < cin) {
      const long long o = sg.off + ((long long)co * taps + tap) * cin + ci;
      const float w = sgd_update(pv[r], gv[r], vv[r], k);
      p[o] = w; v[o] = vv[r];
      if (f_hi) {
        uint16_t a, b; split_f16(w, a, b);
        const long long of = (long long)co * sg.ld_f + tap * cin + ci;
        f_hi[of] = a; if (f_lo) f_lo[of] = b;
      }
      t = cvt_f32_to_16(w, sg.d_fmt);
    }
    tile[lane64][r * 4 + grp] = t;
  }
  }
  if (!d) return;
  __syncthreads();
#pragma unroll 4
  for (int r = 0; r < 16; r++) {
    const int cci = ci0 + r * 4 + grp, co = co0 + lane64;           // consecutive threads -> consecutive co: coalesced 16-bit rows
    if (cci < cin && co < cout) d[(long long)cci * sg.ld_d + (long long)(taps - 1 - tap) * cout + co] = tile[r * 4 + grp][lane64];
  }
}

}  // namespace ssp

using namespace ssp;

extern "C" {
// blocks of one segment, in the decomposition sgd_pack_kernel undoes: 1024 elements per block for a plain tensor, one
// 64(ci) x 64(co) tile of one tap per block for a conv weight
int ssp_sgd_segment_blocks(int cout, int taps, int cin, long long n) {
  if (taps == 0) return (int)((n + 1023) / 1024);
  return ((cin + 63) / 64) * ((cout + 63) / 64) * taps;
}

int ssp_sgd_pack_step(const ssp_sgd_segment* segs_dev, int n_seg, int block_begin, int block_end, float* p, const float* g, float* v,
                      float lr, float mu, float wd, float gscale, void* stream) {
  if (!segs_dev || !p || !g || !v || n_seg <= 0 || block_begin < 0 || block_end < block_begin)
    return fail_msg(SSP_ERR_ARG, "sgd_pack_step: bad argument");
  if (block_end == block_begin) return SSP_OK;
  sgd_pack_kernel<<<(unsigned)(block_end - block_begin), 256, 0, (cudaStream_t)stream>>>(segs_dev, n_seg, block_begin, p, g, v,
                                                                                       SgdScalars{lr, mu, wd, gscale});
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
