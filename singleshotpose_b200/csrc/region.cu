// RegionLoss head (single-object) as ONE kernel: activation, predicted-corner decode, build_targets, masked
// MSE terms, their gradient w.r.t. the raw network output and the log counters -- no host round trip.
// Restates reference region_loss.py:9-78 (build_targets) and :95-175 (RegionLoss.forward) plus
// utils.py:138-187 (corner_confidences / corner_confidence); gradients as derived in SURVEY.md 8a (a9).
// Also the detection decode of utils.py:216-296 (get_region_boxes) as a device arg-max.
#include "ssp_common.cuh"

namespace ssp {

#define SSP_MAX_KP 16

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// mean over keypoints of  (exp(2(1-d/80)) - 1) / (e^2 - 1 [+eps])  for pixel distance d < 80 (640x480 image)
__device__ __forceinline__ float corner_conf(const float* gt, const float* px, const float* py, int K, float eps) {
  const float conf0 = expf(2.f) - 1.f + eps;
  float s = 0.f;
  for (int k = 0; k < K; k++) {
    const float dx = (gt[2 * k] - px[k]) * 640.f, dy = (gt[2 * k + 1] - py[k]) * 480.f;
    const float d = sqrtf(dx * dx + dy * dy);
    if (d < 80.f) s += (expf(2.f * (1.f - d / 80.f)) - 1.f) / conf0;
  }
  return s / (float)K;
}

struct RegionParams {
  const float* out;      // (B, 2K+1+nC, H, W) fp32 NCHW, raw conv output
  const float* target;   // (B, 50*(2K+3)) fp32
  float* grad;           // same shape as out (may be null)
  double* acc;           // [8]: loss_x, loss_y, loss_conf, nGT, nCorrect, nProposals, -, -
  int B, K, nC, H, W;
  float coord_scale, noobject_scale, object_scale, thresh;
  int use_conf;          // epoch > pretrain_num_epochs
  float grad_scale;
};

__global__ void __launch_bounds__(256) region_loss_kernel(const RegionParams p) {
  const int b = blockIdx.x;
  const int K = p.K, HW = p.H * p.W, nch = 2 * K + 1 + p.nC;
  __shared__ float gt[2 * SSP_MAX_KP];
  __shared__ int s_has, s_gi, s_gj;
  __shared__ double sred[8][8];
  const float* t = p.target + (long long)b * 50 * (2 * K + 3);
  if (threadIdx.x == 0) {
    s_has = (t[1] != 0.f) ? 1 : 0;
    s_gi = (int)(t[1] * p.W); s_gj = (int)(t[2] * p.H);
    if (s_gi < 0 || s_gi >= p.W || s_gj < 0 || s_gj >= p.H) s_has = 0;
  }
  if (threadIdx.x < 2 * K) gt[threadIdx.x] = t[1 + threadIdx.x];
  __syncthreads();
  const float* o = p.out + (long long)b * nch * HW;
  float* g = p.grad ? p.grad + (long long)b * nch * HW : nullptr;
  double part[6] = {0, 0, 0, 0, 0, 0};
  if (threadIdx.x == 0 && s_has) part[3] = 1.0;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const int cy = i / p.W, cx = i % p.W;
    float xs[SSP_MAX_KP], ys[SSP_MAX_KP], px[SSP_MAX_KP], py[SSP_MAX_KP];
    for (int k = 0; k < K; k++) {
      float vx = o[(2 * k) * HW + i], vy = o[(2 * k + 1) * HW + i];
      if (k == 0) { vx = sigmoidf_(vx); vy = sigmoidf_(vy); }
      xs[k] = vx; ys[k] = vy;
      px[k] = (vx + (float)cx) / (float)p.W; py[k] = (vy + (float)cy) / (float)p.H;
    }
    const float conf = sigmoidf_(o[(2 * K) * HW + i]);
    if (conf > 0.25f) part[5] += 1.0;
    float conf_mask = p.noobject_scale, tconf = 0.f;
    bool is_gt = false;
    if (s_has) {
      if (corner_conf(gt, px, py, K, 0.f) > p.thresh) conf_mask = 0.f;       // region_loss.py:38-40
      if (cx == s_gi && cy == s_gj) {                                          // region_loss.py:59-76
        is_gt = true;
        conf_mask = p.object_scale;
        tconf = corner_conf(gt, px, py, K, 1e-5f);
        if (tconf > 0.5f) part[4] += 1.0;
      }
    }
    for (int k = 0; k < K; k++) {
      float gx = 0.f, gy = 0.f;
      if (is_gt) {
        const float tx = gt[2 * k] * (float)p.W - (float)s_gi, ty = gt[2 * k + 1] * (float)p.H - (float)s_gj;
        const float ex = xs[k] - tx, ey = ys[k] - ty;
        part[0] += 0.5 * (double)p.coord_scale * (double)(ex * ex);
        part[1] += 0.5 * (double)p.coord_scale * (double)(ey * ey);
        gx = p.coord_scale * ex; gy = p.coord_scale * ey;
        if (k == 0) { gx *= xs[0] * (1.f - xs[0]); gy *= ys[0] * (1.f - ys[0]); }
      }
      if (g) { g[(2 * k) * HW + i] = gx * p.grad_scale; g[(2 * k + 1) * HW + i] = gy * p.grad_scale; }
    }
    const float ec = conf - tconf;
    part[2] += 0.5 * (double)conf_mask * (double)(ec * ec);
    if (g) {
      g[(2 * K) * HW + i] = p.use_conf ? conf_mask * ec * conf * (1.f - conf) * p.grad_scale : 0.f;
      for (int c = 0; c < p.nC; c++) g[(2 * K + 1 + c) * HW + i] = 0.f;
    }
  }
  // block reduction of the 6 partials
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    double v = part[j];
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) sred[j][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) v += sred[threadIdx.x][w];
    if (v != 0.0) atomicAdd(p.acc + threadIdx.x, v);
  }
}

// ------------------------------------------------------------------------------------------------
// get_region_boxes (utils.py:216-296): per-image arg-max of the objectness (strict '>' keeps the first
// maximum in (cy, cx) order), then the reference's whole-batch arg-max on top (max_conf never reset).
// box = [x0/w, y0/h, ..., x8/w, y8/h, det_conf, cls_max_conf, cls_max_id]
__global__ void __launch_bounds__(256) region_decode_kernel(const float* __restrict__ out, int B, int K, int nC, int H, int W,
                                                            int only_objectness, float* __restrict__ boxes /*[B][2K+3]*/,
                                                            float* __restrict__ best_conf /*[B]*/) {
  const int b = blockIdx.x, HW = H * W, nch = 2 * K + 1 + nC;
  const float* o = out + (long long)b * nch * HW;
  __shared__ float sv[256]; __shared__ int si[256];
  float bv = -INFINITY; int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    float conf = sigmoidf_(o[(2 * K) * HW + i]);
    if (!only_objectness) {
      float mx = -INFINITY; for (int c = 0; c < nC; c++) mx = fmaxf(mx, o[(2 * K + 1 + c) * HW + i]);
      float den = 0.f, best = 0.f; for (int c = 0; c < nC; c++) { const float e = expf(o[(2 * K + 1 + c) * HW + i] - mx); den += e; best = fmaxf(best, e); }
      conf *= best / den;
    }
    if (conf > bv) { bv = conf; bi = i; }     // ascending i per thread: first max kept
  }
  sv[threadIdx.x] = bv; si[threadIdx.x] = bi;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const float v2 = sv[threadIdx.x + s]; const int i2 = si[threadIdx.x + s];
      if (v2 > sv[threadIdx.x] || (v2 == sv[threadIdx.x] && i2 < si[threadIdx.x])) { sv[threadIdx.x] = v2; si[threadIdx.x] = i2; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int i = si[0] == 0x7fffffff ? 0 : si[0], cy = i / W, cx = i % W;     // every confidence NaN: decode cell 0 instead of reading out of bounds
    float* bx = boxes + (long long)b * (2 * K + 3);
    for (int k = 0; k < K; k++) {
      float vx = o[(2 * k) * HW + i], vy = o[(2 * k + 1) * HW + i];
      if (k == 0) { vx = sigmoidf_(vx); vy = sigmoidf_(vy); }
      bx[2 * k] = (vx + (float)cx) / (float)W; bx[2 * k + 1] = (vy + (float)cy) / (float)H;
    }
    float mx = -INFINITY; int id = 0;
    for (int c = 0; c < nC; c++) { const float v = o[(2 * K + 1 + c) * HW + i]; if (v > mx) { mx = v; id = c; } }
    float den = 0.f; for (int c = 0; c < nC; c++) den += expf(o[(2 * K + 1 + c) * HW + i] - mx);
    bx[2 * K] = sigmoidf_(o[(2 * K) * HW + i]);
    bx[2 * K + 1] = 1.f / den;
    bx[2 * K + 2] = (float)id;
    best_conf[b] = sv[0];
  }
}

__global__ void region_pick_global_kernel(const float* __restrict__ boxes, const float* __restrict__ best_conf, int B, int nv,
                                          float* __restrict__ box_out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int bb = 0; float bv = best_conf[0];
    for (int b = 1; b < B; b++) if (best_conf[b] > bv) { bv = best_conf[b]; bb = b; }
    for (int j = 0; j < nv; j++) box_out[j] = boxes[(long long)bb * nv + j];
  }
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_region_loss_fwd_bwd(const float* out, const float* target, float* grad, double* acc, int B, int K, int nC, int H, int W,
                            float coord_scale, float noobject_scale, float object_scale, float thresh, int use_conf,
                            float grad_scale, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!out || !target || !acc || K < 1 || K > SSP_MAX_KP) return fail_msg(SSP_ERR_ARG, "region_loss_fwd_bwd: bad argument");
  cudaError_t e = cudaMemsetAsync(acc, 0, 8 * sizeof(double), s);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  RegionParams p{out, target, grad, acc, B, K, nC, H, W, coord_scale, noobject_scale, object_scale, thresh, use_conf, grad_scale};
  region_loss_kernel<<<B, 256, 0, s>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_region_decode_argmax(const float* out, int B, int K, int nC, int H, int W, int only_objectness,
                             float* boxes, float* best_conf, float* box_global, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!out || !boxes || !best_conf || K < 1 || K > SSP_MAX_KP) return fail_msg(SSP_ERR_ARG, "region_decode_argmax: bad argument");
  region_decode_kernel<<<B, 256, 0, s>>>(out, B, K, nC, H, W, only_objectness, boxes, best_conf);
  SSP_CHECK_LAUNCH();
  if (box_global) { region_pick_global_kernel<<<1, 32, 0, s>>>(boxes, best_conf, B, 2 * K + 3, box_global); SSP_CHECK_LAUNCH(); }
  return SSP_OK;
}
}  // extern "C"
