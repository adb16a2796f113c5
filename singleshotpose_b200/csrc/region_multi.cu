// Multi-object RegionLoss head and decode (yolo-pose-multi.cfg: 5 anchors, 13 classes).
// Restates reference multi_obj_pose_estimation/region_loss_multi.py:9-189 (build_targets with IoU anchor choice, the
// masked MSE terms, CrossEntropy(sum) on the class logits) and utils_multi.py:266-382 (get_multi_region_boxes).
// The reference's "best_n = -1" read (region_loss_multi.py:51,63: tconf is computed from the LAST anchor of the
// PREVIOUS image at the ground-truth cell, wrapping to the last image for b = 0) is reproduced on purpose.
#include "ssp_common.cuh"
#include "eval_multi_core.h"
#include "detect_core.h"

namespace ssp {

#define SSPM_MAX_KP 16
#define SSPM_MAX_GT 50
#define SSPM_MAX_ANCHORS 16

__device__ __forceinline__ float sigmoidm_(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float corner_conf_m(const float* gt, const float* px, const float* py, int K, float eps) {
  const float conf0 = expf(2.f) - 1.f + eps;
  float s = 0.f;
  for (int k = 0; k < K; k++) {
    const float dx = (gt[2 * k] - px[k]) * 640.f, dy = (gt[2 * k + 1] - py[k]) * 480.f;
    const float d = sqrtf(dx * dx + dy * dy);
    if (d < 80.f) s += (expf(2.f * (1.f - d / 80.f)) - 1.f) / conf0;
  }
  return s / (float)K;
}

struct RegionMultiParams {
  const float* out; const float* target; float* grad; double* acc;
  int B, K, nC, nA, H, W;
  float anchors[2 * SSPM_MAX_ANCHORS]; int anchor_step;
  float coord_scale, noobject_scale, object_scale, class_scale, thresh;
  int use_conf; float grad_scale;
};

__global__ void __launch_bounds__(256) region_loss_multi_kernel(const RegionMultiParams p) {
  const int b = blockIdx.x, K = p.K, HW = p.H * p.W, nch = 2 * K + 1 + p.nC, nl = 2 * K + 3;
  __shared__ float s_gt[SSPM_MAX_GT][2 * SSPM_MAX_KP];
  __shared__ float s_tconf[SSPM_MAX_GT];
  __shared__ int s_cell[SSPM_MAX_GT], s_anchor[SSPM_MAX_GT], s_cls[SSPM_MAX_GT], s_valid[SSPM_MAX_GT];
  __shared__ int s_n;
  __shared__ double sred[8][8];
  const float* t = p.target + (long long)b * SSPM_MAX_GT * nl;
  if (threadIdx.x == 0) {
    int n = 0;
    while (n < SSPM_MAX_GT && t[n * nl + 1] != 0.f) n++;       // the list ends at the first x0 == 0 (region_loss_multi.py:31,47)
    s_n = n;
  }
  __syncthreads();
  const int nG = s_n;
  const float* o = p.out + (long long)b * p.nA * nch * HW;
  if (threadIdx.x < nG) {
    const int g = threadIdx.x;
    const float* tg = t + g * nl;
    for (int j = 0; j < 2 * K; j++) s_gt[g][j] = tg[1 + j];
    const int gi0 = (int)(tg[1] * p.W), gj0 = (int)(tg[2] * p.H);
    const bool ok = gi0 >= 0 && gi0 < p.W && gj0 >= 0 && gj0 < p.H;
    s_valid[g] = ok; s_cell[g] = gj0 * p.W + gi0; s_cls[g] = (int)tg[0];
    // anchor by IoU of (gw, gh) against the anchor boxes, both centred at the origin
    const float gw = tg[nl - 2] * p.W, gh = tg[nl - 1] * p.H;
    float best = 0.f; int bn = -1;
    for (int n = 0; n < p.nA; n++) {
      const float aw = p.anchors[p.anchor_step * n], ah = p.anchors[p.anchor_step * n + 1];
      const float mx = fminf(-aw / 2.f, -gw / 2.f), Mx = fmaxf(aw / 2.f, gw / 2.f);
      const float my = fminf(-ah / 2.f, -gh / 2.f), My = fmaxf(ah / 2.f, gh / 2.f);
      const float cw = aw + gw - (Mx - mx), ch = ah + gh - (My - my);
      float iou = 0.f;
      if (cw > 0.f && ch > 0.f) { const float ca = cw * ch; iou = ca / (aw * ah + gw * gh - ca); }
      if (iou > best) { best = iou; bn = n; }
    }
    s_anchor[g] = bn < 0 ? p.nA - 1 : bn;                        // python's [-1] indexing when no anchor overlaps
    float tc = 0.f;
    if (ok) {                                                    // prediction of image b-1 (wrapping), last anchor, same cell
      const int pb = (b + p.B - 1) % p.B;
      const float* op = p.out + ((long long)pb * p.nA + (p.nA - 1)) * nch * HW + s_cell[g];
      float px[SSPM_MAX_KP], py[SSPM_MAX_KP];
      for (int k = 0; k < K; k++) {
        float vx = op[(2 * k) * HW], vy = op[(2 * k + 1) * HW];
        if (k == 0) { vx = sigmoidm_(vx); vy = sigmoidm_(vy); }
        px[k] = (vx + (float)gi0) / (float)p.W; py[k] = (vy + (float)gj0) / (float)p.H;
      }
      tc = corner_conf_m(s_gt[g], px, py, K, 1e-5f);
    }
    s_tconf[g] = tc;
  }
  __syncthreads();
  double part[7] = {0, 0, 0, 0, 0, 0, 0};
  if (threadIdx.x < nG && s_valid[threadIdx.x]) { part[3] = 1.0; if (s_tconf[threadIdx.x] > 0.5f) part[4] = 1.0; }
  float* g = p.grad ? p.grad + (long long)b * p.nA * nch * HW : nullptr;
  for (int i = threadIdx.x; i < p.nA * HW; i += blockDim.x) {
    const int a = i / HW, cell = i % HW, cy = cell / p.W, cx = cell % p.W;
    const float* oa = o + (long long)a * nch * HW + cell;
    float* ga = g ? g + (long long)a * nch * HW + cell : nullptr;
    float xs[SSPM_MAX_KP], ys[SSPM_MAX_KP], px[SSPM_MAX_KP], py[SSPM_MAX_KP];
    for (int k = 0; k < K; k++) {
      float vx = oa[(2 * k) * HW], vy = oa[(2 * k + 1) * HW];
      if (k == 0) { vx = sigmoidm_(vx); vy = sigmoidm_(vy); }
      xs[k] = vx; ys[k] = vy;
      px[k] = (vx + (float)cx) / (float)p.W; py[k] = (vy + (float)cy) / (float)p.H;
    }
    const float conf = sigmoidm_(oa[(2 * K) * HW]);
    if (conf > 0.25f) part[5] += 1.0;
    float conf_mask = p.noobject_scale, tconf = 0.f;
    int sel = -1;
    for (int gidx = 0; gidx < nG; gidx++) {
      if (corner_conf_m(s_gt[gidx], px, py, K, 0.f) > p.thresh) conf_mask = 0.f;
      if (s_valid[gidx] && s_anchor[gidx] == a && s_cell[gidx] == cell) sel = gidx;      // the LAST ground truth on this slot wins
    }
    if (sel >= 0) { conf_mask = p.object_scale; tconf = s_tconf[sel]; }
    for (int k = 0; k < K; k++) {
      float gx = 0.f, gy = 0.f;
      if (sel >= 0) {
        const float tx = s_gt[sel][2 * k] * (float)p.W - (float)cx, ty = s_gt[sel][2 * k + 1] * (float)p.H - (float)cy;
        const float ex = xs[k] - tx, ey = ys[k] - ty;
        part[0] += 0.5 * (double)p.coord_scale * (double)(ex * ex);
        part[1] += 0.5 * (double)p.coord_scale * (double)(ey * ey);
        gx = p.coord_scale * ex; gy = p.coord_scale * ey;
        if (k == 0) { gx *= xs[0] * (1.f - xs[0]); gy *= ys[0] * (1.f - ys[0]); }
      }
      if (ga) { ga[(2 * k) * HW] = gx * p.grad_scale; ga[(2 * k + 1) * HW] = gy * p.grad_scale; }
    }
    const float ec = conf - tconf;
    part[2] += 0.5 * (double)conf_mask * (double)(ec * ec);
    if (ga) ga[(2 * K) * HW] = p.use_conf ? conf_mask * ec * conf * (1.f - conf) * p.grad_scale : 0.f;
    // class term: CrossEntropyLoss(sum) over the selected slots
    if (sel >= 0) {
      float mx = -INFINITY;
      for (int c = 0; c < p.nC; c++) mx = fmaxf(mx, oa[(2 * K + 1 + c) * HW]);
      float den = 0.f;
      for (int c = 0; c < p.nC; c++) den += expf(oa[(2 * K + 1 + c) * HW] - mx);
      const int tc = s_cls[sel];
      const float lt = (tc >= 0 && tc < p.nC) ? oa[(2 * K + 1 + tc) * HW] : 0.f;
      part[6] += (double)p.class_scale * (double)(logf(den) + mx - lt);
      if (ga) for (int c = 0; c < p.nC; c++)
        ga[(2 * K + 1 + c) * HW] = p.class_scale * (expf(oa[(2 * K + 1 + c) * HW] - mx) / den - (c == tc ? 1.f : 0.f)) * p.grad_scale;
    } else if (ga) {
      for (int c = 0; c < p.nC; c++) ga[(2 * K + 1 + c) * HW] = 0.f;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 7; j++) {
    double v = part[j];
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) sred[j][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    double v = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) v += sred[threadIdx.x][w];
    if (v != 0.0) atomicAdd(p.acc + threadIdx.x, v);
  }
}

// ------------------------------------------------------------------------------------------------ decode
// dense pass: for every (image, cell, anchor) -- cell-major, anchor fastest, the reference's visiting order -- the box
// [x0/w, y0/h, ..., det_conf, cls_max_conf, cls_max_id], the selection confidence and softmax[correspondingclass]
// (ssp_evm::decode_entry, the arithmetic eval_multi_select_kernel shares)
__global__ void __launch_bounds__(256) region_decode_multi_kernel(const float* __restrict__ out, int B, int K, int nC, int nA, int H, int W,
                                                                  int only_objectness, int corr, float* __restrict__ boxes,
                                                                  float* __restrict__ conf_sel, float* __restrict__ det, float* __restrict__ cls_corr) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int HW = H * W, nch = 2 * K + 1 + nC;
  if (idx >= (long long)B * HW * nA) return;
  const int a = (int)(idx % nA); const int cell = (int)((idx / nA) % HW); const int b = (int)(idx / ((long long)nA * HW));
  const int cy = cell / W, cx = cell % W;
  const float* o = out + ((long long)b * nA + a) * nch * HW + cell;
  float* bx = boxes + idx * (2 * K + 3);
  const ssp_evm::Decoded d = ssp_evm::decode_entry(o, HW, K, nC, cx, cy, W, H, corr, bx);
  bx[2 * K] = d.det; bx[2 * K + 1] = d.cmax; bx[2 * K + 2] = (float)d.id;
  conf_sel[idx] = only_objectness ? d.det : d.det * d.cmax;
  det[idx] = d.det;
  cls_corr[idx] = d.corr;
}

// the reference's running maxima (max_conf reset per image, max_cls_conf and max_ind never reset): inherently sequential
__global__ void region_decode_multi_fallback_kernel(const float* __restrict__ det, const float* __restrict__ cls_corr, int B, int per_image,
                                                    long long* __restrict__ max_ind, float* __restrict__ max_conf, float* __restrict__ max_cls) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float mcls = -INFINITY; long long mind = -1;
  for (int b = 0; b < B; b++) {
    float mconf = -1.f;
    for (int i = 0; i < per_image; i++) {
      const long long idx = (long long)b * per_image + i;
      if (det[idx] > mconf && cls_corr[idx] > mcls) { mconf = det[idx]; mcls = cls_corr[idx]; mind = idx; }
    }
    max_ind[b] = mind; max_conf[b] = mconf; max_cls[b] = mcls;
  }
}

// ------------------------------------------------------------------------------------------------ evaluation selection
// valid_multi.py:97-132 for every image of a batch, each as the reference's own batch-1 call (rules: eval_multi_core.h).
// One CTA per image: the decode of every (cell, anchor) and the per-class best listed box in parallel (a 64-bit shared
// atomicMax over pick_key, so the result does not depend on the order of the atomics), then thread 0 runs the fallback's
// running maxima (only when needed) and the per-ground-truth choice, then one thread per ground truth writes its box and
// PnP inputs.  Ground truths are taken ssp_evm::kMaxGt at a time; the carried-over choice lives in thread 0's registers.
__global__ void __launch_bounds__(256) eval_multi_select_kernel(const float* __restrict__ out, int B, int K, int nC, int nA, int H, int W,
                                                                const float* __restrict__ target, int stride, const int* __restrict__ gt_offset,
                                                                float thr, float imw, float imh, float* __restrict__ boxes,
                                                                int* __restrict__ flags, float* __restrict__ uv) {
  using namespace ssp_evm;
  const int b = blockIdx.x;
  const int g0 = gt_offset[b], ng = gt_offset[b + 1] - g0, G = gt_offset[B];
  if (ng <= 0) return;
  __shared__ float s_det[kMaxEntries], s_corr[kMaxEntries];
  __shared__ unsigned long long s_best[kMaxClasses];
  __shared__ int s_src[kMaxGt], s_flags[kMaxGt];
  __shared__ Fallback s_fb;
  const int HW = H * W, n = HW * nA, nl = 2 * K + 3;
  const float* t = target + (long long)b * stride;
  const int corr = (int)t[0];
  const float* o = out + (long long)b * nA * (2 * K + 1 + nC) * HW;
  for (int c = threadIdx.x; c < nC; c += blockDim.x) s_best[c] = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int cx, cy;
    const float* oi = entry_ptr(o, i, nA, K, nC, W, HW, &cx, &cy);
    const Decoded d = decode_entry(oi, HW, K, nC, cx, cy, W, H, corr, nullptr);
    s_det[i] = d.det; s_corr[i] = d.corr;
    if (listed(d, thr)) atomicMax(&s_best[d.id], pick_key(d.det, i));
  }
  __syncthreads();
  const bool has_corr = corr >= 0 && corr < nC && s_best[corr] != 0ull;
  if (threadIdx.x == 0) {
    Fallback fb = fallback_init();
    if (!has_corr)
      for (int i = 0; i < n; i++) fallback_update(fb, s_det[i], s_corr[i], i);
    s_fb = fb;
  }
  int src = 0, fl = 0;                                     // thread 0: the previous ground truth's choice
  for (int base = 0; base < ng; base += kMaxGt) {
    const int m = min(kMaxGt, ng - base);
    if (threadIdx.x == 0)
      for (int g = 0; g < m; g++) {
        src = select_box(s_best, nC, corr, has_corr, (int)t[(base + g) * nl], src, fl, &fl);
        s_src[g] = src; s_flags[g] = fl;
      }
    __syncthreads();
    for (int g = threadIdx.x; g < m; g += blockDim.x) {
      const long long gi = g0 + base + g;
      float box[2 * kKeypoints + 3];
      write_box(o, s_src[g], s_fb, corr, nA, K, nC, W, H, box);
      for (int j = 0; j < nl; j++) boxes[gi * nl + j] = box[j];
      flags[gi] = s_flags[g];
      write_uv(t + (base + g) * nl, box, imw, imh, uv + gi * 2 * K, uv + (G + gi) * 2 * K);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ prediction selection
// Slot (image, requested class c) = the box valid_multi.py would choose for a first ground truth of class c (eval_multi_core.h
// predict_slot): every image as its own batch-1 call.  One CTA per image for all requested classes: every (cell, anchor) is
// decoded once (det, and the softmax's mx and den kept in dynamic shared memory) and feeds the per-class best listed box (the
// shared atomicMax over pick_key of eval_multi_select_kernel); then one thread per requested class runs, only when its class
// has no listed box, the fallback's sequential scan over shared memory (softmax[c] recomputed where the scan reads it) and
// writes its slot's box, flag and PnP points.
struct PredictMultiParams {
  const float* out; float* boxes; int* flags; float* uv;
  int K, nC, nA, H, W, n_req;
  float thr, frame_w, frame_h;
  int classes[ssp_evm::kMaxClasses];
};

__global__ void __launch_bounds__(256) predict_multi_select_kernel(const PredictMultiParams p) {
  using namespace ssp_evm;
  extern __shared__ float s_ent[];                          // [3][n]: det, mx, den
  __shared__ unsigned long long s_best[kMaxClasses];
  const int b = blockIdx.x, K = p.K, nC = p.nC, nA = p.nA, W = p.W, H = p.H, HW = H * W, n = HW * nA, nl = 2 * K + 3;
  float* s_det = s_ent; float* s_mx = s_ent + n; float* s_den = s_ent + 2 * n;
  const float* o = p.out + (long long)b * nA * (2 * K + 1 + nC) * HW;
  for (int c = threadIdx.x; c < nC; c += blockDim.x) s_best[c] = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int cx, cy;
    const float* oi = entry_ptr(o, i, nA, K, nC, W, HW, &cx, &cy);
    const Decoded d = decode_entry(oi, HW, K, nC, cx, cy, W, H, -1, nullptr);
    s_det[i] = d.det; s_mx[i] = d.mx; s_den[i] = d.den;
    if (listed(d, p.thr)) atomicMax(&s_best[d.id], pick_key(d.det, i));
  }
  __syncthreads();
  for (int q = threadIdx.x; q < p.n_req; q += blockDim.x) {
    const int c = p.classes[q];
    int fl;
    const int src = predict_slot(s_best, nC, c, &fl);
    const Fallback fb = src == kSrcFallback ? fallback_scan(o, s_det, s_mx, s_den, n, c, nA, K, nC, W, HW) : fallback_init();
    const long long slot = (long long)b * p.n_req + q;
    float box[2 * kKeypoints + 3];
    write_box(o, src, fb, c, nA, K, nC, W, H, box);
    for (int j = 0; j < nl; j++) p.boxes[slot * nl + j] = box[j];
    p.flags[slot] = fl;
    for (int k = 0; k < kKeypoints; k++) box_uv(box, p.frame_w, p.frame_h, k, p.uv + slot * 2 * kKeypoints);
  }
}

// ------------------------------------------------------------------------------------------------ every instance
// ssp_detect_instances: the candidates, order and class-wise greedy suppression of detect_core.h, every image as its own call.
// One CTA per image.  Every (cell, anchor) is decoded once; a candidate leaves its rectangle and class in shared memory (indexed by
// entry) and its pick_key in a list whose bitonic sort (descending, zero-padded to a power of two) gives the key order whatever
// order the atomics appended in.  The greedy pass runs one warp per requested class: the warp walks the sorted list, and each
// of its class's candidates is tested against the class's kept boxes 32 at a time (a ballot decides).  A block-wide scan of
// the keep flags in key order then gives each kept box its output slot; the first max_instances are written (the box
// re-decoded by write_box, as the multi-object predictor writes its slots) and the rest of the slots are zeroed.
constexpr int kDetectThreads = 512;

struct DetectParams {
  const float* out; float* boxes; int* cls; float* uv; int* count; int* kept;
  int K, nC, nA, H, W, n_req, max_inst;
  float thr, nms, frame_w, frame_h;
  int classes[ssp_evm::kMaxClasses];
};

__host__ __device__ inline int pow2_at_least(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// dynamic shared memory of an image of n entries: keys [pow2(n)] u64, rectangles [n], kept entries [n] int, keep flags and
// classes [n] bytes each
__host__ __device__ inline int detect_smem_bytes(int n) {
  return pow2_at_least(n) * 8 + n * (int)sizeof(ssp_det::Rect) + n * 4 + 2 * n;
}

__global__ void __launch_bounds__(kDetectThreads) detect_instances_kernel(const DetectParams p) {
  using namespace ssp_evm;
  using ssp_det::Rect;
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ unsigned char s_req[kMaxClasses];
  __shared__ int s_off[kMaxClasses];                      // candidates per class, then the class's offset into s_kidx
  __shared__ int s_ncand;
  __shared__ int s_wsum[kDetectThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, K = p.K, nC = p.nC, nA = p.nA, W = p.W, H = p.H, HW = H * W, n = HW * nA;
  const int nl = 2 * K + 3, M = p.max_inst;
  unsigned long long* s_key = reinterpret_cast<unsigned long long*>(s_raw);
  Rect* s_rect = reinterpret_cast<Rect*>(s_key + pow2_at_least(n));
  int* s_kidx = reinterpret_cast<int*>(s_rect + n);
  unsigned char* s_keep = reinterpret_cast<unsigned char*>(s_kidx + n);
  unsigned char* s_ecls = s_keep + n;
  const float* o = p.out + (long long)b * nA * (2 * K + 1 + nC) * HW;
  for (int c = tid; c < nC; c += blockDim.x) { s_req[c] = 0; s_off[c] = 0; }
  if (tid == 0) s_ncand = 0;
  __syncthreads();
  for (int q = tid; q < p.n_req; q += blockDim.x) s_req[p.classes[q]] = 1;
  __syncthreads();
  for (int t = tid; t < n; t += blockDim.x) {
    const int a = t / HW, cell = t - a * HW, i = cell * nA + a;   // cells fastest across threads; i is the visiting order
    float kp[2 * kKeypoints];
    const Decoded d = decode_entry(o + (long long)a * (2 * K + 1 + nC) * HW + cell, HW, K, nC, cell % W, cell / W, W, H, -1, kp);
    if (ssp_det::candidate(d, p.thr, s_req)) {
      float uv[2 * kKeypoints];
      s_rect[i] = ssp_det::entry_rect(kp, p.frame_w, p.frame_h, uv);
      s_ecls[i] = (unsigned char)d.id;
      atomicAdd(&s_off[d.id], 1);
      s_key[atomicAdd(&s_ncand, 1)] = pick_key(d.det, i);
    }
  }
  __syncthreads();
  const int m = s_ncand, P = pow2_at_least(m);
  for (int j = m + tid; j < P; j += blockDim.x) s_key[j] = 0ull;   // keys are never 0: the padding sorts last
  if (tid == 0)
    for (int c = 0, s = 0; c < nC; c++) { const int h = s_off[c]; s_off[c] = s; s += h; }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < P; t += blockDim.x) {
        const int u = t ^ j;
        if (u > t) {
          const unsigned long long x = s_key[t], y = s_key[u];
          if ((t & k) == 0 ? x < y : x > y) { s_key[t] = y; s_key[u] = x; }
        }
      }
      __syncthreads();
    }
  const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int q = warp; q < p.n_req; q += nw) {
    const int c = p.classes[q];
    int* kl = s_kidx + s_off[c];                            // kept entries of class c, in key order
    int nk = 0;
    for (int j0 = 0; j0 < m; j0 += 32) {
      const int j = j0 + lane;
      const int e = j < m ? key_index(s_key[j]) : 0;
      unsigned mine = __ballot_sync(0xffffffffu, j < m && s_ecls[e] == c);
      while (mine) {
        const int src = __ffs(mine) - 1;
        mine &= mine - 1;
        const int ej = __shfl_sync(0xffffffffu, e, src);
        const Rect r = s_rect[ej];
        bool sup = false;
        for (int k = lane; k < nk && !sup; k += 32) sup = ssp_det::suppresses(s_rect[kl[k]], r, p.nms);
        const bool keep = !__any_sync(0xffffffffu, sup);
        if (lane == 0) { s_keep[j0 + src] = keep; if (keep) kl[nk] = ej; }
        nk += keep;
        __syncwarp();
      }
    }
  }
  __syncthreads();
  int base = 0;                                             // kept boxes before the current chunk (the same in every thread)
  for (int j0 = 0; j0 < m; j0 += blockDim.x) {
    const int j = j0 + tid;
    const bool f = j < m && s_keep[j];
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_wsum[warp] = __popc(bal);
    __syncthreads();
    int rank = base + __popc(bal & ((1u << lane) - 1u)), total = 0;
    for (int w = 0; w < nw; w++) { if (w < warp) rank += s_wsum[w]; total += s_wsum[w]; }
    if (f && rank < M) {
      const long long slot = (long long)b * M + rank;
      float box[2 * kKeypoints + 3];
      write_box(o, key_index(s_key[j]), fallback_init(), -1, nA, K, nC, W, H, box);
      for (int v = 0; v < nl; v++) p.boxes[slot * nl + v] = box[v];
      p.cls[slot] = (int)box[2 * K + 2];
      for (int k = 0; k < kKeypoints; k++) box_uv(box, p.frame_w, p.frame_h, k, p.uv + slot * 2 * kKeypoints);
    }
    base += total;
    __syncthreads();
  }
  const int cnt = min(base, M);
  for (int r = cnt + tid; r < M; r += blockDim.x) {
    const long long slot = (long long)b * M + r;
    for (int v = 0; v < nl; v++) p.boxes[slot * nl + v] = 0.f;
    for (int v = 0; v < 2 * kKeypoints; v++) p.uv[slot * 2 * kKeypoints + v] = 0.f;
    p.cls[slot] = -1;
  }
  if (tid == 0) { p.count[b] = cnt; p.kept[b] = base; }
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_detect_instances(const float* out, int B, int K, int nC, int nA, int H, int W, const int* classes_host, int n_req, float conf_thresh,
                         float nms_thresh, int max_instances, float frame_w, float frame_h, float* boxes, int* cls, float* uv, int* count,
                         int* kept, void* stream) {
  if (!out || !classes_host || !boxes || !cls || !uv || !count || !kept) return fail_msg(SSP_ERR_ARG, "detect_instances: null pointer");
  if (K != ssp_evm::kKeypoints)
    return fail_msg(SSP_ERR_ARG, "detect_instances: num_keypoints must be 9 (the overlap box is the 8 corners of a pose box)");
  if (B < 0 || nC < 1 || nA < 1 || H < 1 || W < 1) return fail_msg(SSP_ERR_ARG, "detect_instances: bad argument");
  if ((long long)H * W * nA > ssp_evm::kMaxEntries)
    return fail_msg(SSP_ERR_ARG, "detect_instances: grid too large (H*W*num_anchors must be at most 4096, e.g. 26x26x5)");
  if (nC > ssp_evm::kMaxClasses) return fail_msg(SSP_ERR_ARG, "detect_instances: at most 256 classes");
  if (n_req < 1 || n_req > nC) return fail_msg(SSP_ERR_ARG, "detect_instances: n_req must be in [1, num_classes]");
  if (!(nms_thresh >= 0.f && nms_thresh <= 1.f)) return fail_msg(SSP_ERR_ARG, "detect_instances: nms_thresh must be in [0, 1]");
  if (max_instances < 1 || max_instances > ssp_det::kMaxInstances)
    return fail_msg(SSP_ERR_ARG, "detect_instances: max_instances must be in [1, 256]");
  DetectParams p;
  bool seen[ssp_evm::kMaxClasses] = {};
  for (int q = 0; q < n_req; q++) {
    const int c = classes_host[q];
    if (c < 0 || c >= nC) return fail_msg(SSP_ERR_ARG, "detect_instances: requested class out of [0, num_classes)");
    if (seen[c]) return fail_msg(SSP_ERR_ARG, "detect_instances: requested class listed twice");
    seen[c] = true; p.classes[q] = c;
  }
  if (B == 0) return SSP_OK;
  static int configured = 0;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(detect_instances_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               detect_smem_bytes(ssp_evm::kMaxEntries));
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  p.out = out; p.boxes = boxes; p.cls = cls; p.uv = uv; p.count = count; p.kept = kept;
  p.K = K; p.nC = nC; p.nA = nA; p.H = H; p.W = W; p.n_req = n_req; p.max_inst = max_instances;
  p.thr = conf_thresh; p.nms = nms_thresh; p.frame_w = frame_w; p.frame_h = frame_h;
  detect_instances_kernel<<<B, kDetectThreads, detect_smem_bytes(H * W * nA), (cudaStream_t)stream>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_predict_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const int* classes_host, int n_req, float conf_thresh,
                             float frame_w, float frame_h, float* boxes, int* flags, float* uv, void* stream) {
  if (!out || !classes_host || !boxes || !flags || !uv) return fail_msg(SSP_ERR_ARG, "predict_multi_select: null pointer");
  if (K != ssp_evm::kKeypoints)
    return fail_msg(SSP_ERR_ARG, "predict_multi_select: num_keypoints must be 9 (the PnP points are the 9 keypoints of a box)");
  if (B < 0 || nC < 1 || nA < 1 || H < 1 || W < 1) return fail_msg(SSP_ERR_ARG, "predict_multi_select: bad argument");
  if ((long long)H * W * nA > ssp_evm::kMaxEntries)
    return fail_msg(SSP_ERR_ARG, "predict_multi_select: grid too large (H*W*num_anchors must be at most 4096, e.g. 26x26x5)");
  if (nC > ssp_evm::kMaxClasses) return fail_msg(SSP_ERR_ARG, "predict_multi_select: at most 256 classes");
  if (n_req < 1 || n_req > nC) return fail_msg(SSP_ERR_ARG, "predict_multi_select: n_req must be in [1, num_classes]");
  PredictMultiParams p;
  bool seen[ssp_evm::kMaxClasses] = {};
  for (int q = 0; q < n_req; q++) {
    const int c = classes_host[q];
    if (c < 0 || c >= nC) return fail_msg(SSP_ERR_ARG, "predict_multi_select: requested class out of [0, num_classes)");
    if (seen[c]) return fail_msg(SSP_ERR_ARG, "predict_multi_select: requested class listed twice");
    seen[c] = true; p.classes[q] = c;
  }
  if (B == 0) return SSP_OK;
  static int configured = 0;
  const int smem = 3 * H * W * nA * (int)sizeof(float);
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(predict_multi_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               3 * ssp_evm::kMaxEntries * (int)sizeof(float));
    if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
    configured = 1;
  }
  p.out = out; p.boxes = boxes; p.flags = flags; p.uv = uv;
  p.K = K; p.nC = nC; p.nA = nA; p.H = H; p.W = W; p.n_req = n_req;
  p.thr = conf_thresh; p.frame_w = frame_w; p.frame_h = frame_h;
  predict_multi_select_kernel<<<B, 256, smem, (cudaStream_t)stream>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_eval_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const float* target, int target_stride,
                          const int* gt_offset, float conf_thresh, float im_width, float im_height, float* boxes, int* flags, float* uv,
                          void* stream) {
  if (K != ssp_evm::kKeypoints)
    return fail_msg(SSP_ERR_ARG, "eval_multi_select: num_keypoints must be 9 (fix_corner_order is defined for the 9 keypoints of a box)");
  if (!out || !target || !gt_offset || !boxes || !flags || !uv || B < 0 || nC < 1 || nA < 1 || H < 1 || W < 1 || target_stride < 2 * K + 3)
    return fail_msg(SSP_ERR_ARG, "eval_multi_select: bad argument");
  if ((long long)H * W * nA > ssp_evm::kMaxEntries)
    return fail_msg(SSP_ERR_ARG, "eval_multi_select: grid too large (H*W*num_anchors must be at most 4096, e.g. 26x26x5)");
  if (nC > ssp_evm::kMaxClasses) return fail_msg(SSP_ERR_ARG, "eval_multi_select: at most 256 classes");
  if (B == 0) return SSP_OK;
  eval_multi_select_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(out, B, K, nC, nA, H, W, target, target_stride, gt_offset, conf_thresh, im_width,
                                                              im_height, boxes, flags, uv);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_region_loss_multi_fwd_bwd(const float* out, const float* target, float* grad, double* acc, int B, int K, int nC, int nA, int H, int W,
                                  const float* anchors_host, int anchor_step, float coord_scale, float noobject_scale, float object_scale,
                                  float class_scale, float thresh, int use_conf, float grad_scale, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!out || !target || !acc || !anchors_host || K < 1 || K > SSPM_MAX_KP || nA < 1 || nA > SSPM_MAX_ANCHORS || anchor_step < 2)
    return fail_msg(SSP_ERR_ARG, "region_loss_multi_fwd_bwd: bad argument");
  cudaError_t e = cudaMemsetAsync(acc, 0, 8 * sizeof(double), s);
  if (e != cudaSuccess) return fail_cuda(e, __FILE__, __LINE__);
  RegionMultiParams p;
  p.out = out; p.target = target; p.grad = grad; p.acc = acc; p.B = B; p.K = K; p.nC = nC; p.nA = nA; p.H = H; p.W = W;
  for (int i = 0; i < 2 * SSPM_MAX_ANCHORS; i++) p.anchors[i] = (i < nA * anchor_step && i < 2 * SSPM_MAX_ANCHORS) ? anchors_host[i] : 0.f;
  p.anchor_step = anchor_step; p.coord_scale = coord_scale; p.noobject_scale = noobject_scale; p.object_scale = object_scale;
  p.class_scale = class_scale; p.thresh = thresh; p.use_conf = use_conf; p.grad_scale = grad_scale;
  region_loss_multi_kernel<<<B, 256, 0, s>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_region_decode_multi(const float* out, int B, int K, int nC, int nA, int H, int W, int only_objectness, int corr, float* boxes,
                            float* conf_sel, float* det, float* cls_corr, long long* max_ind, float* max_conf, float* max_cls, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!out || !boxes || !conf_sel || !det || !cls_corr || !max_ind || !max_conf || !max_cls || K < 1 || K > SSPM_MAX_KP)
    return fail_msg(SSP_ERR_ARG, "region_decode_multi: bad argument");
  const long long total = (long long)B * H * W * nA;
  region_decode_multi_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(out, B, K, nC, nA, H, W, only_objectness, corr, boxes, conf_sel, det, cls_corr);
  SSP_CHECK_LAUNCH();
  region_decode_multi_fallback_kernel<<<1, 32, 0, s>>>(det, cls_corr, B, H * W * nA, max_ind, max_conf, max_cls);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
