// Multi-object decode arithmetic and the evaluation loop's selection rules (reference multi_obj_pose_estimation/utils_multi.py:266-382
// and valid_multi.py:97-149), shared by the CUDA kernels of region_multi.cu and the CPU test harness
// (tests/helpers/eval_multi_host.cpp, built with g++).
//
// Per image (the reference evaluates with batch size 1, so every rule below restarts with each image):
//   * the box list holds every (cell, anchor) with det_conf * cls_max_conf > conf_thresh, in the visiting order (cy, cx, anchor);
//   * a fallback box for correspondingclass = int(target[0]) (the image's first ground-truth class) is appended when no listed box
//     has that class; it takes the keypoints of the running-maximum entry (det > max_conf && cls_corr > max_cls_conf, visited in
//     the same order, max_conf = -1 and max_cls_conf = -inf at the start) and [max_conf, max_cls_conf, correspondingclass];
//   * ground truth k of class c takes the first box in list order whose det_conf is strictly greater than every earlier one among
//     the boxes of class c -- the largest (det bits, ~list index) key, which orders like (det, -index) because det >= 0;
//     when no box has class c it keeps the box of the previous ground truth of the image;
//   * the PnP inputs are the box keypoints times (im_width, im_height) in fp32; the ground truth goes through fix_corner_order.
// The predictor (predict_multi_select_kernel, tests/helpers/predict_multi_host.cpp) applies the same rules without labels: one
// slot per (image, requested class), chosen as for a first ground truth of that class (predict_slot, fallback_scan).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#if defined(__CUDACC__)
#define SSP_EVM_HD __host__ __device__ __forceinline__
#else
#define SSP_EVM_HD inline
#endif

namespace ssp_evm {

constexpr int kKeypoints = 9;         // fix_corner_order (utils_multi.py:244-255) is written for the 9 keypoints of a box
constexpr int kMaxEntries = 4096;     // H*W*num_anchors of one image the select kernel keeps in shared memory (26x26x5 = 3380)
constexpr int kMaxClasses = 256;
constexpr int kMaxGt = 50;            // rows of a label (dataset_multi.py max_num_gt)
constexpr int kSrcFallback = -1;      // select(): the image's fallback box
constexpr int kFlagFallback = 1, kFlagCarried = 2;

// utils_multi.py:244-255: corrected[dst] = label[fix_order(dst)], i.e. {0, 1, 3, 5, 7, 2, 4, 6, 8}
SSP_EVM_HD int fix_order(int dst) { return dst == 0 ? 0 : dst <= 4 ? 2 * dst - 1 : 2 * (dst - 4); }

SSP_EVM_HD float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

struct Decoded {
  float det;    // sigmoid(objectness)
  float cmax;   // max softmax
  float corr;   // softmax at correspondingclass (0 when it is out of range)
  int id;       // arg-max class (first maximum)
  float mx, den;  // the softmax's largest class logit and denominator (class_prob)
};

// softmax[c] of one (cell, anchor) from its decode's mx and den: the arithmetic of Decoded::corr
SSP_EVM_HD float class_prob(const float* o, int HW, int K, int c, float mx, float den) { return expf(o[(2 * K + 1 + c) * HW] - mx) / den; }

// one (cell, anchor): o points at channel 0 of that anchor at the cell, channels HW apart.  kp (2K floats, or null) receives
// [x0/W, y0/H, ..., x_{K-1}/W, y_{K-1}/H].  The arithmetic of the reference's decode, in this order, for every kernel.
SSP_EVM_HD Decoded decode_entry(const float* o, int HW, int K, int nC, int cx, int cy, int W, int H, int corr, float* kp) {
  if (kp)
    for (int k = 0; k < K; k++) {
      float vx = o[(2 * k) * HW], vy = o[(2 * k + 1) * HW];
      if (k == 0) { vx = sigmoid(vx); vy = sigmoid(vy); }
      kp[2 * k] = (vx + (float)cx) / (float)W; kp[2 * k + 1] = (vy + (float)cy) / (float)H;
    }
  Decoded d;
  d.det = sigmoid(o[(2 * K) * HW]);
  float mx = -INFINITY; int id = 0;
  for (int c = 0; c < nC; c++) { const float v = o[(2 * K + 1 + c) * HW]; if (v > mx) { mx = v; id = c; } }
  float den = 0.f;
  for (int c = 0; c < nC; c++) den += expf(o[(2 * K + 1 + c) * HW] - mx);
  d.cmax = 1.f / den;
  d.id = id;
  d.corr = (corr >= 0 && corr < nC) ? class_prob(o, HW, K, corr, mx, den) : 0.f;
  d.mx = mx; d.den = den;
  return d;
}

// entry i of an image in visiting order (cell-major, anchor fastest) -> pointer to its channel 0 and its cell
SSP_EVM_HD const float* entry_ptr(const float* out_img, int i, int nA, int K, int nC, int W, int HW, int* cx, int* cy) {
  const int a = i % nA, cell = i / nA;
  *cx = cell % W; *cy = cell / W;
  return out_img + (long long)a * (2 * K + 1 + nC) * HW + cell;
}

// the box list's filter, conf = det * cls_max_conf compared in fp32 with conf_thresh rounded to fp32
SSP_EVM_HD bool listed(const Decoded& d, float conf_thresh) { return d.det * d.cmax > conf_thresh; }

SSP_EVM_HD uint32_t float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}

// ordering key of a listed box among the boxes of its class: larger det first, then smaller index; never 0
SSP_EVM_HD unsigned long long pick_key(float det, int i) {
  return ((unsigned long long)float_bits(det) << 32) | (unsigned long long)(~(uint32_t)i);
}
SSP_EVM_HD int key_index(unsigned long long key) { return (int)(~(uint32_t)(key & 0xffffffffull)); }

// the fallback's running maxima, one entry at a time in visiting order
struct Fallback {
  float max_conf, max_cls;
  int ind;
};
SSP_EVM_HD Fallback fallback_init() { Fallback f; f.max_conf = -1.f; f.max_cls = -INFINITY; f.ind = -1; return f; }
SSP_EVM_HD void fallback_update(Fallback& f, float det, float cls_corr, int i) {
  if (det > f.max_conf && cls_corr > f.max_cls) { f.max_conf = det; f.max_cls = cls_corr; f.ind = i; }
}

// valid_multi.py:118-123 for ground truth g of class cls: best[c] = largest pick_key of the listed boxes of class c (0: none);
// has_corr = some listed box has correspondingclass.  Returns the chosen entry (kSrcFallback for the fallback box) and its
// flags; prev_src / prev_flags are the previous ground truth's (ignored for g == 0, which always finds a box).
SSP_EVM_HD int select_box(const unsigned long long* best, int nC, int corr, bool has_corr, int cls, int prev_src, int prev_flags,
                          int* flags) {
  if (cls >= 0 && cls < nC && best[cls] != 0ull) { *flags = 0; return key_index(best[cls]); }
  if (cls == corr && !has_corr) { *flags = kFlagFallback; return kSrcFallback; }
  *flags = (prev_flags & kFlagFallback) | kFlagCarried;
  return prev_src;
}

// box [x0/W, y0/H, ..., det_conf, cls_max_conf, cls_max_id] of the chosen entry (or of the fallback's max_ind)
SSP_EVM_HD void write_box(const float* out_img, int src, const Fallback& fb, int corr, int nA, int K, int nC, int W, int H,
                          float* box) {
  const int i = src == kSrcFallback ? fb.ind : src;
  int cx, cy;
  const float* o = entry_ptr(out_img, i, nA, K, nC, W, H * W, &cx, &cy);
  const Decoded d = decode_entry(o, H * W, K, nC, cx, cy, W, H, corr, box);
  if (src == kSrcFallback) { box[2 * K] = fb.max_conf; box[2 * K + 1] = fb.max_cls; box[2 * K + 2] = (float)corr; }
  else { box[2 * K] = d.det; box[2 * K + 1] = d.cmax; box[2 * K + 2] = (float)d.id; }
}

// PnP inputs (valid_multi.py:126-132): label row [cls, x0, y0, ...] -> fix_corner_order'ed pixels; box -> pixels, in fp32
SSP_EVM_HD void box_uv(const float* box, float im_width, float im_height, int k, float* uv_pr) {
  uv_pr[2 * k] = box[2 * k] * im_width; uv_pr[2 * k + 1] = box[2 * k + 1] * im_height;
}
SSP_EVM_HD void write_uv(const float* label_row, const float* box, float im_width, float im_height, float* uv_gt, float* uv_pr) {
  for (int k = 0; k < kKeypoints; k++) {
    const int s = fix_order(k);
    uv_gt[2 * k] = label_row[1 + 2 * s] * im_width; uv_gt[2 * k + 1] = label_row[2 + 2 * s] * im_height;
    box_uv(box, im_width, im_height, k, uv_pr);
  }
}

// ---- prediction (no labels): slot (frame, requested class c) takes the box valid_multi.py would choose for a ground truth of
// class c that is the image's first, i.e. select_box with correspondingclass = cls = c:
//   * the listed box best[c] when some listed box has arg-max class c (flags 0);
//   * otherwise the fallback box for correspondingclass = c (kFlagFallback), from fallback_scan.
SSP_EVM_HD int predict_slot(const unsigned long long* best, int nC, int c, int* flags) {
  return select_box(best, nC, c, c >= 0 && c < nC && best[c] != 0ull, c, kSrcFallback, 0, flags);
}

// the fallback's running maxima for correspondingclass = c over an image's n entries, given each entry's det and its softmax's mx
// and den (Decoded).  softmax[c] is recomputed by class_prob only where the && of fallback_update reads it (det > max_conf), which
// gives the maxima of fallback_update over decode_entry(..., corr = c, ...) bit for bit.
SSP_EVM_HD Fallback fallback_scan(const float* out_img, const float* det, const float* mx, const float* den, int n, int c, int nA, int K,
                                  int nC, int W, int HW) {
  Fallback fb = fallback_init();
  for (int i = 0; i < n; i++)
    if (det[i] > fb.max_conf) {
      int cx, cy;
      fallback_update(fb, det[i], class_prob(entry_ptr(out_img, i, nA, K, nC, W, HW, &cx, &cy), HW, K, c, mx[i], den[i]), i);
    }
  return fb;
}

// valid_multi.py:20-23: label rows up to the first with x0 == 0 (all of them when every row is filled)
SSP_EVM_HD int truths_length(const float* label, int rows, int num_labels) {
  int n = 0;
  while (n < rows && label[n * num_labels + 1] != 0.f) n++;
  return n;
}

}  // namespace ssp_evm
