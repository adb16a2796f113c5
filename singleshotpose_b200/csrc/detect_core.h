// Every instance in a frame: the candidate, ordering, overlap and suppression rules of ssp_detect_instances (region_multi.cu),
// shared with the CPU test harness (tests/helpers/detect_host.cpp, built with g++ -ffp-contract=off).
//
// Per frame, each frame on its own:
//   * candidates: every (cell, anchor) entry i, in eval_multi_core.h's visiting order, that get_multi_region_boxes(...,
//     only_objectness=0) lists (listed(): det_conf * cls_max_conf > conf_thresh; its fallback box is never a candidate) and whose
//     arg-max class is one of the requested classes.  With one anchor and one class (the single-object head) cls_max_conf is 1;
//   * order: descending pick_key(det_conf, i) -- larger det_conf first, the lower entry on ties; keys are unique, so the first
//     instance of class c is the box the multi-object predictor puts in class c's slot;
//   * overlap box: the axis-aligned rectangle of the 8 corner keypoints (k = 1..8) in frame pixels, the fp32 values box_uv gives
//     PnP (the centroid is not part of it, as the label files' width and height are not);
//   * greedy suppression within each class: walking the candidates in key order, one is kept unless a kept box of the SAME class
//     overlaps it with IoU > nms_thresh (strictly, as YOLO's nms); a zero-area union gives IoU 0;
//   * output: the first max_instances kept boxes in key order.  Suppression only looks at earlier keys of the same class, so this
//     is full NMS followed by truncation; kept (before truncation) is reported beside count = min(kept, max_instances).
// The reference's own nms (utils_multi.py:223-241) reads YOLO boxes -- box[4] as the confidence, keypoints 0-1 as centre and
// size -- and cannot run on pose boxes; these rules replace it, they do not restate it.
//
// The IoU is fp32 in the order written below with every operation rounded on its own (__f*_rn on the device, -ffp-contract=off
// on the host), so the kernel and the harness keep the same boxes bit for bit.
#pragma once
#include "eval_multi_core.h"

#if defined(__CUDACC__)
#define SSP_DET_HD __host__ __device__ __forceinline__
#else
#define SSP_DET_HD inline
#endif

namespace ssp_det {

constexpr int kMaxInstances = 256;            // largest max_instances

struct Rect {
  float x0, y0, x1, y1;
};

SSP_DET_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
SSP_DET_HD float sub_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
SSP_DET_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
SSP_DET_HD float div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// rectangle of keypoints 1..8 of uv [9][2] (frame pixels)
SSP_DET_HD Rect corner_rect(const float* uv) {
  Rect r;
  r.x0 = r.x1 = uv[2]; r.y0 = r.y1 = uv[3];
  for (int k = 2; k < ssp_evm::kKeypoints; k++) {
    r.x0 = fminf(r.x0, uv[2 * k]); r.x1 = fmaxf(r.x1, uv[2 * k]);
    r.y0 = fminf(r.y0, uv[2 * k + 1]); r.y1 = fmaxf(r.y1, uv[2 * k + 1]);
  }
  return r;
}

// IoU of two rectangles: inter = (min x1 - max x0) * (min y1 - max y0) when both sides are positive (else 0),
// union = (area a + area b) - inter, IoU = inter / union, 0 when union <= 0
SSP_DET_HD float iou(const Rect& a, const Rect& b) {
  const float iw = sub_rn(fminf(a.x1, b.x1), fmaxf(a.x0, b.x0));
  const float ih = sub_rn(fminf(a.y1, b.y1), fmaxf(a.y0, b.y0));
  if (!(iw > 0.f) || !(ih > 0.f)) return 0.f;
  const float inter = mul_rn(iw, ih);
  const float area_a = mul_rn(sub_rn(a.x1, a.x0), sub_rn(a.y1, a.y0));
  const float area_b = mul_rn(sub_rn(b.x1, b.x0), sub_rn(b.y1, b.y0));
  const float uni = sub_rn(add_rn(area_a, area_b), inter);
  return uni > 0.f ? div_rn(inter, uni) : 0.f;
}

// suppression test of a candidate against one kept box of its class
SSP_DET_HD bool suppresses(const Rect& kept, const Rect& cand, float nms_thresh) { return iou(kept, cand) > nms_thresh; }

// a decoded entry is a candidate: listed, and its arg-max class requested (requested: flags by class id)
SSP_DET_HD bool candidate(const ssp_evm::Decoded& d, float conf_thresh, const unsigned char* requested) {
  return ssp_evm::listed(d, conf_thresh) && requested[d.id];
}

// entry i's keypoints in frame pixels (box_uv of its decoded box) and its rectangle; box receives the 2K keypoint values
SSP_DET_HD Rect entry_rect(const float* box, float frame_w, float frame_h, float* uv) {
  for (int k = 0; k < ssp_evm::kKeypoints; k++) ssp_evm::box_uv(box, frame_w, frame_h, k, uv);
  return corner_rect(uv);
}

}  // namespace ssp_det
