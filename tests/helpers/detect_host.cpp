// Host harness of the instance detection's ordering / IoU / suppression stage: the rules of detect_core.h driven with plain
// loops on decoded entries (det_conf, cls_max_conf, arg-max class and the fp32 pixel keypoints of each entry, in visiting
// order) -- the inputs the kernel derives from decode_entry.  Built with -ffp-contract=off so the IoU is rounded as the kernel's.
// Test infrastructure: built by tests/test_detect_cpu.py into a temporary .so; never loaded by the product.
#include <algorithm>
#include <functional>
#include <vector>

#include "../../singleshotpose_b200/csrc/detect_core.h"

using namespace ssp_evm;

extern "C" {
// one frame of n entries: det, cmax [n], id [n], uv [n][9][2]; requested [num_classes] flags.  Out: entries [max_inst] (the
// kept entries in key order, -1 past count), *count, *kept.
int h_detect_stage(const float* det, const float* cmax, const int* id, const float* uv, int n, const unsigned char* requested,
                   float conf_thresh, float nms_thresh, int max_inst, int* entries, int* count, int* kept) {
  if (n > kMaxEntries || max_inst < 1 || max_inst > ssp_det::kMaxInstances) return -1;
  std::vector<unsigned long long> keys;
  std::vector<ssp_det::Rect> rect(n);
  for (int i = 0; i < n; i++) {
    Decoded d;
    d.det = det[i]; d.cmax = cmax[i]; d.id = id[i]; d.corr = 0.f; d.mx = 0.f; d.den = 0.f;
    if (!ssp_det::candidate(d, conf_thresh, requested)) continue;
    rect[i] = ssp_det::corner_rect(uv + (long long)i * 2 * kKeypoints);
    keys.push_back(pick_key(d.det, i));
  }
  std::sort(keys.begin(), keys.end(), std::greater<unsigned long long>());
  std::vector<std::vector<int>> kept_of(kMaxClasses);
  int nk = 0;
  for (int j = 0; j < max_inst; j++) entries[j] = -1;
  for (unsigned long long key : keys) {
    const int i = key_index(key);
    bool sup = false;
    for (int e : kept_of[id[i]]) sup = sup || ssp_det::suppresses(rect[e], rect[i], nms_thresh);
    if (sup) continue;
    kept_of[id[i]].push_back(i);
    if (nk < max_inst) entries[nk] = i;
    nk++;
  }
  *count = std::min(nk, max_inst);
  *kept = nk;
  return 0;
}

float h_iou(const float* a, const float* b) {
  const ssp_det::Rect ra{a[0], a[1], a[2], a[3]}, rb{b[0], b[1], b[2], b[3]};
  return ssp_det::iou(ra, rb);
}
}
