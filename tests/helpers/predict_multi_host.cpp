// Host harness of the multi-object prediction selection: the rules of eval_multi_core.h driven the way
// predict_multi_select_kernel (region_multi.cu) drives them, with plain loops: every entry decoded once (det, mx, den), the
// per-class best listed box as a running max over pick_key (the kernel uses a shared atomicMax), then per requested class
// predict_slot, fallback_scan when the class is not listed, the box and its PnP points.  Also reports the chosen box's position
// in the reference's box list for that class (listed boxes before it; the fallback comes last).
// Test infrastructure: built by tests/test_predict_multi_cpu.py into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/eval_multi_core.h"

using namespace ssp_evm;

extern "C" {
int h_predict_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const int* classes, int n_req, float conf_thresh,
                           float frame_w, float frame_h, float* boxes, int* flags, float* uv, int* pos) {
  if (K != kKeypoints || H * W * nA > kMaxEntries || nC > kMaxClasses) return -1;
  const int HW = H * W, n = HW * nA, nl = 2 * K + 3;
  std::vector<float> det(n), mx(n), den(n);
  std::vector<int> before(n + 1);
  std::vector<unsigned long long> best(nC);
  for (int b = 0; b < B; b++) {
    const float* o = out + (long long)b * nA * (2 * K + 1 + nC) * HW;
    for (int c = 0; c < nC; c++) best[c] = 0ull;
    before[0] = 0;
    for (int i = 0; i < n; i++) {
      int cx, cy;
      const Decoded d = decode_entry(entry_ptr(o, i, nA, K, nC, W, HW, &cx, &cy), HW, K, nC, cx, cy, W, H, -1, nullptr);
      det[i] = d.det; mx[i] = d.mx; den[i] = d.den;
      const bool l = listed(d, conf_thresh);
      if (l && pick_key(d.det, i) > best[d.id]) best[d.id] = pick_key(d.det, i);
      before[i + 1] = before[i] + (l ? 1 : 0);
    }
    for (int q = 0; q < n_req; q++) {
      const int c = classes[q];
      const long long slot = (long long)b * n_req + q;
      int fl;
      const int src = predict_slot(best.data(), nC, c, &fl);
      const Fallback fb = src == kSrcFallback ? fallback_scan(o, det.data(), mx.data(), den.data(), n, c, nA, K, nC, W, HW) : fallback_init();
      write_box(o, src, fb, c, nA, K, nC, W, H, boxes + slot * nl);
      flags[slot] = fl;
      pos[slot] = src == kSrcFallback ? before[n] : before[src];
      for (int k = 0; k < kKeypoints; k++) box_uv(boxes + slot * nl, frame_w, frame_h, k, uv + slot * 2 * K);
    }
  }
  return 0;
}
}
