// Host harness of the multi-object evaluation selection: the rules of eval_multi_core.h driven the way eval_multi_select_kernel
// (region_multi.cu) drives them, with plain loops: the per-class best listed box as a running max over pick_key (the kernel
// uses a shared atomicMax), the fallback scan, the per-ground-truth choice and the packing of boxes and PnP points.
// Also reports the chosen box's position in the reference's box list (listed boxes before it; the fallback comes last).
// Test infrastructure: built by tests/test_eval_multi_cpu.py into a temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/eval_multi_core.h"

using namespace ssp_evm;

extern "C" {
int h_eval_multi_select(const float* out, int B, int K, int nC, int nA, int H, int W, const float* target, int stride, const int* gt_offset,
                        float conf_thresh, float im_width, float im_height, float* boxes, int* flags, float* uv, int* pos) {
  if (K != kKeypoints || H * W * nA > kMaxEntries || nC > kMaxClasses) return -1;
  const int HW = H * W, n = HW * nA, nl = 2 * K + 3, G = gt_offset[B];
  std::vector<float> det(n), corr_p(n);
  std::vector<int> before(n + 1);
  std::vector<unsigned long long> best(nC);
  for (int b = 0; b < B; b++) {
    const int g0 = gt_offset[b], ng = gt_offset[b + 1] - g0;
    if (ng <= 0) continue;
    const float* t = target + (long long)b * stride;
    const int corr = (int)t[0];
    const float* o = out + (long long)b * nA * (2 * K + 1 + nC) * HW;
    for (int c = 0; c < nC; c++) best[c] = 0ull;
    before[0] = 0;
    for (int i = 0; i < n; i++) {
      int cx, cy;
      const Decoded d = decode_entry(entry_ptr(o, i, nA, K, nC, W, HW, &cx, &cy), HW, K, nC, cx, cy, W, H, corr, nullptr);
      det[i] = d.det; corr_p[i] = d.corr;
      const bool l = listed(d, conf_thresh);
      if (l && pick_key(d.det, i) > best[d.id]) best[d.id] = pick_key(d.det, i);
      before[i + 1] = before[i] + (l ? 1 : 0);
    }
    const bool has_corr = corr >= 0 && corr < nC && best[corr] != 0ull;
    Fallback fb = fallback_init();
    if (!has_corr)
      for (int i = 0; i < n; i++) fallback_update(fb, det[i], corr_p[i], i);
    int src = 0, fl = 0;
    for (int g = 0; g < ng; g++) {
      const long long gi = g0 + g;
      src = select_box(best.data(), nC, corr, has_corr, (int)t[g * nl], src, fl, &fl);
      write_box(o, src, fb, corr, nA, K, nC, W, H, boxes + gi * nl);
      flags[gi] = fl;
      pos[gi] = src == kSrcFallback ? before[n] : before[src];
      write_uv(t + g * nl, boxes + gi * nl, im_width, im_height, uv + gi * 2 * K, uv + (G + gi) * 2 * K);
    }
  }
  return 0;
}
}
