// Host harness of the multi-object ops: plans one phase with the same recording back end the CUDA path uses
// (multi_batch_plan, augment_core.h) and executes the op table stage by stage with plain loops; OP_COUNT's per-sample
// reduction is a plain sum here (aug_stage_kernel uses warp sums + integer atomics).
// Test infrastructure: built by tests/test_augment_multi_cpu.py into a temporary .so; never loaded by the product.
#include "../../singleshotpose_b200/csrc/augment_core.h"

using namespace ssp_aug;

extern "C" {
long long h_multi_op_bytes() { return (long long)sizeof(AugOp); }
long long h_multi_item_bytes() { return (long long)sizeof(AugMultiItem); }
long long h_multi_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) { return multi_work_bytes(in_w, in_h, out_w, out_h, resample); }
int h_multi_max_stages() { return kMaxMultiStages; }
// plans `phase` for n items into table (kMaxMultiStages * n ops) and runs it; returns the planner's code
int h_multi_run(int phase, const AugMultiItem* items, int n, int out_w, int out_h, int resample, AugOp* table, int* stage_dims) {
  const int rc = multi_batch_plan(phase, items, n, out_w, out_h, resample, table, stage_dims);
  if (rc) return rc;
  for (int s = 0; s < kMaxMultiStages; s++)
    for (int i = 0; i < n; i++) {
      const AugOp& o = table[(long long)s * n + i];
      if (o.kind == OP_NONE) continue;
      for (int y = 0; y < o.ny; y++)
        for (int x = 0; x < o.nx; x++) {
          if (o.kind == OP_COUNT) {
            unsigned sum = 0, inter = 0;
            count_px(o, x, y, &sum, &inter);
            o.counts[0] += sum; o.counts[1] += inter;
          } else {
            op_element(o, x, y);
          }
        }
    }
  return 0;
}
}
