// Host harness of the tracking rule (singleshotpose_b200/csrc/track_core.h) driven with plain serial loops on the state layout of
// ssp_track_associate / ssp_track_commit, and of the warm-started PnP (pnp_core.h's pnp_solve_one with a guess).  Built with
// -ffp-contract=off so the rectangle IoU is rounded as the kernels'.  Test infrastructure: built by tests/test_track_cpu.py into a
// temporary .so; never loaded by the product.
#include <vector>

#include "../../singleshotpose_b200/csrc/pnp_core.h"
#include "../../singleshotpose_b200/csrc/track_core.h"

using namespace ssp_trk;

extern "C" {
// steps 1-3 for B streams; the arguments are those of ssp_track_associate (host arrays)
int h_track_associate(int B, int T, int M, const int* count, const int* cls, const float* uv, float match_iou, int max_misses,
                      int* tracks, const float* rects, const double* poses, int* next_id, int* slot, int* track_id, double* guess,
                      int* use_guess) {
  if (B < 0 || T < 1 || T > kMaxTracks || M < 1 || M > ssp_det::kMaxInstances || max_misses < 0) return -1;
  for (int b = 0; b < B; b++) {
    int* st = tracks + (long long)b * T * kFields;
    const int n = count[b] < 0 ? 0 : (count[b] > M ? M : count[b]);
    std::vector<int> dslot(M, -1);
    std::vector<bool> taken(T, false), warm(M, false);
    for (int m = 0; m < n; m++) {                                       // 1. match
      const ssp_det::Rect r = ssp_det::corner_rect(uv + ((long long)b * M + m) * 18);
      const int c = cls[(long long)b * M + m];
      int best = -1;
      float best_iou = 0.f;
      for (int s = 0; s < T; s++) {
        const float* q = rects + ((long long)b * T + s) * 4;
        const float v = ssp_det::iou(ssp_det::Rect{q[0], q[1], q[2], q[3]}, r);
        if (can_match(st + s * kFields, taken[s], c, v, match_iou) && (best < 0 || v > best_iou)) { best = s; best_iou = v; }
      }
      if (best >= 0) { taken[best] = true; dslot[m] = best; warm[m] = true; }
    }
    for (int s = 0; s < T; s++) {                                       // 2. age
      int* f = st + s * kFields;
      if (f[kAlive] && !taken[s]) {
        f[kMisses] += 1;
        if (dies(f[kMisses], max_misses)) f[kAlive] = 0;
      }
    }
    for (int m = 0; m < M; m++) track_id[(long long)b * M + m] = warm[m] ? st[dslot[m] * kFields + kId] : -1;
    for (int m = 0; m < n; m++) {                                       // 3. birth
      if (warm[m]) continue;
      int s = 0;
      while (s < T && st[s * kFields + kAlive]) s++;
      if (s == T) continue;                                             // untracked
      int* f = st + s * kFields;
      f[kAlive] = 1; f[kId] = next_id[b]++; f[kCls] = cls[(long long)b * M + m]; f[kMisses] = 0; f[kHits] = 0;
      dslot[m] = s;
      track_id[(long long)b * M + m] = f[kId];
    }
    for (int m = 0; m < M; m++) {
      const long long o = (long long)b * M + m;
      slot[o] = dslot[m];
      use_guess[o] = warm[m];
      for (int i = 0; i < 6; i++) guess[o * 6 + i] = warm[m] ? poses[((long long)b * T + dslot[m]) * 6 + i] : 0.0;
    }
  }
  return 0;
}

// step 5; the arguments are those of ssp_track_commit (host arrays)
int h_track_commit(int B, int T, int M, const int* count, const float* uv, const int* slot, const double* params, int* tracks, float* rects,
                   double* poses) {
  for (int b = 0; b < B; b++)
    for (int m = 0; m < count[b] && m < M; m++) {
      const long long o = (long long)b * M + m;
      const int s = slot[o];
      if (s < 0) continue;
      const long long ts = (long long)b * T + s;
      const ssp_det::Rect r = ssp_det::corner_rect(uv + o * 18);
      rects[ts * 4] = r.x0; rects[ts * 4 + 1] = r.y0; rects[ts * 4 + 2] = r.x1; rects[ts * 4 + 3] = r.y1;
      for (int i = 0; i < 6; i++) poses[ts * 6 + i] = params[o * 6 + i];
      tracks[ts * kFields + kMisses] = 0;
      tracks[ts * kFields + kHits] += 1;
    }
  return 0;
}

// n problems with per-problem points; guess [n][6] used where use_guess[i] != 0.  Out: R [n][9], t [n][3], params [n][6], work [n][3]
int h_pnp_guess(const float* p3, const float* uv, const float* K, int np, long long n, int max_iter, const double* guess,
                const int* use_guess, double* R, double* t, double* params, int* work) {
  if (np < 6 || np > PNP_MAXP) return -1;
  for (long long i = 0; i < n; i++)
    ssp_pnp::pnp_solve_one(p3 + i * 3 * np, uv + i * 2 * np, K, np, max_iter, R + i * 9, t + i * 3, work + i * 3, nullptr,
                           use_guess[i] ? guess + i * 6 : nullptr, params + i * 6);
  return 0;
}
}
