// Host harness of the world-instance tracking (singleshotpose_b200/csrc/world_track_core.h): the launches of world_track.cu run
// serially over the header's functions.  Built with -ffp-contract=off, as world_track.cu is built with -fmad=false.  Test
// infrastructure: built by the tests into a temporary .so; never loaded by the product.
#include <cmath>
#include <vector>

#include "../../singleshotpose_b200/csrc/world_track_core.h"

using namespace ssp_wt;

static bool pos_finite(double x) { return x > 0.0 && std::isfinite(x); }

extern "C" {
// ssp_world_track_associate on host arrays; -1 for the arguments the entry point refuses
int h_world_track_associate(int G, int C, int T, int M, const int* world_count, const int* world_cls, const double* t_world,
                            const int* world_index, const double* class_size, int num_classes, double match_dist, int max_misses, int* tracks,
                            const double* poses, double* filter, const double* dt, double accel_rot, double accel_trans, int* next_id,
                            int* wslot, int* world_track_id, int* matched, int* track_id) {
  if (G < 0 || T < 1 || T > kMaxTracks || M < 1 || M > kMaxWorld || C < 1 || C > 16 || num_classes < 1 || max_misses < 0 ||
      !pos_finite(match_dist) || !pos_finite(accel_rot) || !pos_finite(accel_trans) || (!filter) != (!dt))
    return -1;
  const ssp_pf::FilterParams p = {accel_rot * accel_rot, accel_trans * accel_trans, 0.0, 0.0, 0.0};
  std::vector<double> pos(3 * T);
  std::vector<unsigned char> taken(T);
  for (int g = 0; g < G; g++) {
    int* st = tracks + (long long)g * T * kFields;
    const int n = world_count[g] < 0 ? 0 : (world_count[g] > M ? M : world_count[g]);
    for (int s = 0; s < T; s++) {                                   // 1. predict
      const long long ts = (long long)g * T + s;
      double* f = filter ? filter + ts * ssp_pf::kFilterDoubles : nullptr;
      if (f) predict_slot(st + s * kFields, f, dt[g], p);
      const double* q = position(poses + ts * kPoseDoubles, f);
      for (int i = 0; i < 3; i++) pos[3 * s + i] = q[i];
      taken[s] = 0;
    }
    std::vector<int> sl(M, -1);
    for (int w = 0; w < n; w++) {                                   // 2. match
      const long long gw = (long long)g * M + w;
      const int k = world_cls[gw];
      if (!tracked_class(k, num_classes)) continue;
      const double r2 = radius2(match_dist, class_size[k]);
      double best = 0.0;
      int bs = -1;
      for (int s = 0; s < T; s++) {
        const double d2 = dist2(t_world + gw * 3, &pos[3 * s]);
        if (can_match(st + s * kFields, taken[s], k, d2, r2) && closer(d2, s, best, bs)) { best = d2; bs = s; }
      }
      if (bs >= 0) { taken[bs] = 1; sl[w] = bs; }
    }
    for (int s = 0; s < T; s++) {                                   // 3. age
      int* f = st + s * kFields;
      if (f[kAlive] && !taken[s]) {
        f[kMisses] += 1;
        if (ssp_trk::dies(f[kMisses], max_misses)) f[kAlive] = 0;
      }
    }
    std::vector<int> ids(M, -1);
    for (int w = 0; w < M; w++) {                                   // 4. birth
      const long long gw = (long long)g * M + w;
      matched[gw] = w < n && sl[w] >= 0;
      if (w < n && sl[w] >= 0) {
        ids[w] = st[sl[w] * kFields + kId];
      } else if (w < n && tracked_class(world_cls[gw], num_classes)) {
        int s = 0;
        while (s < T && st[s * kFields + kAlive]) s++;
        if (s < T) {
          int* f = st + s * kFields;
          f[kAlive] = 1; f[kId] = next_id[g]++; f[kCls] = world_cls[gw]; f[kMisses] = 0; f[kHits] = 0;
          sl[w] = s;
          ids[w] = f[kId];
        }
      }
      wslot[gw] = sl[w];
      world_track_id[gw] = ids[w];
    }
    for (long long i = (long long)g * C * M; i < (long long)(g + 1) * C * M; i++) {
      const int w = world_index[i];
      track_id[i] = w >= 0 && w < n ? ids[w] : -1;
    }
  }
  return 0;
}

// ssp_world_track_commit on host arrays; -1 for the arguments the entry point refuses
int h_world_track_commit(int G, int T, int M, const int* world_count, const double* R_world, const double* t_world, const double* world_cov,
                         const int* fuse_status, const int* wslot, const int* matched, int* tracks, double* poses, double* filter, double v0_rot,
                         double v0_trans, double gate, double* R_filt, double* t_filt, double* pose_cov, double* velocity, int* reinit) {
  if (G < 0 || T < 1 || T > kMaxTracks || M < 1 || M > kMaxWorld || !pos_finite(v0_rot) || !pos_finite(v0_trans) || !pos_finite(gate))
    return -1;
  const ssp_pf::FilterParams p = {0.0, 0.0, v0_rot * v0_rot, v0_trans * v0_trans, gate};
  for (long long o = 0; o < (long long)G * M; o++) {
    const int g = (int)(o / M), w = (int)(o % M);
    const int n = world_count[g] < 0 ? 0 : (world_count[g] > M ? M : world_count[g]);
    const int s = w < n ? wslot[o] : -1;
    const long long ts = (long long)g * T + s;
    if (s >= 0) store(tracks + ts * kFields, poses + ts * kPoseDoubles, R_world + o * 9, t_world + o * 3);
    if (filter)
      filter_slot(s < 0 ? nullptr : filter + ts * ssp_pf::kFilterDoubles, matched[o] != 0, R_world + o * 9, t_world + o * 3, world_cov + o * 36,
                  fuse_status[o], p, R_filt + o * 9, t_filt + o * 3, pose_cov + o * 36, velocity + o * 6, reinit + o);
  }
  return 0;
}
}
