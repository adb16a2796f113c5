// Tracking the world instances of a camera rig over time: the rule of ssp_world_track_associate / ssp_world_track_commit
// (world_track.cu), shared with the CPU test harness (tests/helpers/world_track_host.cpp, g++ -ffp-contract=off; world_track.cu is
// built with -fmad=false) and restated with whole arrays in oracle/world_track_ref.py.  fp64 throughout.  It reuses the slot fields
// and the ageing rule of track_core.h and the pose filter of pose_filter_core.h unchanged.
//
// Each capture g of a call (rows g C .. g C + C - 1 of ssp_fuse_instances) is its own stream.  Stream g owns T = max_tracks slots
// and a next_id counter: tracks [T][kFields] (track_core.h: alive, id, cls, misses, hits), poses [T][12] = R (row-major) and t of
// the track's last fused world pose, and with motion filter [T][kFilterDoubles] (pose_filter_core.h's layout; only the frame
// changes: the left perturbation is in world axes, as the fusion's world_cov is).  Per capture and stream the inputs are what
// ssp_fuse_instances wrote: world_count, world_cls [M], R_world [M][9], t_world [M][3], world_cov [M][36], fuse_status [M].  In
// this order:
//   1. predict (with motion only): every alive slot whose filter has started moves by the stream's dt, in place (ssp_pf::predict,
//      as ssp_track_predict does).  A slot's position is then its filter's t, else the t of its last fused pose;
//   2. match: the world instances w = 0 .. world_count - 1 are walked in slot order, the fusion's emission order (most views
//      first).  Instance w of class k may take an alive track of class k that no earlier instance took this capture when
//      |t_w - position|^2 < r_k^2 (strictly); it takes the smallest squared distance, the lower slot on a tie.  r_k = match_dist
//      d_k, d_k (class_size) the largest distance between two of class k's 8 box corners, computed once on the host from the fp32
//      object table, so the kernels and the harness read the same bits;
//   3. age: every alive track left unmatched gets misses += 1 and dies when misses > max_misses (track_core.h step 2);
//   4. birth: the unmatched instances, in slot order, each take the lowest free slot and id = next_id++ (track_core.h step 3);
//      with no free slot the instance is untracked (world_track_id -1).  An instance whose class lies outside [0, num_classes)
//      matches nothing and is untracked;
//   5. commit: a matched or born track stores the instance's R, t, misses = 0, hits += 1; with motion, ssp_pf::update_slot then
//      runs with matched = step 2's result and the measurement (R_world, t_world, world_cov), usable when fuse_status lacks the
//      singular bit: the gate, restart and Joseph update of the single-camera filter.
// Steps 1-4 are ssp_world_track_associate, step 5 ssp_world_track_commit.  A freed slot keeps its stale fields with alive = 0.
//
// Why a metric gate on translation, not the IoU of projected boxes or a Mahalanobis distance: the rig gives metric 3-D positions
// directly.  Two solid instances of one class cannot have centres much closer than their size, so a radius scaled by the object
// is unambiguous, and it means the same with and without motion.  A fresh filter's translation covariance is the fusion's, a few
// millimetres, with no velocity yet, so a Mahalanobis gate would refuse a moving object's second capture; the filter's own chi^2
// gate still decides when a matched track restarts.
#pragma once
#include "pose_filter_core.h"

namespace ssp_wt {

using ssp_trk::kAlive;
using ssp_trk::kCls;
using ssp_trk::kFields;
using ssp_trk::kHits;
using ssp_trk::kId;
using ssp_trk::kMaxTracks;
using ssp_trk::kMisses;

constexpr int kPoseDoubles = 12;       // R [9], t [3] of a track's last fused pose
constexpr int kMaxWorld = 256;         // largest number of world slots per capture
constexpr int kFuseSingular = 4;       // ssp_fuse_instances' fuse_status bit: world_cov is not usable

SSP_HD bool tracked_class(int k, int num_classes) { return k >= 0 && k < num_classes; }

// r_k^2 of step 2
SSP_HD double radius2(double match_dist, double class_size) {
  const double r = match_dist * class_size;
  return r * r;
}

SSP_HD double dist2(const double* a, const double* b) {
  const double x = a[0] - b[0], y = a[1] - b[1], z = a[2] - b[2];
  return x * x + y * y + z * z;
}

// step 1 for one slot: st its int fields, f its filter
SSP_HD void predict_slot(const int* st, double* f, double dt, const ssp_pf::FilterParams& p) {
  if (st[kAlive] && f[ssp_pf::kOffValid] == 1.0) ssp_pf::predict(f, dt, p);
}

// the position a slot is matched at after step 1: its started filter's t (f null: no motion), else its last fused t
SSP_HD const double* position(const double* pose, const double* f) {
  return f && f[ssp_pf::kOffValid] == 1.0 ? f + ssp_pf::kOffT : pose + 9;
}

// step 2: may an instance of class wcls at squared distance d2 take track st that `taken` says is (not) matched yet
SSP_HD bool can_match(const int* st, bool taken, int wcls, double d2, double r2) {
  return st[kAlive] && !taken && st[kCls] == wcls && d2 < r2;
}

// step 2's order: (d2, s) before the best so far (best_s < 0: none)
SSP_HD bool closer(double d2, int s, double best_d2, int best_s) {
  return best_s < 0 || d2 < best_d2 || (d2 == best_d2 && s < best_s);
}

// step 5's store for a matched or born track
SSP_HD void store(int* st, double* pose, const double* R, const double* t) {
  for (int i = 0; i < 9; i++) pose[i] = R[i];
  for (int i = 0; i < 3; i++) pose[9 + i] = t[i];
  st[kMisses] = 0;
  st[kHits] += 1;
}

// step 5's filter for one world slot: f the filter of its track slot, or null (an empty or untracked world slot: zero outputs)
SSP_HD void filter_slot(double* f, bool matched, const double* R, const double* t, const double* cov, int fuse_status,
                        const ssp_pf::FilterParams& p, double* R_filt, double* t_filt, double* pose_cov, double* velocity, int* reinit) {
  ssp_pf::update_slot(f, matched, R, t, cov, (fuse_status & kFuseSingular) ? 1 : 0, p, R_filt, t_filt, pose_cov, velocity, reinit);
}

}  // namespace ssp_wt
