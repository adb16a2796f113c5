// Tracking instances across camera frames: the rule of ssp_track_associate / ssp_track_commit (track.cu), shared with the CPU test
// harness (tests/helpers/track_host.cpp, built with g++ -ffp-contract=off).
//
// Each row b of a call is its own camera stream.  Stream b owns T = max_tracks slots and a next_id counter.  A slot holds alive, id
// (int32, per stream, from 0 after a reset), cls, misses (consecutive frames without a match), hits, rect (the fp32 corner rectangle of
// its last detection, ssp_det::corner_rect) and pose (the fp64 LM vector (rvec, t) of its last solve: what cv2.solvePnP returns as
// rvec, tvec).  Per frame and stream, the input is what ssp_detect_instances wrote: count, cls [M], uv [M][9][2].  In this order:
//   1. match: the detections m = 0..count-1 are walked in the detector's order (descending det_conf).  Detection m may take an alive
//      track of the SAME class that no earlier detection took this frame and whose rectangle has iou(track.rect, rect_m) > match_iou
//      (strictly; ssp_det::iou itself); it takes the highest IoU, the lower slot on a tie;
//   2. age: every alive track left unmatched gets misses += 1 and dies (its slot is freed) when misses > max_misses, so a track seen
//      again after max_misses missed frames survives;
//   3. birth: the unmatched detections, in order, each take the lowest free slot (slots freed in step 2 included) and get
//      id = next_id++; when no slot is free the detection is untracked (track_id -1, a cold solve, nothing stored);
//   4. PnP: a detection matched to a track starts LM from the track's pose (warm, ssp_pnp_batched_guess); the others get the DLT +
//      LM of ssp_pnp_batched_counted (cold);
//   5. commit: each matched or born track takes rect <- rect_m, pose <- the final LM vector of m's solve, misses <- 0, hits += 1 (a new
//      track starts at 1).
// There is no motion model: a track is matched against its last rectangle, and the guess is its last pose.  Steps 1-3 are
// ssp_track_associate, step 5 ssp_track_commit.  A freed slot keeps its stale fields with alive = 0; only alive slots are read.
// The only arithmetic is the fp32 rectangle and IoU of detect_core.h, so the kernels and the harness agree bit for bit.
#pragma once
#include "detect_core.h"

namespace ssp_trk {

constexpr int kMaxTracks = 256;               // largest max_tracks
// the int fields of a slot: tracks [B][T][kFields]
enum Field { kAlive = 0, kId = 1, kCls = 2, kMisses = 3, kHits = 4, kFields = 5 };

// step 1: may a detection of class dcls with rectangle-IoU `iou` take track st (int fields) that `taken` says is (not) matched yet
SSP_DET_HD bool can_match(const int* st, bool taken, int dcls, float iou, float match_iou) {
  return st[kAlive] && !taken && st[kCls] == dcls && iou > match_iou;
}

// step 1: the arg-max key of a matchable track: larger IoU first, then the lower slot.  A matchable IoU is > match_iou >= 0, so its
// bits order as the values and the key is never 0 (0 = no track)
SSP_DET_HD unsigned long long match_key(float iou, int slot) {
  unsigned u;
#if defined(__CUDA_ARCH__)
  u = __float_as_uint(iou);
#else
  __builtin_memcpy(&u, &iou, 4);
#endif
  return ((unsigned long long)u << 32) | (unsigned)(kMaxTracks - slot);
}
SSP_DET_HD int key_slot(unsigned long long key) { return kMaxTracks - (int)(unsigned)(key & 0xffffffffull); }

// step 2: an unmatched alive track after misses += 1
SSP_DET_HD bool dies(int misses, int max_misses) { return misses > max_misses; }

}  // namespace ssp_trk
