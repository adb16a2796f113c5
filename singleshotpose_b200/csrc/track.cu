// Tracking instances across camera frames (rules: track_core.h).  Two launches around the PnP of the instance head, both fed from
// device memory (the detector's count, cls, uv and the solve's LM vectors), so a graph replay needs no host read-back:
//   ssp_track_associate  steps 1-3, one CTA of one warp per stream.  The stream's slots and its detections' rectangles are staged in
//                        shared memory; lane l owns slots l, l + 32, ...  Step 1 visits the detections serially (a matched track is
//                        taken), each one a warp arg-max of match_key over the slots (shuffles, no block barrier).  Step 3 lists the
//                        free slots in ascending order with ballots; the k-th unmatched detection (ballot prefix) takes the k-th.
//   ssp_track_commit     step 5, one thread per detection slot: a slot is matched or born by at most one detection per frame.
#include "ssp_common.cuh"
#include "track_core.h"

namespace ssp {

constexpr int kTrackWarp = 32;

struct TrackParams {
  const int* count; const int* cls; const float* uv; const double* poses; const float* rects;
  int* tracks; int* next_id; int* slot; int* track_id; double* guess; int* use_guess;
  int T, M, max_misses;
  float match_iou;
};

__global__ void __launch_bounds__(kTrackWarp) track_associate_kernel(const TrackParams p) {
  using namespace ssp_trk;
  using ssp_det::Rect;
  __shared__ int s_st[kMaxTracks * kFields];
  __shared__ Rect s_trect[kMaxTracks];
  __shared__ unsigned char s_taken[kMaxTracks];
  __shared__ Rect s_drect[ssp_det::kMaxInstances];
  __shared__ int s_dcls[ssp_det::kMaxInstances];
  __shared__ int s_dslot[ssp_det::kMaxInstances];
  __shared__ int s_free[kMaxTracks];
  const int b = blockIdx.x, lane = threadIdx.x, T = p.T, M = p.M;
  const int n = min(max(p.count[b], 0), M);
  int* st = p.tracks + (long long)b * T * kFields;
  for (int i = lane; i < T * kFields; i += kTrackWarp) s_st[i] = st[i];
  for (int s = lane; s < T; s += kTrackWarp) {
    const float* r = p.rects + ((long long)b * T + s) * 4;
    s_trect[s] = Rect{r[0], r[1], r[2], r[3]};
    s_taken[s] = 0;
  }
  for (int m = lane; m < n; m += kTrackWarp) {
    s_drect[m] = ssp_det::corner_rect(p.uv + ((long long)b * M + m) * 2 * ssp_evm::kKeypoints);
    s_dcls[m] = p.cls[(long long)b * M + m];
    s_dslot[m] = -1;
  }
  __syncwarp();
  // 1. match
  for (int m = 0; m < n; m++) {
    const Rect r = s_drect[m];
    const int c = s_dcls[m];
    unsigned long long key = 0;
    for (int s = lane; s < T; s += kTrackWarp) {
      const float v = ssp_det::iou(s_trect[s], r);
      if (can_match(s_st + s * kFields, s_taken[s], c, v, p.match_iou)) key = max(key, match_key(v, s));
    }
    for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    if (key) {
      const int s = key_slot(key);
      if (lane == 0) { s_taken[s] = 1; s_dslot[m] = s; }
    }
    __syncwarp();
  }
  // 2. age
  for (int s = lane; s < T; s += kTrackWarp) {
    int* f = s_st + s * kFields;
    if (f[kAlive] && !s_taken[s]) {
      f[kMisses] += 1;
      if (dies(f[kMisses], p.max_misses)) f[kAlive] = 0;
    }
  }
  __syncwarp();
  // 3. birth: the free slots in ascending order, then the k-th unmatched detection takes the k-th
  int nfree = 0;
  for (int s0 = 0; s0 < T; s0 += kTrackWarp) {
    const int s = s0 + lane;
    const bool fr = s < T && !s_st[s * kFields + kAlive];
    const unsigned bal = __ballot_sync(0xffffffffu, fr);
    if (fr) s_free[nfree + __popc(bal & ((1u << lane) - 1u))] = s;
    nfree += __popc(bal);
  }
  __syncwarp();
  const int id0 = p.next_id[b];
  int born = 0;
  for (int m0 = 0; m0 < n; m0 += kTrackWarp) {
    const int m = m0 + lane;
    const bool warm = m < n && s_dslot[m] >= 0;
    const bool um = m < n && !warm;
    const unsigned bal = __ballot_sync(0xffffffffu, um);
    const int k = born + __popc(bal & ((1u << lane) - 1u));
    int sl = warm ? s_dslot[m] : -1, tid = warm ? s_st[sl * kFields + kId] : -1;
    if (um && k < nfree) {
      sl = s_free[k];
      tid = id0 + k;
      int* f = s_st + sl * kFields;
      f[kAlive] = 1; f[kId] = tid; f[kCls] = s_dcls[m]; f[kMisses] = 0; f[kHits] = 0;
    }
    if (m < n) {
      const long long o = (long long)b * M + m;
      p.slot[o] = sl;
      p.track_id[o] = tid;
      p.use_guess[o] = warm;
      const double* pose = p.poses + ((long long)b * T + (warm ? sl : 0)) * 6;
      for (int i = 0; i < 6; i++) p.guess[o * 6 + i] = warm ? pose[i] : 0.0;
    }
    born += __popc(bal);
  }
  for (int m = n + lane; m < M; m += kTrackWarp) {
    const long long o = (long long)b * M + m;
    p.slot[o] = -1; p.track_id[o] = -1; p.use_guess[o] = 0;
    for (int i = 0; i < 6; i++) p.guess[o * 6 + i] = 0.0;
  }
  __syncwarp();
  for (int i = lane; i < T * kFields; i += kTrackWarp) st[i] = s_st[i];
  if (lane == 0) p.next_id[b] = id0 + min(born, nfree);
}

__global__ void track_commit_kernel(int B, int T, int M, const int* __restrict__ count, const float* __restrict__ uv,
                                    const int* __restrict__ slot, const double* __restrict__ params, int* __restrict__ tracks,
                                    float* __restrict__ rects, double* __restrict__ poses) {
  using namespace ssp_trk;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)B * M) return;
  const int b = (int)(o / M), m = (int)(o % M);
  if (m >= count[b]) return;
  const int s = slot[o];
  if (s < 0) return;
  const long long ts = (long long)b * T + s;
  const ssp_det::Rect r = ssp_det::corner_rect(uv + o * 2 * ssp_evm::kKeypoints);
  rects[ts * 4] = r.x0; rects[ts * 4 + 1] = r.y0; rects[ts * 4 + 2] = r.x1; rects[ts * 4 + 3] = r.y1;
  for (int i = 0; i < 6; i++) poses[ts * 6 + i] = params[o * 6 + i];
  tracks[ts * kFields + kMisses] = 0;
  tracks[ts * kFields + kHits] += 1;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_track_associate(int B, int max_tracks, int max_det, const int* count, const int* cls, const float* uv, float match_iou,
                        int max_misses, int* tracks, const float* rects, const double* poses, int* next_id, int* slot, int* track_id,
                        double* guess, int* use_guess, void* stream) {
  if (!count || !cls || !uv || !tracks || !rects || !poses || !next_id || !slot || !track_id || !guess || !use_guess)
    return fail_msg(SSP_ERR_ARG, "track_associate: null pointer");
  if (B < 0 || max_tracks < 1 || max_tracks > ssp_trk::kMaxTracks || max_det < 1 || max_det > ssp_det::kMaxInstances)
    return fail_msg(SSP_ERR_ARG, "track_associate: bad argument (B >= 0, 1 <= max_tracks <= 256, 1 <= max_det <= 256)");
  if (!(match_iou >= 0.f && match_iou <= 1.f)) return fail_msg(SSP_ERR_ARG, "track_associate: match_iou must be in [0, 1]");
  if (max_misses < 0) return fail_msg(SSP_ERR_ARG, "track_associate: max_misses must be >= 0");
  if (B == 0) return SSP_OK;
  TrackParams p;
  p.count = count; p.cls = cls; p.uv = uv; p.poses = poses; p.rects = rects; p.tracks = tracks; p.next_id = next_id; p.slot = slot;
  p.track_id = track_id; p.guess = guess; p.use_guess = use_guess;
  p.T = max_tracks; p.M = max_det; p.max_misses = max_misses; p.match_iou = match_iou;
  track_associate_kernel<<<B, kTrackWarp, 0, (cudaStream_t)stream>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_track_commit(int B, int max_tracks, int max_det, const int* count, const float* uv, const int* slot, const double* params,
                     int* tracks, float* rects, double* poses, void* stream) {
  if (!count || !uv || !slot || !params || !tracks || !rects || !poses) return fail_msg(SSP_ERR_ARG, "track_commit: null pointer");
  if (B < 0 || max_tracks < 1 || max_tracks > ssp_trk::kMaxTracks || max_det < 1 || max_det > ssp_det::kMaxInstances)
    return fail_msg(SSP_ERR_ARG, "track_commit: bad argument (B >= 0, 1 <= max_tracks <= 256, 1 <= max_det <= 256)");
  const long long n = (long long)B * max_det;
  if (n == 0) return SSP_OK;
  track_commit_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(B, max_tracks, max_det, count, uv, slot, params, tracks,
                                                                                    rects, poses);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
