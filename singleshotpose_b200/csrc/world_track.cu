// Tracking the world instances of a camera rig over time (rules: world_track_core.h).  Two launches after ssp_fuse_instances, both
// fed from device memory (the fusion's outputs), so a graph replay needs no host read-back:
//   ssp_world_track_associate  steps 1-4, one CTA per stream, one thread per track slot.  Every thread predicts its slot's filter
//                              (with motion) and stages the slot and its position in shared memory; warp 0 then walks the world
//                              instances serially (a matched track is taken), each one a warp arg-min of (d2, slot) over the slots
//                              (lane l owns slots l, l + 32, ...; shuffles, no block barrier), ages the tracks and lists the free
//                              slots in ascending order with ballots, the k-th unmatched instance taking the k-th.  Last, every
//                              thread writes the slots back and gathers each detection's track id through world_index.
//   ssp_world_track_commit     step 5, one thread per world slot: a track slot is matched or born by at most one instance per capture.
// Built with -fmad=false, as the host harness is built with -ffp-contract=off.
#include <math.h>

#include "ssp_common.cuh"
#include "world_track_core.h"

namespace ssp {

static_assert(ssp_wt::kFuseSingular == SSP_FUSE_SINGULAR, "world_track_core.h reads ssp_fuse_instances' singular bit");
static_assert(ssp_pf::kFilterDoubles == SSP_FILTER_DOUBLES, "the filter layout of pose_filter_core.h");

constexpr int kWtWarp = 32;
constexpr int kWtMaxThreads = ssp_wt::kMaxTracks;

struct WorldTrackParams {
  const int* world_count; const int* world_cls; const double* t_world; const int* world_index; const double* class_size;
  const double* poses; const double* dt;
  int* tracks; double* filter; int* next_id; int* wslot; int* world_track_id; int* matched; int* track_id;
  ssp_pf::FilterParams fp;
  double match_dist;
  int C, T, M, num_classes, max_misses;
};

__global__ void __launch_bounds__(kWtMaxThreads) world_track_associate_kernel(const WorldTrackParams p) {
  using namespace ssp_wt;
  __shared__ int s_st[kMaxTracks * kFields];
  __shared__ double s_pos[kMaxTracks * 3];
  __shared__ unsigned char s_taken[kMaxTracks];
  __shared__ int s_free[kMaxTracks];
  __shared__ double s_wt[kMaxWorld * 3];
  __shared__ double s_r2[kMaxWorld];
  __shared__ int s_wcls[kMaxWorld];
  __shared__ int s_wslot[kMaxWorld];
  __shared__ int s_wid[kMaxWorld];
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, T = p.T, M = p.M;
  const int n = min(max(p.world_count[g], 0), M);
  int* st = p.tracks + (long long)g * T * kFields;
  for (int i = tid; i < T * kFields; i += nt) s_st[i] = st[i];
  __syncthreads();
  // 1. predict, and each slot's position
  for (int s = tid; s < T; s += nt) {
    const long long ts = (long long)g * T + s;
    double* f = p.filter ? p.filter + ts * ssp_pf::kFilterDoubles : nullptr;
    if (f) predict_slot(s_st + s * kFields, f, p.dt[g], p.fp);
    const double* q = position(p.poses + ts * kPoseDoubles, f);
    for (int i = 0; i < 3; i++) s_pos[s * 3 + i] = q[i];
    s_taken[s] = 0;
  }
  for (int w = tid; w < n; w += nt) {
    const long long gw = (long long)g * M + w;
    const int k = p.world_cls[gw];
    s_wcls[w] = k;
    for (int i = 0; i < 3; i++) s_wt[w * 3 + i] = p.t_world[gw * 3 + i];
    s_r2[w] = tracked_class(k, p.num_classes) ? radius2(p.match_dist, p.class_size[k]) : 0.0;
    s_wslot[w] = -1;
  }
  __syncthreads();
  if (tid < kWtWarp) {
    const int lane = tid;
    // 2. match
    for (int w = 0; w < n; w++) {
      const int k = s_wcls[w];
      double best = 0.0;
      int bs = -1;
      if (tracked_class(k, p.num_classes))
        for (int s = lane; s < T; s += kWtWarp) {
          const double d2 = dist2(s_wt + w * 3, s_pos + s * 3);
          if (can_match(s_st + s * kFields, s_taken[s], k, d2, s_r2[w]) && closer(d2, s, best, bs)) { best = d2; bs = s; }
        }
      for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, best, o);
        const int os = __shfl_xor_sync(0xffffffffu, bs, o);
        if (os >= 0 && closer(od, os, best, bs)) { best = od; bs = os; }
      }
      if (bs >= 0 && lane == 0) { s_taken[bs] = 1; s_wslot[w] = bs; }
      __syncwarp();
    }
    // 3. age
    for (int s = lane; s < T; s += kWtWarp) {
      int* f = s_st + s * kFields;
      if (f[kAlive] && !s_taken[s]) {
        f[kMisses] += 1;
        if (ssp_trk::dies(f[kMisses], p.max_misses)) f[kAlive] = 0;
      }
    }
    __syncwarp();
    // 4. birth: the free slots in ascending order, then the k-th unmatched instance takes the k-th
    int nfree = 0;
    for (int s0 = 0; s0 < T; s0 += kWtWarp) {
      const int s = s0 + lane;
      const bool fr = s < T && !s_st[s * kFields + kAlive];
      const unsigned bal = __ballot_sync(0xffffffffu, fr);
      if (fr) s_free[nfree + __popc(bal & ((1u << lane) - 1u))] = s;
      nfree += __popc(bal);
    }
    __syncwarp();
    const int id0 = p.next_id[g];
    int born = 0;
    for (int w0 = 0; w0 < M; w0 += kWtWarp) {
      const int w = w0 + lane;
      const bool hit = w < n && s_wslot[w] >= 0;
      const bool um = w < n && !hit && tracked_class(s_wcls[w], p.num_classes);
      const unsigned bal = __ballot_sync(0xffffffffu, um);
      const int k = born + __popc(bal & ((1u << lane) - 1u));
      int sl = hit ? s_wslot[w] : -1, id = hit ? s_st[sl * kFields + kId] : -1;
      if (um && k < nfree) {
        sl = s_free[k];
        id = id0 + k;
        int* f = s_st + sl * kFields;
        f[kAlive] = 1; f[kId] = id; f[kCls] = s_wcls[w]; f[kMisses] = 0; f[kHits] = 0;
      }
      if (w < M) {
        const long long gw = (long long)g * M + w;
        p.wslot[gw] = sl;
        p.world_track_id[gw] = id;
        p.matched[gw] = hit;
        s_wid[w] = id;
      }
      born += __popc(bal);
    }
    if (lane == 0) p.next_id[g] = id0 + min(born, nfree);
  }
  __syncthreads();
  for (int i = tid; i < T * kFields; i += nt) st[i] = s_st[i];
  // each detection of the capture: its world instance's track id
  const long long r0 = (long long)g * p.C * M;
  for (int i = tid; i < p.C * M; i += nt) {
    const int w = p.world_index[r0 + i];
    p.track_id[r0 + i] = w >= 0 && w < n ? s_wid[w] : -1;
  }
}

__global__ void __launch_bounds__(128) world_track_commit_kernel(int G, int T, int M, const int* __restrict__ world_count,
                                                                  const double* __restrict__ R_world, const double* __restrict__ t_world,
                                                                  const double* __restrict__ world_cov, const int* __restrict__ fuse_status,
                                                                  const int* __restrict__ wslot, const int* __restrict__ matched,
                                                                  int* __restrict__ tracks, double* __restrict__ poses, double* __restrict__ filter,
                                                                  const ssp_pf::FilterParams fp, double* __restrict__ R_filt,
                                                                  double* __restrict__ t_filt, double* __restrict__ pose_cov,
                                                                  double* __restrict__ velocity, int* __restrict__ reinit) {
  using namespace ssp_wt;
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)G * M) return;
  const int g = (int)(o / M), w = (int)(o % M);
  const int s = w < min(max(world_count[g], 0), M) ? wslot[o] : -1;
  const long long ts = (long long)g * T + s;
  if (s >= 0) store(tracks + ts * kFields, poses + ts * kPoseDoubles, R_world + o * 9, t_world + o * 3);
  if (filter)
    filter_slot(s < 0 ? nullptr : filter + ts * ssp_pf::kFilterDoubles, matched[o] != 0, R_world + o * 9, t_world + o * 3, world_cov + o * 36,
                fuse_status[o], fp, R_filt + o * 9, t_filt + o * 3, pose_cov + o * 36, velocity + o * 6, reinit + o);
}

static inline bool positive_finite(double x) { return x > 0.0 && isfinite(x); }

static bool bad_sizes(int groups, int max_tracks, int slots) {
  return groups < 0 || max_tracks < 1 || max_tracks > ssp_wt::kMaxTracks || slots < 1 || slots > ssp_wt::kMaxWorld;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_world_track_associate(int groups, int views, int max_tracks, int slots, const int* world_count, const int* world_cls,
                              const double* t_world, const int* world_index, const double* class_size, int num_classes, double match_dist,
                              int max_misses, int* tracks, const double* poses, double* filter, const double* dt, double accel_sigma_rot,
                              double accel_sigma_trans, int* next_id, int* wslot, int* world_track_id, int* matched, int* track_id,
                              void* stream) {
  if (!world_count || !world_cls || !t_world || !world_index || !class_size || !tracks || !poses || !next_id || !wslot || !world_track_id ||
      !matched || !track_id || (!filter) != (!dt))
    return fail_msg(SSP_ERR_ARG, "world_track_associate: null pointer (filter and dt are both given or both null)");
  if (bad_sizes(groups, max_tracks, slots))
    return fail_msg(SSP_ERR_ARG, "world_track_associate: bad size (groups >= 0, 1 <= max_tracks <= 256, 1 <= slots <= 256)");
  if (views < 1 || views > SSP_RIG_MAX_VIEWS || num_classes < 1 || max_misses < 0)
    return fail_msg(SSP_ERR_ARG, "world_track_associate: bad argument (1 <= views <= 16, num_classes >= 1, max_misses >= 0)");
  if (!positive_finite(match_dist) || !positive_finite(accel_sigma_rot) || !positive_finite(accel_sigma_trans))
    return fail_msg(SSP_ERR_ARG, "world_track_associate: match_dist and the acceleration sigmas must be > 0 and finite");
  if (groups == 0) return SSP_OK;
  WorldTrackParams p;
  p.world_count = world_count; p.world_cls = world_cls; p.t_world = t_world; p.world_index = world_index; p.class_size = class_size;
  p.poses = poses; p.dt = dt; p.tracks = tracks; p.filter = filter; p.next_id = next_id; p.wslot = wslot; p.world_track_id = world_track_id;
  p.matched = matched; p.track_id = track_id;
  p.fp = ssp_pf::FilterParams{accel_sigma_rot * accel_sigma_rot, accel_sigma_trans * accel_sigma_trans, 0.0, 0.0, 0.0};
  p.match_dist = match_dist;
  p.C = views; p.T = max_tracks; p.M = slots; p.num_classes = num_classes; p.max_misses = max_misses;
  const int threads = (max_tracks + kWtWarp - 1) / kWtWarp * kWtWarp;
  world_track_associate_kernel<<<(unsigned)groups, threads, 0, (cudaStream_t)stream>>>(p);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}

int ssp_world_track_commit(int groups, int max_tracks, int slots, const int* world_count, const double* R_world, const double* t_world,
                           const double* world_cov, const int* fuse_status, const int* wslot, const int* matched, int* tracks, double* poses,
                           double* filter, double init_velocity_sigma_rot, double init_velocity_sigma_trans, double gate, double* R_filt,
                           double* t_filt, double* pose_cov, double* velocity, int* reinit, void* stream) {
  if (!world_count || !R_world || !t_world || !world_cov || !fuse_status || !wslot || !matched || !tracks || !poses ||
      (filter && (!R_filt || !t_filt || !pose_cov || !velocity || !reinit)))
    return fail_msg(SSP_ERR_ARG, "world_track_commit: null pointer (with a filter, every filter output is required)");
  if (bad_sizes(groups, max_tracks, slots))
    return fail_msg(SSP_ERR_ARG, "world_track_commit: bad size (groups >= 0, 1 <= max_tracks <= 256, 1 <= slots <= 256)");
  if (!positive_finite(init_velocity_sigma_rot) || !positive_finite(init_velocity_sigma_trans) || !positive_finite(gate))
    return fail_msg(SSP_ERR_ARG, "world_track_commit: the initial velocity sigmas and the gate must be > 0 and finite");
  const long long n = (long long)groups * slots;
  if (n == 0) return SSP_OK;
  const ssp_pf::FilterParams fp = {0.0, 0.0, init_velocity_sigma_rot * init_velocity_sigma_rot,
                                   init_velocity_sigma_trans * init_velocity_sigma_trans, gate};
  world_track_commit_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(groups, max_tracks, slots, world_count, R_world,
                                                                                          t_world, world_cov, fuse_status, wslot, matched,
                                                                                          tracks, poses, filter, fp, R_filt, t_filt,
                                                                                          pose_cov, velocity, reinit);
  SSP_CHECK_LAUNCH(); return SSP_OK;
}
}  // extern "C"
