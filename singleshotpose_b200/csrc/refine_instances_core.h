// Refinement of every world instance of a rig's capture against every camera's depth frame, with each depth pixel owned by the
// instance drawn in front of it: the rule of ssp_refine_instances_rig (refine_instances.cu), shared with the CPU test harness
// (tests/helpers/refine_instances_host.cpp, g++ -ffp-contract=off; the kernels are built with -fmad=false) and restated with whole
// arrays in oracle/refine_instances_ref.py.  fp64 but for the drawn vertices' fp32 pixels.  refine_depth_core.h, refine_rig_core.h,
// multiview_core.h and render_core.h are used unchanged.
//
// Problems.  One problem is world slot w of capture g, with ssp_fuse_instances' world_cls, R_world, t_world and fuse_status.  The
// slot is empty when w >= world_count[g] or its class lies outside [0, num_classes); its class's model points and diameter are
// ssp_refine_depth_rig's (model / offsets / diam), its faces are class-local vertex indices (faces / face_offsets).  A slot at
// w >= world_count[g] gets zeros and status 0, as in ssp_refine_depth_rig; a slot of an unknown class runs the rig rule with no
// points (SSP_REFINE_FEW_POINTS), as there.
// Iteration k (gate tau_k = d g_k as ssp_refine_depth_rig) has three steps.
//   1. Drawing set: every non-empty slot whose input_status (refine_rig_core.h) is 0, at the pose it holds when the iteration
//      starts: its current iterate while it runs, its input pose once a status bit has stopped it (the pose it will output).
//   2. Owner buffers: camera c of the capture gets O [H][W] uint64, all ones at the start.  Every face of every drawn instance:
//      its vertices mapped to camera c by ssp_mv::to_camera of the world pose, camera depth z = the third row of that pose
//      (ssp_mv::project's arithmetic), fp32 pixels by ssp_mv::project with camera c's fp64 K and coefficients (edges straight
//      between the distorted vertices); the face is skipped when a vertex has z <= 0 or a coordinate outside +-2^20 px
//      (render_core.h's vertex_status); the vertices are snapped and the triangle set up and tested with render_core.h's exact
//      int64 rule.  At a covered pixel centre the depth is z = 1 / ((l_0 / z_0 + l_1 / z_1) + l_2 / z_2), l_i = E_i / A each
//      multiplied by the fp64 1 / z_i, where E_i is the unbiased edge value of the edge opposite the clockwise vertex i and A the
//      triangle's doubled area (oracle.refine_depth_ref.render_depth_ref's weights).  The key (bits of (float)z) << 32 | w goes
//      into O = min(O, key): the minimum is independent of the order, so the lower slot wins a tie.
//   3. Pairing and solve: refine_rig_core.h's world_pair, and the pair is dropped (counted in view_hidden) when the pixel find_pair
//      read (recomputed here with its arithmetic, pair_pixel) has an owner other than w; pixels owned by w or by nobody keep the
//      rig's rule.  Each camera's kept pairs go into its accumulator in refine_depth_core.h's order, the cameras are added in
//      camera order and solve_update runs: ssp_refine_depth_rig's steps, status rules and "a status bit outputs the input pose".
// Outputs: ssp_refine_depth_rig's for every slot, view_hidden [C] (the pairs dropped for ownership in the last iteration that ran),
// and instance_map [H][W] int16 per frame: the owner of every pixel under the output poses, drawn once more after the last
// iteration, -1 where no instance is drawn.
// An owner buffer that holds only w or nobody rejects nothing, so a capture whose only drawn instance is w gives
// ssp_refine_depth_rig's outputs for w bit for bit (and with C = 1 and identity extrinsics ssp_refine_depth's).
// Only the libm functions sin and cos (so3_exp) may round differently on the device and the host.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "refine_rig_core.h"
#include "render_core.h"

namespace ssp_ri {

constexpr unsigned long long kNobody = ~0ull;
constexpr int kAcc = ssp_rr::kAcc + 1;        // the rig's accumulator, then the count of pairs dropped for ownership
constexpr int kOffHidden = ssp_rr::kAcc;

SSP_HD unsigned long long float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return (unsigned long long)__float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}

// the owner key of slot w at depth z (> 0): ordered by depth, then slot
SSP_HD unsigned long long owner_key(double z, int w) { return (float_bits((float)z) << 32) | (unsigned)w; }

// a slot is drawn when it is not empty and its input pose is usable
SSP_HD bool drawn(bool empty, const double R_in[9], const double t_in[3], int fuse_status) {
  return !empty && ssp_rr::input_status(R_in, t_in, fuse_status) == 0;
}

// vertex X [3] under the camera pose (Rc, tc): its fp32 pixel and camera depth; false when it stops its face from being drawn
SSP_HD bool draw_vertex(const double Rc[9], const double tc[3], const double* X, const double* Kd, const double* dist, float* u, float* v,
                        double* z) {
  *z = Rc[6] * X[0] + Rc[7] * X[1] + Rc[8] * X[2] + tc[2];
  if (!(*z > 0.0)) return false;
  ssp_mv::project(Rc, tc, X[0], X[1], X[2], Kd, dist, u, v);
  return ssp_render::vertex_status(*u, *v, *z) == 0;
}

// the unbiased edge value of edge i of a set-up triangle at the snapped centre (px, py)
SSP_HD long long edge_raw(const ssp_render::Tri& T, int i, long long px, long long py) {
  const int j = i == 2 ? 0 : i + 1;
  return (long long)(T.x[j] - T.x[i]) * (py - T.y[i]) - (long long)(T.y[j] - T.y[i]) * (px - T.x[i]);
}

// one face with drawn vertices (u, v, z [3]) in a W x H frame: visit(pixel index, depth) for every covered pixel centre
template <class F>
SSP_HD void draw_face(const float u[3], const float v[3], const double z[3], int W, int H, F visit) {
  ssp_render::Tri T;
  const int sx0 = ssp_render::snap(u[0]), sy0 = ssp_render::snap(v[0]), sx1 = ssp_render::snap(u[1]), sy1 = ssp_render::snap(v[1]);
  const int sx2 = ssp_render::snap(u[2]), sy2 = ssp_render::snap(v[2]);
  if (!ssp_render::tri_setup(sx0, sy0, sx1, sy1, sx2, sy2, T)) return;
  const long long area2 = (long long)(sx1 - sx0) * (sy2 - sy0) - (long long)(sy1 - sy0) * (sx2 - sx0);
  const bool flip = area2 < 0;                                    // tri_setup swapped vertices 1 and 2
  const double area = (double)(flip ? -area2 : area2);
  const double iz0 = 1.0 / z[0], iz1 = 1.0 / (flip ? z[2] : z[1]), iz2 = 1.0 / (flip ? z[1] : z[2]);
  int x0, y0, x1, y1;
  if (!ssp_render::tri_bbox(T, W, H, x0, y0, x1, y1)) return;
  for (int y = y0; y <= y1; y++)
    for (int x = x0; x <= x1; x++) {
      if (!ssp_render::covers(T, x, y)) continue;
      const long long px = (long long)x * ssp_render::kSubpixel, py = (long long)y * ssp_render::kSubpixel;
      const double l0 = (double)edge_raw(T, 1, px, py) / area, l1 = (double)edge_raw(T, 2, px, py) / area;
      const double l2 = (double)edge_raw(T, 0, px, py) / area;
      visit((long long)y * W + x, 1.0 / ((l0 * iz0 + l1 * iz1) + l2 * iz2));
    }
}

// face f (class-local vertex indices at face [3]) of a drawn instance with model rows x6 at `model` (its class's first row), under
// the camera pose (Rc, tc) of camera c: visit(pixel, depth) for every pixel it covers
template <class F>
SSP_HD void draw_model_face(const double* model, const int* face, const double Rc[9], const double tc[3], const double* Kd, const double* dist,
                            int W, int H, F visit) {
  float u[3], v[3];
  double z[3];
  for (int i = 0; i < 3; i++)
    if (!draw_vertex(Rc, tc, model + (long long)face[i] * 6, Kd, dist, u + i, v + i, z + i)) return;
  draw_face(u, v, z, W, H, visit);
}

// the pixel find_pair reads for model point x6 under the camera pose (R, t), with find_pair's arithmetic; call it only for a point
// find_pair paired (the pixel is then inside the frame)
SSP_HD long long pair_pixel(const double* x6, const double R[9], const double t[3], const ssp_rd::Camera& cam) {
  double p[3];
  for (int i = 0; i < 3; i++) p[i] = (R[3 * i] * x6[0] + R[3 * i + 1] * x6[1] + R[3 * i + 2] * x6[2]) + t[i];
  const double iz = 1.0 / p[2], xn = p[0] * iz, yn = p[1] * iz;
  double u, v;
  if (cam.dist) {
    double xd, yd;
    ssp_pnp::distort(cam.dist, xn, yn, &xd, &yd, nullptr);
    u = xd * cam.fx + cam.cx; v = yd * cam.fy + cam.cy;
  } else {
    u = xn * cam.fx + cam.cx; v = yn * cam.fy + cam.cy;
  }
  return (long long)floor(v + 0.5) * cam.W + (long long)floor(u + 0.5);
}

// add model point x6's world-axis pair in one camera to acc [kAcc] when it makes one and its pixel is not owned by another slot
// (ssp_rr::accumulate_point's additions); a pair dropped for ownership adds 1 to acc[kOffHidden]
SSP_HD void accumulate_point(const double* x6, const double R[9], const double t[3], const double Rc[9], const double tc[3], const ssp_mv::Cam& ext,
                             const ssp_rd::Camera& cam, const unsigned short* depth, const unsigned long long* owner, int w, double tau,
                             double* acc) {
  double r, J[6], qw[3];
  if (!ssp_rr::world_pair(x6, R, t, Rc, tc, ext, cam, depth, tau, &r, J, qw)) return;
  const unsigned long long key = owner[pair_pixel(x6, Rc, tc, cam)];
  if (key != kNobody && (unsigned)(key & 0xffffffffull) != (unsigned)w) {
    acc[kOffHidden] += 1.0;
    return;
  }
  int k = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) acc[k++] += J[i] * J[j];
  for (int i = 0; i < 6; i++) acc[ssp_rd::kOffJr + i] += J[i] * r;
  acc[ssp_rd::kOffR2] += r * r;
  acc[ssp_rd::kOffN] += 1.0;
}

// the instance map's entry of an owner key
SSP_HD short map_entry(unsigned long long key) { return key == kNobody ? (short)-1 : (short)(key & 0xffffffffull); }

}  // namespace ssp_ri
