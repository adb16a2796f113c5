// Silhouette masks of a triangle mesh under n poses: the rules shared by the kernels of render.cu and the CPU test harness
// (tests/helpers/render_host.cpp, built with g++).
//
// What a mask is:
//   * vertex positions are the fp32 pixel coordinates (u, v) that ssp_project_points returns for the same X, Rt and K
//     (render.cu calls that kernel), so a mask and a label file made from the same pose never disagree;
//   * each coordinate is snapped to 1/256 pixel, s = round-half-even(u * 256) -- exact: a power-of-two scale of an fp32 value,
//     then an integer -- and every edge function is evaluated in int64 on the snapped integers, so the mask depends on nothing
//     but (u, v): not on FMA contraction, the compiler or the platform;
//   * pixel (x, y) is covered when its centre, the point (x, y) of compute_projection's coordinates (the OpenCV convention:
//     pixel centres at integer coordinates), lies inside at least one non-degenerate triangle, of either winding;
//   * a centre exactly on an edge counts only for a top or a left edge (Direct3D's rule), so the triangles of a watertight mesh
//     leave no cracks and cover a shared edge once;
//   * a covered pixel is 255, any other 0 (LINEMOD's masks and the round(m / 255) tables of the image pipeline read 255 as the
//     object).  No depth test: the mask is the full silhouette, as LINEMOD's masks are.
//
// Status of a pose (any bit set -> that pose's mask is all zeros):
//   bit 0  a vertex at camera depth <= 0 (z of [R | t] X, explicit FMAs so every build computes the same bits);
//   bit 1  a projected coordinate that is not finite or lies outside +-2^20 px -- the guard that keeps snapped values within
//          +-2^28 and the edge functions (products of two differences of at most 2^29) exact in int64;
//   bit 2  a face index outside [0, nv) (the face is never read through).
//
// Orientation: with y pointing down, a triangle (a, b, c) whose cross product (b - a) x (c - a) is positive runs clockwise on
// screen; a negative one has b and c swapped first, and zero is degenerate (culled).  For a clockwise triangle the edge
// function of edge a -> b at p, E = (b.x - a.x)(p.y - a.y) - (b.y - a.y)(p.x - a.x), is positive inside; the edge is a top edge
// when it is horizontal and runs in +x (dy == 0, dx > 0) and a left edge when it runs up (dy < 0).  A centre is inside when
// every E > 0, or E == 0 on a top or left edge: E + bias >= 0 with bias = 0 on top-left edges and -1 on the others.
#pragma once
#include <math.h>
#include <stdint.h>
#if defined(__CUDACC__)
#define SSP_RENDER_HD __host__ __device__ __forceinline__
#else
#define SSP_RENDER_HD inline
#endif

namespace ssp_render {

constexpr int kTile = 32;                       // tile edge in pixels: one CTA per (pose, 32 x 32 tile)
constexpr int kThreads = 256;                   // threads of a tile CTA: 4 pixels each
constexpr int kMaxSize = 16384;                 // largest width / height (pixel coordinates fit int16)
constexpr float kGuard = 1048576.0f;            // 2^20 px
constexpr int kSubpixel = 256;                  // snapping grid: 1/256 px
enum { kBadDepth = 1, kBadCoord = 2, kBadFace = 4 };

// camera-frame depth of X under T = [R | t] (row-major [3][4]); w = 1 for 3-row X
SSP_RENDER_HD double camera_depth(const double* T, double x, double y, double z, double w) {
  return fma(T[8], x, fma(T[9], y, fma(T[10], z, T[11] * w)));
}

SSP_RENDER_HD int vertex_status(float u, float v, double depth) {
  int s = depth > 0.0 ? 0 : kBadDepth;                      // NaN depth counts as bad
  if (!(fabsf(u) <= kGuard) || !(fabsf(v) <= kGuard)) s |= kBadCoord;   // also catches NaN
  return s;
}

// round-half-even(u * 256) of a coordinate that passed the guard (|u| <= 2^20: the product is exact)
SSP_RENDER_HD int snap(float u) { return (int)rintf(u * (float)kSubpixel); }

SSP_RENDER_HD long long floor_div256(long long a) { return a >> 8; }          // arithmetic shift: floor for negatives too
SSP_RENDER_HD long long ceil_div256(long long a) { return -((-a) >> 8); }
SSP_RENDER_HD int min3(int a, int b, int c) { return a < b ? (a < c ? a : c) : (b < c ? b : c); }
SSP_RENDER_HD int max3(int a, int b, int c) { return a > b ? (a > c ? a : c) : (b > c ? b : c); }

// A triangle after set-up: clockwise vertices (snapped), and the pixel box of centres it can cover, clipped to the image.
struct Tri {
  int x[3], y[3];
};

// Orient (a, b, c) clockwise.  Returns false for a degenerate triangle (zero area).
SSP_RENDER_HD bool tri_setup(int ax, int ay, int bx, int by, int cx, int cy, Tri& t) {
  const long long area = (long long)(bx - ax) * (cy - ay) - (long long)(by - ay) * (cx - ax);
  if (area == 0) return false;
  t.x[0] = ax; t.y[0] = ay;
  if (area > 0) { t.x[1] = bx; t.y[1] = by; t.x[2] = cx; t.y[2] = cy; }
  else { t.x[1] = cx; t.y[1] = cy; t.x[2] = bx; t.y[2] = by; }
  return true;
}

// Pixel box [x0, x1] x [y0, y1] of the centres inside the triangle's bounding box, clipped to the W x H image.  Returns false
// when it is empty (the triangle covers no centre of the image).
SSP_RENDER_HD bool tri_bbox(const Tri& t, int W, int H, int& x0, int& y0, int& x1, int& y1) {
  const long long a = ceil_div256(min3(t.x[0], t.x[1], t.x[2])), b = floor_div256(max3(t.x[0], t.x[1], t.x[2]));
  const long long c = ceil_div256(min3(t.y[0], t.y[1], t.y[2])), d = floor_div256(max3(t.y[0], t.y[1], t.y[2]));
  x0 = (int)(a < 0 ? 0 : a); x1 = (int)(b > W - 1 ? W - 1 : b);
  y0 = (int)(c < 0 ? 0 : c); y1 = (int)(d > H - 1 ? H - 1 : d);
  return x0 <= x1 && y0 <= y1;
}

// Edge i runs from vertex i to vertex (i + 1) % 3.  E(px, py) = A px + B py + C with A = -dy, B = dx; `bias` folds the tie rule.
SSP_RENDER_HD bool top_left(int dx, int dy) { return (dy == 0 && dx > 0) || dy < 0; }

// E + bias at the snapped point (px, py) = 256 * (x, y); inside when >= 0
SSP_RENDER_HD long long edge_value(const Tri& t, int i, long long px, long long py) {
  const int j = i == 2 ? 0 : i + 1;
  const int dx = t.x[j] - t.x[i], dy = t.y[j] - t.y[i];
  return (long long)dx * (py - t.y[i]) - (long long)dy * (px - t.x[i]) + (top_left(dx, dy) ? 0 : -1);
}

SSP_RENDER_HD bool covers(const Tri& t, int x, int y) {
  const long long px = (long long)x * kSubpixel, py = (long long)y * kSubpixel;
  return edge_value(t, 0, px, py) >= 0 && edge_value(t, 1, px, py) >= 0 && edge_value(t, 2, px, py) >= 0;
}

}  // namespace ssp_render
