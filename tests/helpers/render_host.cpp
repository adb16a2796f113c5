// Host harness of the silhouette rules of render_core.h: the same status checks, snapping, set-up and coverage test as
// render.cu, driven with plain loops and the direct edge functions (render_tile_kernel evaluates them incrementally from the
// tile origin; both are exact integers, so both give the same masks).  Test infrastructure: built by the render tests into a
// temporary .so; never loaded by the product.
#include <string.h>

#include "../../singleshotpose_b200/csrc/render_core.h"

using namespace ssp_render;

extern "C" {
// X [rows][nv]; faces [nf][3]; Rt [n][3][4]; uv [n][2][nv], the projected coordinates; masks [n][H][W]; status [n]
int h_render_masks(const float* X, int rows, int nv, const int* faces, int nf, const double* Rt, const float* uv, long long n, int W,
                   int H, unsigned char* masks, int* status) {
  if ((rows != 3 && rows != 4) || nv < 3 || nf < 1 || n < 0 || W < 1 || W > kMaxSize || H < 1 || H > kMaxSize) return -1;
  for (long long p = 0; p < n; p++) {
    const float* u = uv + 2 * p * nv;
    unsigned char* m = masks + p * (long long)W * H;
    memset(m, 0, (size_t)W * H);
    int s = 0;
    for (int v = 0; v < nv; v++) {
      const double w = rows == 4 ? (double)X[3LL * nv + v] : 1.0;
      s |= vertex_status(u[v], u[nv + v], camera_depth(Rt + 12 * p, X[v], X[nv + v], X[2LL * nv + v], w));
    }
    for (int f = 0; f < nf; f++)
      for (int k = 0; k < 3; k++)
        if (faces[3LL * f + k] < 0 || faces[3LL * f + k] >= nv) s |= kBadFace;
    status[p] = s;
    if (s) continue;
    for (int f = 0; f < nf; f++) {
      const int* fi = faces + 3LL * f;
      Tri t;
      int x0, y0, x1, y1;
      if (!tri_setup(snap(u[fi[0]]), snap(u[nv + fi[0]]), snap(u[fi[1]]), snap(u[nv + fi[1]]), snap(u[fi[2]]), snap(u[nv + fi[2]]), t) ||
          !tri_bbox(t, W, H, x0, y0, x1, y1))
        continue;
      for (int y = y0; y <= y1; y++)
        for (int x = x0; x <= x1; x++)
          if (covers(t, x, y)) m[(long long)y * W + x] = 255;
    }
  }
  return 0;
}
}
