// Silhouette masks of a triangle mesh under n poses, for making a training set from camera poses (the mask/<n>.png files that
// image.py:131,135 opens for every training image).  The rules -- what a mask is, the snapping, the edge functions, the
// top-left tie rule and the status bits -- are in render_core.h.
//
// Per call, five steps on one stream (the face and tile kernels once per 65535 poses):
//   1. ssp_project_points (pnp.cu): the fp32 pixel coordinates of every vertex under every pose -- the very numbers the label
//      files are made from;
//   2. render_init_kernel: status[p] = 0 and an empty pose box;
//   3. render_vertex_kernel: one thread per (pose, vertex): the depth and guard-band checks, OR-ed into status[p];
//   4. render_face_kernel: one thread per (pose, face): the face-index check, snap, orientation, the pixel box of the centres
//      the triangle can cover (clipped to the image); degenerate and off-screen triangles get an empty box.  The pose box is
//      the union of the triangle boxes (reduced over each warp, then atomicMin / atomicMax: order-independent);
//   5. render_tile_kernel: one CTA per (pose, 32 x 32 tile), 256 threads, 4 pixels each (one column, rows 8 apart).  A tile
//      outside the pose box, or of a pose with a status bit, writes zeros without reading a triangle.  Otherwise the CTA
//      streams the pose's triangle boxes in batches of 256, keeps those that overlap the tile in shared memory as three edge
//      functions at the tile origin plus its pixel box, and every thread whose pixels meet that box tests them against the
//      edge functions (the triangles of a LINEMOD-sized mesh at 640 x 480 span a pixel or two, so most threads skip most
//      triangles); the CTA stops early once every pixel of the tile is covered.  Every mask byte is written once, by the thread
//      that owns the pixel: no atomics on the output, and the mask does not depend on the order of the triangles (coverage is
//      an OR).  Measured (tools/bench_render.py, H100 80GB HBM3 at 700 W, 12000 faces, 640 x 480, n = 1024): this kernel takes
//      7.7 of the 8.3 ms, 9.0 ms before the per-thread box test; what remains is every active tile streaming all nf boxes of
//      its pose, so tile binning (count, scan, scatter the triangles per tile) is the next step.
#include <limits.h>

#include "ssp_common.cuh"
#include "render_core.h"

namespace ssp {
using namespace ssp_render;

struct RenderWork {
  float* uv;          // [n][2][nv]  projected coordinates
  short4* boxes;      // [n][nf]     pixel box of each triangle (x0, y0, x1, y1); empty: x0 > x1
  Tri* tris;          // [n][nf]     clockwise snapped vertices
  int4* pbox;         // [n]         union of the triangle boxes
};

static long long align256(long long b) { return (b + 255) & ~255LL; }

static bool render_sizes_ok(int rows, int nv, int nf, long long n, int W, int H) {
  return (rows == 3 || rows == 4) && nv >= 3 && nf >= 1 && n >= 0 && n <= INT_MAX && W >= 1 && W <= kMaxSize && H >= 1 &&
         H <= kMaxSize;
}

static long long render_work_layout(int nv, int nf, long long n, char* base, RenderWork* w) {
  const long long b_uv = align256(n * 2 * nv * (long long)sizeof(float));
  const long long b_box = align256(n * nf * (long long)sizeof(short4));
  const long long b_tri = align256(n * nf * (long long)sizeof(Tri));
  const long long b_pb = align256(n * (long long)sizeof(int4));
  if (w) {
    w->uv = reinterpret_cast<float*>(base);
    w->boxes = reinterpret_cast<short4*>(base + b_uv);
    w->tris = reinterpret_cast<Tri*>(base + b_uv + b_box);
    w->pbox = reinterpret_cast<int4*>(base + b_uv + b_box + b_tri);
  }
  return b_uv + b_box + b_tri + b_pb;
}

__global__ void render_init_kernel(long long n, int W, int H, int* __restrict__ status, int4* __restrict__ pbox) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  status[p] = 0;
  pbox[p] = make_int4(W, H, -1, -1);
}

__global__ void render_vertex_kernel(const float* __restrict__ X, int rows, int nv, const double* __restrict__ Rt,
                                     const float* __restrict__ uv, long long n, int* __restrict__ status) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * nv) return;
  const long long p = idx / nv;
  const int v = (int)(idx % nv);
  const double w = rows == 4 ? (double)X[3LL * nv + v] : 1.0;
  const double z = camera_depth(Rt + 12 * p, X[v], X[nv + v], X[2LL * nv + v], w);
  const int s = vertex_status(uv[(2 * p) * nv + v], uv[(2 * p + 1) * nv + v], z);
  if (s) atomicOr(status + p, s);
}

// grid (face blocks, poses p0 + blockIdx.y): every warp belongs to one pose, so the pose box is reduced over the warp first and
// one lane does the four atomics (one set per triangle would serialise n * nf atomics on 4 n addresses)
__global__ void __launch_bounds__(256) render_face_kernel(const float* __restrict__ uv, int nv, const int* __restrict__ faces, int nf,
                                                          long long p0, int W, int H, int* __restrict__ status, short4* __restrict__ boxes,
                                                          Tri* __restrict__ tris, int4* __restrict__ pbox) {
  const long long p = p0 + blockIdx.y;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const long long idx = p * nf + f;
  int x0 = W, y0 = H, x1 = -1, y1 = -1;                       // the identity of the box union
  if (f < nf) {
    short4 box = make_short4(SHRT_MAX, SHRT_MAX, -1, -1);     // empty
    int vi[3];
    bool ok = true;
    for (int k = 0; k < 3; k++) {
      vi[k] = faces[3LL * f + k];
      ok &= vi[k] >= 0 && vi[k] < nv;
    }
    if (!ok) atomicOr(status + p, kBadFace);
    const float* u = uv + 2 * p * nv;
    int sx[3], sy[3];
    for (int k = 0; k < 3 && ok; k++) {
      const float a = u[vi[k]], b = u[nv + vi[k]];
      ok = vertex_status(a, b, 1.0) == 0;                     // else the pose is flagged by render_vertex_kernel
      sx[k] = ok ? snap(a) : 0;
      sy[k] = ok ? snap(b) : 0;
    }
    Tri t;
    int bx0, by0, bx1, by1;
    if (ok && tri_setup(sx[0], sy[0], sx[1], sy[1], sx[2], sy[2], t) && tri_bbox(t, W, H, bx0, by0, bx1, by1)) {
      tris[idx] = t;
      box = make_short4((short)bx0, (short)by0, (short)bx1, (short)by1);
      x0 = bx0; y0 = by0; x1 = bx1; y1 = by1;
    }
    boxes[idx] = box;
  }
  x0 = __reduce_min_sync(0xffffffffu, x0); y0 = __reduce_min_sync(0xffffffffu, y0);
  x1 = __reduce_max_sync(0xffffffffu, x1); y1 = __reduce_max_sync(0xffffffffu, y1);
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    int* pb = reinterpret_cast<int*>(pbox + p);
    atomicMin(pb, x0); atomicMin(pb + 1, y0); atomicMax(pb + 2, x1); atomicMax(pb + 3, y1);
  }
}

// the three edge functions of a triangle at the tile origin (bias folded in) and their steps per pixel
struct TileTri {
  long long e0[3];
  int a[3], b[3];       // dE per pixel in x (-256 dy) and in y (256 dx) are a * 256, b * 256
  short4 box;           // the centres the triangle can cover: a thread outside it skips the edge functions
};

__global__ void __launch_bounds__(kThreads) render_tile_kernel(const short4* __restrict__ boxes, const Tri* __restrict__ tris,
                                                               const int4* __restrict__ pbox, const int* __restrict__ status, int nf,
                                                               int W, int H, int tiles_x, long long p0, unsigned char* __restrict__ masks) {
  __shared__ TileTri s_tri[kThreads];
  __shared__ int s_n;
  const long long p = p0 + blockIdx.y;
  const int t = threadIdx.x, lx = t & (kTile - 1), ly = t / kTile;
  const int tx0 = (int)(blockIdx.x % tiles_x) * kTile, ty0 = (int)(blockIdx.x / tiles_x) * kTile;
  const int tx1 = min(tx0 + kTile, W) - 1, ty1 = min(ty0 + kTile, H) - 1;
  constexpr int kRows = kTile * kTile / kThreads;              // pixels per thread, rows kThreads / kTile apart
  constexpr int kRowStep = kThreads / kTile;
  const int x = tx0 + lx;
  unsigned done = 0;                                           // bit k: pixel k is covered or outside the image
#pragma unroll
  for (int k = 0; k < kRows; k++)
    if (x >= W || ty0 + ly + kRowStep * k >= H) done |= 1u << k;
  unsigned cov = 0;
  const int4 pb = pbox[p];
  const bool active = status[p] == 0 && pb.x <= tx1 && pb.z >= tx0 && pb.y <= ty1 && pb.w >= ty0;
  if (active) {
    const long long ox = (long long)tx0 * kSubpixel, oy = (long long)ty0 * kSubpixel;
    const short4* bx = boxes + p * nf;
    const Tri* tr = tris + p * nf;
    for (int base = 0; base < nf; base += kThreads) {
      if (t == 0) s_n = 0;
      __syncthreads();
      const int i = base + t;
      if (i < nf) {
        const short4 b = bx[i];
        if (b.x <= tx1 && b.z >= tx0 && b.y <= ty1 && b.w >= ty0) {
          const Tri tri = tr[i];
          TileTri e;
          e.box = b;
#pragma unroll
          for (int k = 0; k < 3; k++) {
            e.e0[k] = edge_value(tri, k, ox, oy);
            const int j = k == 2 ? 0 : k + 1;
            e.a[k] = -(tri.y[j] - tri.y[k]);
            e.b[k] = tri.x[j] - tri.x[k];
          }
          s_tri[atomicAdd(&s_n, 1)] = e;
        }
      }
      __syncthreads();
      const int cnt = s_n;
      if (done != (1u << kRows) - 1) {
        for (int j = 0; j < cnt; j++) {
          const TileTri& e = s_tri[j];
          if (x < e.box.x || x > e.box.z || ty0 + ly + kRowStep * (kRows - 1) < e.box.y || ty0 + ly > e.box.w) continue;
          long long ev[3];
#pragma unroll
          for (int k = 0; k < 3; k++)
            ev[k] = e.e0[k] + (long long)e.a[k] * (kSubpixel * lx) + (long long)e.b[k] * (kSubpixel * ly);
#pragma unroll
          for (int r = 0; r < kRows; r++) {
            if (ev[0] >= 0 && ev[1] >= 0 && ev[2] >= 0) cov |= 1u << r;
#pragma unroll
            for (int k = 0; k < 3; k++) ev[k] += (long long)e.b[k] * (kSubpixel * kRowStep);
          }
        }
        done |= cov;
      }
      if (__syncthreads_and(done == (1u << kRows) - 1)) break;   // also orders this batch's reads before the next batch's writes
    }
  }
  if (x < W) {
    unsigned char* m = masks + p * (long long)W * H;
#pragma unroll
    for (int r = 0; r < kRows; r++) {
      const int y = ty0 + ly + kRowStep * r;
      if (y < H) m[(long long)y * W + x] = (cov >> r) & 1 ? 255 : 0;
    }
  }
}

}  // namespace ssp

using namespace ssp;

extern "C" {
long long ssp_render_work_bytes(int nv, int nf, long long n, int W, int H) {
  if (!render_sizes_ok(3, nv, nf, n, W, H)) return SSP_ERR_ARG;
  const long long per_pose = render_work_layout(nv, nf, 1, nullptr, nullptr);
  if (n > (LLONG_MAX / 2) / per_pose) return SSP_ERR_ARG;
  return render_work_layout(nv, nf, n, nullptr, nullptr);
}

int ssp_render_masks(const float* X, int rows, int nv, const int* faces, int nf, const double* Rt, const double* K, long long n,
                     int W, int H, unsigned char* masks, int* status, void* work, long long work_bytes, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (!X || !faces || !Rt || !K || !masks || !status || !work)
    return fail_msg(SSP_ERR_ARG, "render_masks: bad argument (null pointer)");
  if (!render_sizes_ok(rows, nv, nf, n, W, H))
    return fail_msg(SSP_ERR_ARG, "render_masks: bad argument (rows not 3 or 4, nv < 3, nf < 1, n < 0, or W, H outside [1, 16384])");
  const long long need = ssp_render_work_bytes(nv, nf, n, W, H);
  if (need < 0 || work_bytes < need) return fail_msg(SSP_ERR_ARG, "render_masks: work buffer smaller than ssp_render_work_bytes()");
  if (n == 0) return SSP_OK;
  RenderWork w;
  render_work_layout(nv, nf, n, static_cast<char*>(work), &w);
  const int rc = ssp_project_points(X, rows, nv, Rt, K, n, w.uv, stream);
  if (rc != SSP_OK) return rc;
  render_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(n, W, H, status, w.pbox);
  SSP_CHECK_LAUNCH();
  render_vertex_kernel<<<(unsigned)((n * nv + 255) / 256), 256, 0, s>>>(X, rows, nv, Rt, w.uv, n, status);
  SSP_CHECK_LAUNCH();
  const int tiles_x = (W + kTile - 1) / kTile, tiles = tiles_x * ((H + kTile - 1) / kTile);
  for (long long p0 = 0; p0 < n; p0 += 65535) {                // gridDim.y <= 65535 poses per launch
    const unsigned np = (unsigned)(n - p0 < 65535 ? n - p0 : 65535);
    render_face_kernel<<<dim3((unsigned)((nf + 255) / 256), np), 256, 0, s>>>(w.uv, nv, faces, nf, p0, W, H, status, w.boxes, w.tris,
                                                                               w.pbox);
    SSP_CHECK_LAUNCH();
  }
  for (long long p0 = 0; p0 < n; p0 += 65535) {
    const unsigned np = (unsigned)(n - p0 < 65535 ? n - p0 : 65535);
    render_tile_kernel<<<dim3((unsigned)tiles, np), kThreads, 0, s>>>(w.boxes, w.tris, w.pbox, status, nf, W, H, tiles_x, p0, masks);
    SSP_CHECK_LAUNCH();
  }
  return SSP_OK;
}
}  // extern "C"
