// Training-image pipeline on the GPU: change_background + data_augmentation + ToTensor of the reference
// (image.py:110-127, 46-75, 14-32; dataset.py:100-109), byte-exact with the Pillow routines those functions call.
// Compiled with -fmad=false: the coefficient set-up (double) and the HSV conversions (float/double) must round operation by
// operation exactly like the C originals.  All arithmetic and the pass sequencing live in augment_core.h, which the CPU
// test-suite compiles for the host and checks against Pillow; this file only maps output pixels to threads.
// HBM-bound byte work (about 2.4 MB in, 2.1 MB out per 640x480 -> 416x416 sample); one thread per output pixel,
// consecutive threads on consecutive pixels (coalesced 3-byte RGB rows), tables in shared memory.
#include "ssp_common.cuh"
#include "augment_core.h"
#include <stdio.h>

namespace ssp {
using namespace ssp_aug;

__global__ void aug_coeffs_kernel(int in_size, int in0, int in1, int out_size, int resample, int ksize, int* __restrict__ bounds,
                                  int* __restrict__ kk) {
  const int xx = blockIdx.x * blockDim.x + threadIdx.x;
  if (xx < out_size) coeff_row(in_size, in0, in1, out_size, resample, ksize, xx, bounds + 2 * xx, kk + (long long)xx * ksize);
}

__global__ void aug_pass_kernel(const PassArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < a.dst_w && y < a.dst_h) resample_pass_px(a, x, y);
}

__global__ void aug_nearest_kernel(const PassArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < a.dst_w && y < a.dst_h) nearest_px(a, x, y);
}

// mode 1: rgb -> hsv only ; 2: hsv -> rgb only (the halves of distort_px, for exhaustive parity tests)
__global__ void aug_distort_kernel(const uint8_t* __restrict__ src, long long n_px, int mode, uint8_t* __restrict__ out_u8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_px; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t* s = src + 3 * i;
    uint8_t o[3];
    if (mode == 1) rgb2hsv_px(s[0], s[1], s[2], o);
    else hsv2rgb_px(s[0], s[1], s[2], o);
    out_u8[3 * i] = o[0]; out_u8[3 * i + 1] = o[1]; out_u8[3 * i + 2] = o[2];
  }
}

// torchvision ToTensor of a dense uint8 HWC RGB image: float32 CHW planes, byte / 255 as an IEEE division (dataset.py:103-118 transform)
__global__ void aug_to_tensor_kernel(const uint8_t* __restrict__ src, long long n_px, float* __restrict__ out_chw) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_px; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t* s = src + 3 * i;
    out_chw[i] = (float)s[0] / 255.0f;
    out_chw[n_px + i] = (float)s[1] / 255.0f;
    out_chw[2 * n_px + i] = (float)s[2] / 255.0f;
  }
}

// one STAGE of a batch: op table column per sample (blockIdx.z), one thread per element of the op's (nx, ny) extent
__global__ void __launch_bounds__(256) aug_stage_kernel(const AugOp* __restrict__ ops) {
  const AugOp& op = ops[blockIdx.z];
  if (op.kind == OP_NONE) return;                  // uniform per block: the whole block works on one sample's op
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (op.kind == OP_COUNT) {
    // overlap counts of a multi-object candidate: warp sums, then one integer atomic per warp with a non-zero sum, so the
    // per-sample totals do not depend on the order of the additions
    unsigned s = 0, i = 0;
    if (x < op.nx && y < op.ny) count_px(op, x, y, &s, &i);
    s = __reduce_add_sync(0xffffffffu, s);
    i = __reduce_add_sync(0xffffffffu, i);
    if ((threadIdx.x & 31) == 0) {
      if (s) atomicAdd(op.counts, s);
      if (i) atomicAdd(op.counts + 1, i);
    }
    return;
  }
  op_element(op, x, y);
}

namespace {
inline int blocks_for(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  const long long cap = (long long)ssp_sm_count() * 16;      // grid-stride: a few waves of the device's SMs
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}
struct CudaBackend {
  cudaStream_t s;
  void coeffs(int in_size, int in0, int in1, int out_size, int resample, int ksize, int* bounds, int* kk) {
    aug_coeffs_kernel<<<(out_size + 127) / 128, 128, 0, s>>>(in_size, in0, in1, out_size, resample, ksize, bounds, kk);
  }
  void pass(const PassArgs& a) {
    dim3 b(32, 8), g((a.dst_w + 31) / 32, (a.dst_h + 7) / 8);
    aug_pass_kernel<<<g, b, 0, s>>>(a);
  }
  void nearest(const PassArgs& a) {
    dim3 b(32, 8), g((a.dst_w + 31) / 32, (a.dst_h + 7) / 8);
    aug_nearest_kernel<<<g, b, 0, s>>>(a);
  }
};
int driver_rc(int rc, const char* who) {
  if (rc == 0) return SSP_OK;
  static thread_local char buf[160];
  snprintf(buf, sizeof(buf), rc == -2 ? "%s: work buffer too small (see the matching *_work_bytes function)" : "%s: bad size or resample filter", who);
  return fail_msg(SSP_ERR_ARG, buf);
}
}  // namespace

// ssp_aug_rgb2hsv_u8 (mode 1) and ssp_aug_hsv2rgb_u8 (mode 2)
static int aug_convert_u8(const uint8_t* src, uint8_t* dst, long long n_px, int mode, cudaStream_t s) {
  if (!src || !dst || n_px < 0 || (mode != 1 && mode != 2)) return fail_msg(SSP_ERR_ARG, "ssp_aug_rgb2hsv_u8/hsv2rgb_u8: bad argument");
  if (n_px == 0) return SSP_OK;
  aug_distort_kernel<<<blocks_for(n_px, 256), 256, 0, s>>>(src, n_px, mode, dst);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

// ssp_augm_plan_begin / _attempt / _finish (phase MULTI_BEGIN / MULTI_ATTEMPT / MULTI_FINISH)
static int augm_plan(int phase, const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes,
                     int* stage_dims) {
  static_assert(sizeof(ssp_augm_item) == sizeof(AugMultiItem), "ssp_augm_item (include/ssp_b200.h) must mirror AugMultiItem (augment_core.h)");
  static const char* who[3] = {"ssp_augm_plan_begin", "ssp_augm_plan_attempt", "ssp_augm_plan_finish"};
  if (!items || !table_host || !stage_dims || n <= 0 || table_bytes < ssp_augm_table_bytes(n)) return fail_msg(SSP_ERR_ARG, "ssp_augm_plan_*: bad argument");
  for (int i = 0; i < n; i++) {
    const ssp_augm_item& it = items[i];
    const bool common = it.img && it.luts && it.work && it.main_img && it.main_mask && it.total_img && it.total_mask && (uintptr_t)it.work % 16 == 0;
    const bool phase_ok = phase == MULTI_BEGIN ? it.mask != nullptr
                        : phase == MULTI_ATTEMPT ? it.mask && it.counts
                        : (it.out_u8 || it.out_chw);
    if (!common || !phase_ok || it.src_w <= 0 || it.src_h <= 0)
      return fail_msg(SSP_ERR_ARG, "ssp_augm_plan_*: null pointer, misaligned work buffer or empty source in an item");
  }
  const int rc = multi_batch_plan(phase, reinterpret_cast<const AugMultiItem*>(items), n, out_w, out_h, resample, (AugOp*)table_host, stage_dims);
  if (rc) return driver_rc(rc, who[phase]);
  return SSP_OK;
}
}  // namespace ssp

using namespace ssp;

extern "C" {
long long ssp_aug_resize_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) {
  if (in_w <= 0 || in_h <= 0 || out_w <= 0 || out_h <= 0) return SSP_ERR_ARG;
  return resize_work_bytes(in_w, in_h, out_w, out_h, resample);
}
long long ssp_aug_sample_work_bytes(int ow, int oh, int bw, int bh, int cw, int ch, int out_w, int out_h, int resample) {
  if (ow <= 0 || oh <= 0 || bw <= 0 || bh <= 0 || cw <= 0 || ch <= 0 || out_w <= 0 || out_h <= 0) return SSP_ERR_ARG;
  return augment_work_bytes(ow, oh, bw, bh, cw, ch, out_w, out_h, resample);
}

int ssp_aug_resize_u8(const void* src, int src_w, int src_h, int x0, int y0, int in_w, int in_h, void* dst, int out_w, int out_h, int resample,
                      void* work, long long work_bytes, void* stream) {
  if (!src || !dst || !work || src_w <= 0 || src_h <= 0) return fail_msg(SSP_ERR_ARG, "ssp_aug_resize_u8: null pointer or empty source");
  if ((uintptr_t)work % 16) return fail_msg(SSP_ERR_ARG, "ssp_aug_resize_u8: work buffer must be 16-B aligned");
  CudaBackend be{(cudaStream_t)stream};
  const int rc = resize_u8_driver(be, (const uint8_t*)src, src_w, src_h, x0, y0, in_w, in_h, (uint8_t*)dst, out_w, out_h, resample, (uint8_t*)work,
                                  work_bytes);
  if (rc) return driver_rc(rc, "ssp_aug_resize_u8");
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

int ssp_aug_rgb2hsv_u8(const void* rgb, void* hsv, long long n_pixels, void* stream) {
  return aug_convert_u8((const uint8_t*)rgb, (uint8_t*)hsv, n_pixels, 1, (cudaStream_t)stream);
}
int ssp_aug_hsv2rgb_u8(const void* hsv, void* rgb, long long n_pixels, void* stream) {
  return aug_convert_u8((const uint8_t*)hsv, (uint8_t*)rgb, n_pixels, 2, (cudaStream_t)stream);
}

int ssp_aug_to_tensor_u8(const void* src, long long n_px, float* out_chw, void* stream) {
  if (!src || !out_chw || n_px < 0) return fail_msg(SSP_ERR_ARG, "ssp_aug_to_tensor_u8: bad argument");
  if (n_px == 0) return SSP_OK;
  aug_to_tensor_kernel<<<blocks_for(n_px, 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)src, n_px, out_chw);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

long long ssp_aug_batch_table_bytes(int n) { return n > 0 ? (long long)kMaxStages * n * (long long)sizeof(AugOp) : SSP_ERR_ARG; }

// host side of the batched path: items (device pointers, host array) -> op table (host memory, to be copied to the device with the
// batch) + per-stage launch extents
int ssp_aug_batch_plan(const ssp_aug_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* stage_dims) {
  static_assert(sizeof(ssp_aug_item) == sizeof(AugItem), "ssp_aug_item (include/ssp_b200.h) must mirror AugItem (augment_core.h)");
  if (!items || !table_host || !stage_dims || n <= 0 || table_bytes < ssp_aug_batch_table_bytes(n)) return fail_msg(SSP_ERR_ARG, "ssp_aug_batch_plan: bad argument");
  for (int i = 0; i < n; i++)
    if (!items[i].img || !items[i].mask || !items[i].bg || !items[i].luts || !items[i].work || (!items[i].out_u8 && !items[i].out_chw) ||
        ((uintptr_t)items[i].work % 16))
      return fail_msg(SSP_ERR_ARG, "ssp_aug_batch_plan: null pointer or misaligned work buffer in an item");
  const int rc = augment_batch_plan(reinterpret_cast<const AugItem*>(items), n, out_w, out_h, resample, (AugOp*)table_host, stage_dims);
  if (rc) return driver_rc(rc, "ssp_aug_batch_plan");
  return SSP_OK;
}

int ssp_aug_batch_run(const void* table_dev, int n, const int* stage_dims, void* stream) {
  if (!table_dev || !stage_dims || n <= 0 || n > 65535) return fail_msg(SSP_ERR_ARG, "ssp_aug_batch_run: bad argument");
  const AugOp* ops = (const AugOp*)table_dev;
  for (int st = 0; st < kMaxStages; st++) {
    const int nx = stage_dims[2 * st], ny = stage_dims[2 * st + 1];
    if (nx <= 0 || ny <= 0) continue;
    dim3 grid((nx + 31) / 32, (ny + 7) / 8, n);
    aug_stage_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ops + (long long)st * n);
  }
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}

// ---- multi-object pipeline: three planned phases over the same stage kernel
long long ssp_augm_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) {
  if (in_w <= 0 || in_h <= 0 || out_w <= 0 || out_h <= 0) return SSP_ERR_ARG;
  return multi_work_bytes(in_w, in_h, out_w, out_h, resample);
}
long long ssp_augm_table_bytes(int n) { return n > 0 ? (long long)kMaxMultiStages * n * (long long)sizeof(AugOp) : SSP_ERR_ARG; }

int ssp_augm_plan_begin(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(MULTI_BEGIN, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}
int ssp_augm_plan_attempt(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(MULTI_ATTEMPT, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}
int ssp_augm_plan_finish(const ssp_augm_item* items, int n, int out_w, int out_h, int resample, void* table_host, long long table_bytes, int* dims) {
  return augm_plan(MULTI_FINISH, items, n, out_w, out_h, resample, table_host, table_bytes, dims);
}

int ssp_augm_run(const void* table_dev, int n, const int* stage_dims, void* stream) {
  if (!table_dev || !stage_dims || n <= 0 || n > 65535) return fail_msg(SSP_ERR_ARG, "ssp_augm_run: bad argument");
  const AugOp* ops = (const AugOp*)table_dev;
  for (int st = 0; st < kMaxMultiStages; st++) {
    const int nx = stage_dims[2 * st], ny = stage_dims[2 * st + 1];
    if (nx <= 0 || ny <= 0) continue;
    dim3 grid((nx + 31) / 32, (ny + 7) / 8, n);
    aug_stage_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ops + (long long)st * n);
  }
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
