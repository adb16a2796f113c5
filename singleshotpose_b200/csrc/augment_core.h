// Per-pixel arithmetic of the training-image pipeline (reference image.py:14-32, 46-75, 110-127), i.e. of the Pillow routines
// those functions call: ImagingResample (coefficient set-up + 8bpc fixed-point passes), rgb2hsv_row / hsv2rgb, point tables.
// Everything here is SSP_HD so that the SAME source is compiled (a) by nvcc into the kernels of augment.cu (with -fmad=false:
// no multiply-add contraction, every operation rounds like the C original) and (b) by g++ into the host harness of
// tests/helpers/augment_host.cpp, which the CPU test-suite checks bit-exactly against Pillow (HSV over all 2^24 colours).
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define SSP_HD __host__ __device__ __forceinline__
#else
#define SSP_HD inline
#endif

namespace ssp_aug {

enum { RESAMPLE_NEAREST = 0, RESAMPLE_BILINEAR = 2, RESAMPLE_BICUBIC = 3 };   // PIL.Image.Resampling values
enum { PRECISION_BITS = 32 - 8 - 2 };

SSP_HD double filter_eval(int resample, double x) {
  if (x < 0.0) x = -x;
  if (resample == RESAMPLE_BICUBIC) {
    const double a = -0.5;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
  }
  if (x < 1.0) return 1.0 - x;       // bilinear
  return 0.0;
}
SSP_HD double filter_support(int resample) { return resample == RESAMPLE_BICUBIC ? 2.0 : 1.0; }

// maximum number of coefficients per output sample (Resample.c precompute_coeffs)
SSP_HD int coeff_ksize(int in0, int in1, int out_size, int resample) {
  double filterscale = (double)(in1 - in0) / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = filter_support(resample) * filterscale;
  return (int)ceil(support) * 2 + 1;
}

// coefficients of output sample xx: bounds[0] = first input sample, bounds[1] = count, kk[0..ksize) fixed-point weights
SSP_HD void coeff_row(int in_size, int in0, int in1, int out_size, int resample, int ksize, int xx, int* bounds, int* kk) {
  const double scale = (double)(in1 - in0) / out_size;
  double filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = filter_support(resample) * filterscale;
  const double center = in0 + (xx + 0.5) * scale;
  const double ss = 1.0 / filterscale;
  int xmin = (int)(center - support + 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)(center + support + 0.5);
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; x++) ww += filter_eval(resample, (x + xmin - center + 0.5) * ss);
  for (int x = 0; x < ksize; x++) {
    int q = 0;
    if (x < xmax) {
      double w = filter_eval(resample, (x + xmin - center + 0.5) * ss);
      if (ww != 0.0) w /= ww;
      q = w < 0 ? (int)(-0.5 + w * (1 << PRECISION_BITS)) : (int)(0.5 + w * (1 << PRECISION_BITS));   // normalize_coeffs_8bpc
    }
    kk[x] = q;
  }
  bounds[0] = xmin; bounds[1] = xmax;
}

SSP_HD uint8_t clip8_fixed(int acc) {          // Resample.c clip8(): table lookup of acc >> PRECISION_BITS, saturating
  const int v = acc >> PRECISION_BITS;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}
SSP_HD uint8_t clip8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// Geometry.c ImagingScaleAffine with the nearest filter: source index of output sample x (the C code accumulates xo += a)
SSP_HD int nearest_index(int in_size, int out_size, int x) {
  const double a = (double)in_size / out_size;
  double xo = a * 0.5;
  for (int i = 0; i < x; i++) xo += a;
  int xin = xo >= 0 ? (int)floor(xo) : -1;
  return xin < 0 ? 0 : (xin >= in_size ? in_size - 1 : xin);
}

// Convert.c rgb2hsv_row
SSP_HD void rgb2hsv_px(uint8_t r, uint8_t g, uint8_t b, uint8_t* out) {
  const uint8_t maxc = r > g ? (r > b ? r : b) : (g > b ? g : b);
  const uint8_t minc = r < g ? (r < b ? r : b) : (g < b ? g : b);
  out[2] = maxc;
  if (minc == maxc) { out[0] = 0; out[1] = 0; return; }
  const float cr = (float)(maxc - minc);
  const float s = cr / (float)maxc;
  const float rc = ((float)(maxc - r)) / cr;
  const float gc = ((float)(maxc - g)) / cr;
  const float bc = ((float)(maxc - b)) / cr;
  float h;
  if (r == maxc) h = bc - gc;
  else if (g == maxc) h = (float)(2.0 + (double)rc - (double)bc);
  else h = (float)(4.0 + (double)gc - (double)rc);
  h = (float)fmod(((double)h / 6.0 + 1.0), 1.0);
  out[0] = clip8((int)((double)h * 255.0));
  out[1] = clip8((int)((double)s * 255.0));
}

SSP_HD int round_half_away(double x) { return (int)(x >= 0.0 ? floor(x + 0.5) : -floor(-x + 0.5)); }

// Convert.c hsv2rgb
SSP_HD void hsv2rgb_px(uint8_t h, uint8_t s, uint8_t v, uint8_t* out) {
  if (s == 0) { out[0] = v; out[1] = v; out[2] = v; return; }
  const double hf = (double)(float)h * 6.0 / 255.0;
  const int i = (int)floor(hf);
  const float f = (float)(hf - (double)(float)i);
  const float fs = (float)((double)(float)s / 255.0);
  const double vd = (double)(float)v;
  const uint8_t p = clip8(round_half_away(vd * (1.0 - (double)fs)));
  const uint8_t q = clip8(round_half_away(vd * (1.0 - (double)(fs * f))));
  const uint8_t t = clip8(round_half_away(vd * (1.0 - (double)fs * (1.0 - (double)f))));     // fs * (1.0 - f): double in C
  switch (i % 6) {
    case 0: out[0] = v; out[1] = t; out[2] = p; break;
    case 1: out[0] = q; out[1] = v; out[2] = p; break;
    case 2: out[0] = p; out[1] = v; out[2] = t; break;
    case 3: out[0] = p; out[1] = q; out[2] = v; break;
    case 4: out[0] = t; out[1] = p; out[2] = v; break;
    default: out[0] = v; out[1] = p; out[2] = q; break;
  }
}

// distort_image (image.py:14-32): RGB -> HSV, three point() tables (hue, sat, val), HSV -> RGB
SSP_HD void distort_px(const uint8_t* rgb, const uint8_t* lut_h, const uint8_t* lut_s, const uint8_t* lut_v, uint8_t* out) {
  uint8_t hsv[3];
  rgb2hsv_px(rgb[0], rgb[1], rgb[2], hsv);
  hsv2rgb_px(lut_h[hsv[0]], lut_s[hsv[1]], lut_v[hsv[2]], out);
}

// change_background (image.py:110-127): a*c + b*d in int32, then .convert('L') saturates
SSP_HD uint8_t composite_px(uint8_t img, uint8_t bg, uint8_t mask, const uint8_t* lut_pos, const uint8_t* lut_neg) {
  return clip8((int)img * (int)lut_pos[mask] + (int)bg * (int)lut_neg[mask]);
}


// ------------------------------------------------------------------------------------------------------------------------
// One separable pass / one nearest gather, per OUTPUT pixel.  The logical input of a pass is the window
// [x0, x0+in_w) x [y0, y0+in_h) of the physical image src (src_w x src_h); samples outside the physical image read as zero
// (this is Image.crop() with a box that sticks out of the image, fused into the read).
struct PassArgs {
  const uint8_t* src; int src_w, src_h, x0, y0, in_w, in_h;
  uint8_t* dst; int dst_w, dst_h;
  int axis;                       // 1: horizontal (dst_w = out_w, dst_h = in_h); 0: vertical (dst_w = in_w, dst_h = out_h)
  const int* bounds; const int* kk; int ksize;
};
SSP_HD int fetch3(const PassArgs& a, int lx, int ly, int* px) {
  const int x = a.x0 + lx, y = a.y0 + ly;
  if (x < 0 || y < 0 || x >= a.src_w || y >= a.src_h) { px[0] = px[1] = px[2] = 0; return 0; }
  const uint8_t* s = a.src + ((long long)y * a.src_w + x) * 3;
  px[0] = s[0]; px[1] = s[1]; px[2] = s[2];
  return 1;
}
SSP_HD void resample_pass_px(const PassArgs& a, int ox, int oy) {
  const int o = a.axis ? ox : oy;
  const int lo = a.bounds[2 * o], n = a.bounds[2 * o + 1];
  const int* k = a.kk + (long long)o * a.ksize;
  int acc0 = 1 << (PRECISION_BITS - 1), acc1 = acc0, acc2 = acc0;
  for (int i = 0; i < n; i++) {
    int px[3];
    if (a.axis) fetch3(a, lo + i, oy, px); else fetch3(a, ox, lo + i, px);
    acc0 += px[0] * k[i]; acc1 += px[1] * k[i]; acc2 += px[2] * k[i];
  }
  uint8_t* d = a.dst + ((long long)oy * a.dst_w + ox) * 3;
  d[0] = clip8_fixed(acc0); d[1] = clip8_fixed(acc1); d[2] = clip8_fixed(acc2);
}
SSP_HD void nearest_px(const PassArgs& a, int ox, int oy) {      // dst_w x dst_h = output size; also the plain window copy
  int px[3];
  fetch3(a, nearest_index(a.in_w, a.dst_w, ox), nearest_index(a.in_h, a.dst_h, oy), px);
  uint8_t* d = a.dst + ((long long)oy * a.dst_w + ox) * 3;
  d[0] = (uint8_t)px[0]; d[1] = (uint8_t)px[1]; d[2] = (uint8_t)px[2];
}

// ------------------------------------------------------------------------------------------------------------------------
// Drivers, shared by the CUDA back end (augment.cu: every method is a kernel launch) and the host harness (plain loops).
// Backend methods: coeffs(in_size, in0, in1, out_size, resample, ksize, bounds, kk), pass(PassArgs), nearest(PassArgs),
//                  composite(img, bg, mask, lut_pos, lut_neg, n_bytes, out), distort(src, w, h, luts3, out_u8, out_chw)
static inline long long align16(long long v) { return (v + 15) & ~15LL; }

static inline long long resize_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) {
  if (resample == RESAMPLE_NEAREST || (in_w == out_w && in_h == out_h)) return 16;
  const int ks_h = coeff_ksize(0, in_w, out_w, resample), ks_v = coeff_ksize(0, in_h, out_h, resample);
  long long b = align16(8LL * out_w) + align16(4LL * out_w * ks_h) + align16(8LL * out_h) + align16(4LL * out_h * ks_v);
  const long long t1 = 3LL * out_w * in_h, t2 = 3LL * in_w * out_h;
  return b + align16(t1 > t2 ? t1 : t2);
}

// Image.resize(size, resample) of the window (x0, y0, in_w, in_h) of src -> dst (out_w x out_h, dense HWC)
template <class Backend>
int resize_u8_driver(Backend& be, const uint8_t* src, int src_w, int src_h, int x0, int y0, int in_w, int in_h, uint8_t* dst,
                     int out_w, int out_h, int resample, uint8_t* work, long long work_bytes) {
  if (in_w <= 0 || in_h <= 0 || out_w <= 0 || out_h <= 0) return -1;
  if (resample != RESAMPLE_NEAREST && resample != RESAMPLE_BILINEAR && resample != RESAMPLE_BICUBIC) return -1;
  if (work_bytes < resize_work_bytes(in_w, in_h, out_w, out_h, resample)) return -2;
  PassArgs a{src, src_w, src_h, x0, y0, in_w, in_h, dst, out_w, out_h, 1, nullptr, nullptr, 0};
  if (resample == RESAMPLE_NEAREST || (in_w == out_w && in_h == out_h)) {   // same size: Image.resize returns a copy
    be.nearest(a);
    return 0;
  }
  const int ks_h = coeff_ksize(0, in_w, out_w, resample), ks_v = coeff_ksize(0, in_h, out_h, resample);
  uint8_t* w = work;
  int* bounds_h = (int*)w; w += align16(8LL * out_w);
  int* kk_h = (int*)w;     w += align16(4LL * out_w * ks_h);
  int* bounds_v = (int*)w; w += align16(8LL * out_h);
  int* kk_v = (int*)w;     w += align16(4LL * out_h * ks_v);
  uint8_t* temp = w;
  const bool need_h = out_w != in_w, need_v = out_h != in_h;
  if (need_h) be.coeffs(in_w, 0, in_w, out_w, resample, ks_h, bounds_h, kk_h);
  if (need_v) be.coeffs(in_h, 0, in_h, out_h, resample, ks_v, bounds_v, kk_v);
  const bool vfirst = in_h > in_w * 100 && out_h < in_h;        // Image.py resize(): very tall images shrink vertically first
  PassArgs ph = a, pv = a;
  ph.axis = 1; ph.bounds = bounds_h; ph.kk = kk_h; ph.ksize = ks_h;
  pv.axis = 0; pv.bounds = bounds_v; pv.kk = kk_v; pv.ksize = ks_v;
  if (need_h && need_v) {
    PassArgs& first = vfirst ? pv : ph;
    PassArgs& second = vfirst ? ph : pv;
    first.dst = temp;
    first.dst_w = vfirst ? in_w : out_w; first.dst_h = vfirst ? out_h : in_h;
    be.pass(first);
    second.src = temp; second.src_w = first.dst_w; second.src_h = first.dst_h; second.x0 = 0; second.y0 = 0;
    second.in_w = first.dst_w; second.in_h = first.dst_h;
    second.dst = dst; second.dst_w = out_w; second.dst_h = out_h;
    be.pass(second);
  } else if (need_h) {
    ph.dst_w = out_w; ph.dst_h = in_h; be.pass(ph);
  } else {
    pv.dst_w = in_w; pv.dst_h = out_h; be.pass(pv);
  }
  return 0;
}

static inline long long augment_work_bytes(int ow, int oh, int bw, int bh, int cw, int ch, int out_w, int out_h, int resample) {
  const long long r1 = resize_work_bytes(bw, bh, ow, oh, resample), r2 = resize_work_bytes(cw, ch, out_w, out_h, resample);
  return align16(3LL * ow * oh) * 2 + align16(3LL * out_w * out_h) + align16(r1 > r2 ? r1 : r2);
}

// change_background + data_augmentation (+ ToTensor) of ONE sample, image.py:110-127 / 46-75 / dataset.py transform.
// luts: 5 x 256 bytes = posmask, negmask, hue, saturation, value tables.  Crop window = (pleft, ptop, cw, ch), image.py:64.
template <class Backend>
int augment_sample_driver(Backend& be, const uint8_t* img, const uint8_t* mask, int ow, int oh, const uint8_t* bg, int bw, int bh,
                          const uint8_t* luts, int pleft, int ptop, int cw, int ch, int out_w, int out_h, int resample,
                          uint8_t* work, long long work_bytes, uint8_t* out_u8, float* out_chw) {
  if (ow <= 0 || oh <= 0 || bw <= 0 || bh <= 0 || cw <= 0 || ch <= 0 || out_w <= 0 || out_h <= 0) return -1;
  if (work_bytes < augment_work_bytes(ow, oh, bw, bh, cw, ch, out_w, out_h, resample)) return -2;
  uint8_t* w = work;
  uint8_t* bg_r = w;  w += align16(3LL * ow * oh);
  uint8_t* comp = w;  w += align16(3LL * ow * oh);
  uint8_t* sized = w; w += align16(3LL * out_w * out_h);
  const long long rest = work_bytes - (w - work);
  int rc = resize_u8_driver(be, bg, bw, bh, 0, 0, bw, bh, bg_r, ow, oh, resample, w, rest);
  if (rc) return rc;
  be.composite(img, bg_r, mask, luts, luts + 256, 3LL * ow * oh, comp);
  rc = resize_u8_driver(be, comp, ow, oh, pleft, ptop, cw, ch, sized, out_w, out_h, resample, w, rest);
  if (rc) return rc;
  be.distort(sized, out_w, out_h, luts + 512, out_u8, out_chw);
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------------
// Batched execution (one launch per STAGE per batch instead of ~10 launches per sample).  A recording back end runs the very
// same drivers as above for every sample and files the k-th call of a sample under stage k of an op table [stage][sample];
// stages are then executed in order (the only dependencies are between consecutive calls of ONE sample), every op by
// op_element() per element of its (nx, ny) extent -- on the GPU one thread per element with blockIdx.z = sample
// (augment.cu), in the host harness plain loops.  The table holds device pointers and is copied with the batch's bytes.
enum { OP_NONE = 0, OP_COEFFS = 1, OP_PASS = 2, OP_NEAREST = 3, OP_COMPOSITE = 4, OP_DISTORT = 5,
       // multi-object pipeline (image_multi.py), see the drivers further down
       OP_MASKBG = 6, OP_PLACE_MAIN = 7, OP_ZERO_COUNTS = 8, OP_COUNT = 9, OP_SUPERIMPOSE = 10, OP_FINISH = 11 };
static constexpr int kMaxStages = 10;       // 2 x (2 coefficient tables + 2 passes) + composite + distort
struct AugOp {
  int kind, nx, ny, pad_;
  PassArgs pass;                                                          // OP_PASS / OP_NEAREST
  int in_size, in0, in1, out_size, resample, ksize; int* bounds; int* kk;  // OP_COEFFS
  const uint8_t* img; const uint8_t* bg; const uint8_t* mask; const uint8_t* lut_pos; const uint8_t* lut_neg; uint8_t* comp_out;   // OP_COMPOSITE (nx = bytes per row)
  const uint8_t* src; const uint8_t* luts; uint8_t* out_u8; float* out_chw;   // OP_DISTORT (nx x ny pixels)
  // multi-object ops: network-size object (img, mask above: unshifted, unflipped), per-sample totals and counters
  uint8_t* main_img; uint8_t* main_mask; uint8_t* total_img; uint8_t* total_mask; unsigned* counts;
  int flip, shift_x, shift_y, pad2_;
};

SSP_HD int wrap_index(int v, int n) { const int r = v % n; return r < 0 ? r + n : r; }

// shifted_data_augmentation_with_mask's ImageChops.offset(dx, dy) then FLIP_LEFT_RIGHT, followed by mask_background
// (image_multi.py:218-223, 38-50), as one index mapping from the network-size resize outputs; initialises the totals
// (:321-322).  out[y][x] = sized[(y - dy) mod H][(x' - dx) mod W] with x' = W-1-x when flipped.
SSP_HD void place_main_px(const AugOp& op, int x, int y) {
  const int W = op.nx, H = op.ny;
  const long long s = ((long long)wrap_index(y - op.shift_y, H) * W + wrap_index((op.flip ? W - 1 - x : x) - op.shift_x, W)) * 3;
  const long long d = ((long long)y * W + x) * 3;
  for (int c = 0; c < 3; c++) {
    const uint8_t m = op.mask[s + c];
    const uint8_t a = clip8((int)op.img[s + c] * (int)op.lut_pos[m]);
    op.main_img[d + c] = a; op.total_img[d + c] = a;
    op.main_mask[d + c] = m; op.total_mask[d + c] = m;
  }
}
// the overlap test of augment_objects (image_multi.py:344-352) for one pixel of the (flipped) candidate mask:
// s = bytes > 200 of the candidate, i = those that are also > 200 in the total mask
SSP_HD void count_px(const AugOp& op, int x, int y, unsigned* s, unsigned* i) {
  const long long src = ((long long)y * op.nx + (op.flip ? op.nx - 1 - x : x)) * 3, d = ((long long)y * op.nx + x) * 3;
  for (int c = 0; c < 3; c++) {
    const unsigned xx = op.mask[src + c] > 200;
    *s += xx; *i += xx & (unsigned)(op.total_mask[d + c] > 200);
  }
}
// accept iff float(I) / float(S) < 0.2 with S != 0 (image_multi.py:349-353): a double division, as in Python
SSP_HD bool accept_counts(const unsigned* counts) { return counts[0] != 0 && (double)counts[1] / (double)counts[0] < 0.2; }
// superimpose_masks + superimpose_masked_imgs (image_multi.py:355-356, 265-297) of one pixel, predicated on the accept decision
SSP_HD void superimpose_px(const AugOp& op, int x, int y) {
  const bool acc = accept_counts(op.counts);
  if (x == 0 && y == 0) op.counts[2] = acc;
  if (!acc) return;
  const long long src = ((long long)y * op.nx + (op.flip ? op.nx - 1 - x : x)) * 3, d = ((long long)y * op.nx + x) * 3;
  for (int c = 0; c < 3; c++) {
    const uint8_t m = op.mask[src + c];
    op.total_mask[d + c] = clip8((int)m + (int)op.total_mask[d + c] * (int)op.lut_neg[m]);
    op.total_img[d + c] = composite_px(op.img[src + c], op.total_img[d + c], m, op.lut_pos, op.lut_neg);
  }
}
// main object on top (image_multi.py:363), change_background with the network-size background (:380), ToTensor
SSP_HD void finish_px(const AugOp& op, int x, int y) {
  const long long n = (long long)op.nx * op.ny, i = (long long)y * op.nx + x;
  for (int c = 0; c < 3; c++) {
    const long long k = 3 * i + c;
    const uint8_t t = composite_px(op.main_img[k], op.total_img[k], op.main_mask[k], op.lut_pos, op.lut_neg);
    const uint8_t v = composite_px(t, op.bg[k], op.total_mask[k], op.lut_pos, op.lut_neg);
    if (op.out_u8) op.out_u8[k] = v;
    if (op.out_chw) op.out_chw[c * n + i] = (float)v / 255.0f;
  }
}

SSP_HD void op_element(const AugOp& op, int x, int y) {
  if (x >= op.nx || y >= op.ny) return;
  switch (op.kind) {
    case OP_COEFFS: coeff_row(op.in_size, op.in0, op.in1, op.out_size, op.resample, op.ksize, x, op.bounds + 2 * x, op.kk + (long long)x * op.ksize); break;
    case OP_PASS: resample_pass_px(op.pass, x, y); break;
    case OP_NEAREST: nearest_px(op.pass, x, y); break;
    case OP_COMPOSITE: { const long long i = (long long)y * op.nx + x; op.comp_out[i] = composite_px(op.img[i], op.bg[i], op.mask[i], op.lut_pos, op.lut_neg); } break;
    case OP_DISTORT: {
      const long long n = (long long)op.nx * op.ny, i = (long long)y * op.nx + x;
      uint8_t o[3];
      distort_px(op.src + 3 * i, op.luts, op.luts + 256, op.luts + 512, o);
      if (op.out_u8) { op.out_u8[3 * i] = o[0]; op.out_u8[3 * i + 1] = o[1]; op.out_u8[3 * i + 2] = o[2]; }
      if (op.out_chw) { op.out_chw[i] = (float)o[0] / 255.0f; op.out_chw[n + i] = (float)o[1] / 255.0f; op.out_chw[2 * n + i] = (float)o[2] / 255.0f; }
    } break;
    case OP_MASKBG: { const long long i = (long long)y * op.nx + x; op.comp_out[i] = clip8((int)op.img[i] * (int)op.lut_pos[op.mask[i]]); } break;
    case OP_PLACE_MAIN: place_main_px(op, x, y); break;
    case OP_ZERO_COUNTS: op.counts[0] = op.counts[1] = op.counts[2] = 0; break;
    case OP_COUNT: break;             // a per-sample reduction: done by the executor (aug_stage_kernel, host harness) with count_px
    case OP_SUPERIMPOSE: superimpose_px(op, x, y); break;
    case OP_FINISH: finish_px(op, x, y); break;
    default: break;
  }
}
// records the calls of ONE sample into column `sample` of the table
struct PlanBackend {
  AugOp* table; int n_samples, sample, call; bool overflow;
  AugOp* next() {
    if (call >= max_stages) { overflow = true; return nullptr; }
    AugOp* o = table + (long long)call * n_samples + sample;
    call++;
    return o;
  }
  void coeffs(int in_size, int in0, int in1, int out_size, int resample, int ksize, int* bounds, int* kk) {
    if (AugOp* o = next()) { o->kind = OP_COEFFS; o->nx = out_size; o->ny = 1; o->in_size = in_size; o->in0 = in0; o->in1 = in1; o->out_size = out_size;
                             o->resample = resample; o->ksize = ksize; o->bounds = bounds; o->kk = kk; }
  }
  void pass(const PassArgs& a) { if (AugOp* o = next()) { o->kind = OP_PASS; o->nx = a.dst_w; o->ny = a.dst_h; o->pass = a; } }
  void nearest(const PassArgs& a) { if (AugOp* o = next()) { o->kind = OP_NEAREST; o->nx = a.dst_w; o->ny = a.dst_h; o->pass = a; } }
  void composite(const uint8_t* img, const uint8_t* bg, const uint8_t* mask, const uint8_t* lp, const uint8_t* ln, long long n, uint8_t* out) {
    if (AugOp* o = next()) { o->kind = OP_COMPOSITE; o->nx = row_bytes; o->ny = (int)(n / row_bytes); o->img = img; o->bg = bg; o->mask = mask;
                             o->lut_pos = lp; o->lut_neg = ln; o->comp_out = out; }
  }
  void distort(const uint8_t* src, int w, int h, const uint8_t* luts, uint8_t* out_u8, float* out_chw) {
    if (AugOp* o = next()) { o->kind = OP_DISTORT; o->nx = w; o->ny = h; o->src = src; o->luts = luts; o->out_u8 = out_u8; o->out_chw = out_chw; }
  }
  int row_bytes;      // 3 * ow of the sample being planned (composite is a flat byte op; rows give it a 2-D extent)
  int max_stages = kMaxStages;
  // multi-object ops: one op per network-size image (nx x ny pixels) unless stated
  AugOp* multi(int kind, int w, int h) {
    AugOp* o = next();
    if (o) { o->kind = kind; o->nx = w; o->ny = h; }
    return o;
  }
  void mask_bg(uint8_t* img, const uint8_t* mask, int w, int h, const uint8_t* lp) {      // in place, flat bytes
    if (AugOp* o = multi(OP_MASKBG, 3 * w, h)) { o->img = img; o->mask = mask; o->comp_out = img; o->lut_pos = lp; }
  }
};
struct AugItem {      // one sample of a batch: the arguments of augment_sample_driver (device pointers)
  const uint8_t* img; const uint8_t* mask; int ow, oh; const uint8_t* bg; int bw, bh; const uint8_t* luts; int pleft, ptop, cw, ch;
  uint8_t* work; long long work_bytes; uint8_t* out_u8; float* out_chw;
};
// fills table[kMaxStages][n] (zeroed here) and stage_dims[kMaxStages][2] = largest (nx, ny) of every stage; 0 ok, < 0 error
static inline int augment_batch_plan(const AugItem* items, int n, int out_w, int out_h, int resample, AugOp* table, int* stage_dims) {
  for (long long i = 0; i < (long long)kMaxStages * n; i++) { AugOp z = AugOp(); table[i] = z; }
  for (int s = 0; s < 2 * kMaxStages; s++) stage_dims[s] = 0;
  for (int i = 0; i < n; i++) {
    const AugItem& it = items[i];
    PlanBackend be{table, n, i, 0, false, 3 * it.ow};
    const int rc = augment_sample_driver(be, it.img, it.mask, it.ow, it.oh, it.bg, it.bw, it.bh, it.luts, it.pleft, it.ptop, it.cw, it.ch, out_w, out_h,
                                         resample, it.work, it.work_bytes, it.out_u8, it.out_chw);
    if (rc) return rc;
    if (be.overflow) return -3;
    for (int s = 0; s < be.call; s++) {
      const AugOp& o = table[(long long)s * n + i];
      if (o.nx > stage_dims[2 * s]) stage_dims[2 * s] = o.nx;
      if (o.ny > stage_dims[2 * s + 1]) stage_dims[2 * s + 1] = o.ny;
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------------
// Multi-object pipeline (multi_obj_pose_estimation/image_multi.py load_data_detection / augment_objects), batched in three
// phases over per-sample network-size state (main object, total image, total mask: W x H x 3 bytes each):
//   begin   - jitter crop + resize of the main object's image and mask (the resize driver above), then offset + flip +
//             mask_background in one index mapping (OP_PLACE_MAIN), which also initialises the totals;
//   attempt - one candidate per sample: mask_background at source resolution (in place, only for a candidate that is not yet
//             masked), zero the counters, crop + resize image and mask, count (> 200 bytes of the flipped candidate and their
//             overlap with the total mask; a per-sample integer reduction), then the accept decision on the device and the
//             predicated superimpose of mask and image (OP_SUPERIMPOSE writes the decision to counts[2]);
//   finish  - resize of the background, main object on top, change_background, ToTensor (OP_FINISH).
// Flip is folded into the index mapping of the op that reads the resized candidate.  All resizing is resize_u8_driver.
static constexpr int kMaxMultiStages = 16;  // attempt: mask_bg + zero + 2 x (2 coefficient tables + 2 passes) + count + superimpose
struct AugMultiItem {   // one sample of one phase (device pointers); fields a phase does not read may be null
  uint8_t* img; const uint8_t* mask; int src_w, src_h;   // begin: main object; attempt: candidate; finish: background (img)
  int pleft, ptop, cw, ch;                                  // crop window (cw = swidth - 1, image_multi.py:203,248)
  int flip, shift_x, shift_y, mask_bg;                      // mask_bg: attempt masks `img` in place first
  uint8_t* main_img; uint8_t* main_mask; uint8_t* total_img; uint8_t* total_mask;
  unsigned* counts;                                         // [S, I, accepted, unused]
  const uint8_t* luts;                                      // posmask | negmask, 2 x 256 bytes
  uint8_t* work; long long work_bytes; uint8_t* out_u8; float* out_chw;
};
static inline long long multi_work_bytes(int in_w, int in_h, int out_w, int out_h, int resample) {
  return 2 * align16(3LL * out_w * out_h) + align16(resize_work_bytes(in_w, in_h, out_w, out_h, resample));
}
enum { MULTI_BEGIN = 0, MULTI_ATTEMPT = 1, MULTI_FINISH = 2 };

static inline int multi_sample_plan(PlanBackend& be, int phase, const AugMultiItem& it, int W, int H, int resample) {
  const uint8_t* lp = it.luts;
  const uint8_t* ln = it.luts + 256;
  uint8_t* sized_img = it.work;
  uint8_t* sized_mask = it.work + align16(3LL * W * H);
  uint8_t* rest = sized_mask + align16(3LL * W * H);
  const long long rest_bytes = it.work_bytes - (rest - it.work);
  if (phase == MULTI_FINISH) {
    if (it.work_bytes < multi_work_bytes(it.src_w, it.src_h, W, H, resample)) return -2;
    int rc = resize_u8_driver(be, it.img, it.src_w, it.src_h, 0, 0, it.src_w, it.src_h, sized_img, W, H, resample, rest, rest_bytes);
    if (rc) return rc;
    if (AugOp* o = be.multi(OP_FINISH, W, H)) {
      o->main_img = it.main_img; o->main_mask = it.main_mask; o->total_img = it.total_img; o->total_mask = it.total_mask;
      o->bg = sized_img; o->lut_pos = lp; o->lut_neg = ln; o->out_u8 = it.out_u8; o->out_chw = it.out_chw;
    }
    return 0;
  }
  if (it.cw <= 0 || it.ch <= 0) return -1;
  if (it.work_bytes < multi_work_bytes(it.cw, it.ch, W, H, resample)) return -2;
  if (phase == MULTI_ATTEMPT) {
    if (it.mask_bg) be.mask_bg(it.img, it.mask, it.src_w, it.src_h, lp);
    if (AugOp* o = be.multi(OP_ZERO_COUNTS, 1, 1)) o->counts = it.counts;
  }
  int rc = resize_u8_driver(be, it.img, it.src_w, it.src_h, it.pleft, it.ptop, it.cw, it.ch, sized_img, W, H, resample, rest, rest_bytes);
  if (rc) return rc;
  rc = resize_u8_driver(be, it.mask, it.src_w, it.src_h, it.pleft, it.ptop, it.cw, it.ch, sized_mask, W, H, resample, rest, rest_bytes);
  if (rc) return rc;
  const int kinds[2] = {phase == MULTI_BEGIN ? OP_PLACE_MAIN : OP_COUNT, phase == MULTI_BEGIN ? OP_NONE : OP_SUPERIMPOSE};
  for (int k = 0; k < 2 && kinds[k] != OP_NONE; k++)
    if (AugOp* o = be.multi(kinds[k], W, H)) {
      o->img = sized_img; o->mask = sized_mask; o->lut_pos = lp; o->lut_neg = ln; o->flip = it.flip; o->shift_x = it.shift_x; o->shift_y = it.shift_y;
      o->main_img = it.main_img; o->main_mask = it.main_mask; o->total_img = it.total_img; o->total_mask = it.total_mask; o->counts = it.counts;
    }
  return 0;
}

// fills table[kMaxMultiStages][n] and stage_dims[kMaxMultiStages][2] for one phase of a batch; 0 ok, < 0 error
static inline int multi_batch_plan(int phase, const AugMultiItem* items, int n, int out_w, int out_h, int resample, AugOp* table, int* stage_dims) {
  if (phase < MULTI_BEGIN || phase > MULTI_FINISH || out_w <= 0 || out_h <= 0) return -1;
  for (long long i = 0; i < (long long)kMaxMultiStages * n; i++) { AugOp z = AugOp(); table[i] = z; }
  for (int s = 0; s < 2 * kMaxMultiStages; s++) stage_dims[s] = 0;
  for (int i = 0; i < n; i++) {
    PlanBackend be{table, n, i, 0, false, 3 * out_w};
    be.max_stages = kMaxMultiStages;
    const int rc = multi_sample_plan(be, phase, items[i], out_w, out_h, resample);
    if (rc) return rc;
    if (be.overflow) return -3;
    for (int s = 0; s < be.call; s++) {
      const AugOp& o = table[(long long)s * n + i];
      if (o.nx > stage_dims[2 * s]) stage_dims[2 * s] = o.nx;
      if (o.ny > stage_dims[2 * s + 1]) stage_dims[2 * s + 1] = o.ny;
    }
  }
  return 0;
}

}  // namespace ssp_aug
