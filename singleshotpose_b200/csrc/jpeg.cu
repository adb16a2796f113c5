// Baseline JPEG decode for a whole batch, byte-identical to Pillow's Image.open(f).convert('RGB') (rules: jpeg_core.h).
//
// Host (ssp_jpeg_batch_plan): parses each file again, copies its entropy-coded segment into the pinned staging buffer without
// the stuffed zero bytes and the restart markers (checking the RST sequence), records where each restart interval starts and
// cuts every interval into subsequences of kSubBits bits.  The per-image records, payloads and interval tables then travel to
// the device in the caller's single host->device copy.
//
// Device, three launches for the whole batch on the caller's stream:
//   entropy_kernel   one CTA per image.  The self-synchronising parallel Huffman decode (Weissenberger & Schmidt, ICPP 2018):
//                    1. every subsequence is decoded from its first bit once per block phase of the MCU (guessed state:
//                       that block, DC next), recording the candidate state at the first codeword boundary at or past its end;
//                    2. each candidate of subsequence t-1 is decoded exactly through subsequence t; the candidate of t it ends
//                       in (if any) is its link;
//                    3. per restart interval, one thread follows the links from the interval's exact start and decodes
//                       serially only where a state has no link (jpeg_core.h walk_interval);
//                    4. exclusive scan of the per-subsequence block counts -> each subsequence's first block;
//                    5. a second decode from the exact states writes the coefficients;
//                    6. per-component prefix sums of the DC differences, reset at every restart interval.
//                    Why the walked states are the true ones: the first subsequence of an interval starts from the exact
//                    state (its first bit, block 0, DC next), and every further state is either the end of an exact decode
//                    from the previous true state or reached through a link, which step 2 established by an exact decode from
//                    that very state.  By induction each state is the sequential decoder's.  Quick synchronisation of the
//                    guesses only saves serial decodes; it is never assumed.
//   idct_kernel      8 threads per 8x8 block: dequantise + ISLOW IDCT into the component planes.
//   color_kernel     one thread per output pixel: fancy upsampling + YCbCr->RGB into the (H, W, 3) uint8 output.
// No allocation, no synchronisation, no atomics on output values (the IDCT range flag is an atomicOr into its own word).  Each
// image's output depends on its own bytes only: identical across launches and batch compositions.
#include <limits.h>
#include <string.h>

#include <vector>

#include "ssp_common.cuh"
#include "../../include/ssp_b200.h"
#include "jpeg_core.h"

namespace ssp {
using namespace ssp_jpeg;

namespace {
constexpr int kSubBits = 1024;      // subsequence length; the CPU tests also run a tiny one through the same rules
constexpr int kEntropyThreads = 256;
constexpr int kIdctBlocksPerCta = 32;

struct ImgRec {
  Desc d;
  long long data_off, ist_off, ipref_off;   // staging offsets: unstuffed bits, interval starts (nint + 1), sub prefix (nint + 1)
  long long nint, nsub;
  long long coef_off, cand_off, link_off, lcnt_off, cnt0_off, s_off, cnt_off, plane_off[kMaxComp];   // workspace offsets
  uint8_t* out;
  int pre_status, pad;
};

long long align16(long long x) { return (x + 15) & ~15LL; }

// Workspace of one image: coefficients, candidates / links / link counts per (subsequence, phase), first-subsequence counts,
// exact states, counts, planes.
long long image_work(const Desc& d, long long nsub_max, ImgRec* r, long long at) {
  const long long start = at;
  auto take = [&](long long bytes) { const long long o = at; at = align16(at + bytes); return o; };
  const long long coef = take(total_blocks(d) * 64 * 2);
  const long long cand = take(nsub_max * d.bpm * 8), link = take(nsub_max * d.bpm * 4), lcnt = take(nsub_max * d.bpm * 8);
  const long long cnt0 = take(nsub_max * 8), st = take(nsub_max * 8), cnt = take(nsub_max * 8);
  long long pl[kMaxComp] = {0, 0, 0};
  for (int c = 0; c < d.ncomp; c++) pl[c] = take((long long)d.comp[c].bw * d.comp[c].bh * 64);
  if (r) {
    r->coef_off = coef; r->cand_off = cand; r->link_off = link; r->lcnt_off = lcnt; r->cnt0_off = cnt0; r->s_off = st; r->cnt_off = cnt;
    for (int c = 0; c < kMaxComp; c++) r->plane_off[c] = pl[c];
  }
  return at - start;
}
long long nsub_bound(const Desc& d) { return n_intervals(d) + (d.seg_len * 8) / kSubBits + 1; }

// -------------------------------------------------------------------------------------------------------------- kernels
struct SubGeom { uint32_t start, end, limit; bool first; };
__device__ SubGeom sub_geom(const uint32_t* ist, const int* ipref, long long nint, long long t) {
  long long lo = 0, hi = nint - 1;                // the interval j with ipref[j] <= t < ipref[j + 1]
  while (lo < hi) {
    const long long mid = (lo + hi + 1) / 2;
    if (ipref[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const long long u = t - ipref[lo];
  SubGeom g;
  g.limit = ist[lo + 1];
  g.start = ist[lo] + (uint32_t)(u * kSubBits);
  g.end = g.start + kSubBits < g.limit ? g.start + kSubBits : g.limit;
  g.first = u == 0;
  return g;
}

// in-place exclusive scan of v[0..n) by one CTA; returns the total
__device__ long long cta_exclusive_scan(long long* v, long long n, long long* sh) {
  const int tid = threadIdx.x;
  const long long chunk = (n + blockDim.x - 1) / blockDim.x, lo = tid * chunk, hi = lo + chunk < n ? lo + chunk : n;
  long long s = 0;
  for (long long i = lo; i < hi; i++) s += v[i];
  sh[tid] = s;
  __syncthreads();
  if (tid == 0) {
    long long c = 0;
    for (int u = 0; u < (int)blockDim.x; u++) { const long long x = sh[u]; sh[u] = c; c += x; }
    sh[blockDim.x] = c;
  }
  __syncthreads();
  s = sh[tid];
  for (long long i = lo; i < hi; i++) { const long long x = v[i]; v[i] = s; s += x; }
  const long long total = sh[blockDim.x];
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kEntropyThreads) entropy_kernel(const uint8_t* __restrict__ stage, uint8_t* __restrict__ work,
                                                                  int* __restrict__ status, int nimg) {
  __shared__ Desc sd;
  __shared__ long long sh[kEntropyThreads + 1];
  __shared__ unsigned char shr[kEntropyThreads];
  const int tid = threadIdx.x, img = blockIdx.x;
  const ImgRec& rec = reinterpret_cast<const ImgRec*>(stage)[img];
  if (tid == 0) status[nimg + img] = 0;          // the IDCT's range flag
  if (rec.pre_status) {
    if (tid == 0) { status[img] = rec.pre_status; status[2 * nimg + img] = 0; }
    return;
  }
  for (int i = tid; i < (int)(sizeof(Desc) / 4); i += blockDim.x)
    reinterpret_cast<int*>(&sd)[i] = reinterpret_cast<const int*>(&rec.d)[i];
  __syncthreads();
  const uint8_t* data = stage + rec.data_off;
  const uint32_t* ist = reinterpret_cast<const uint32_t*>(stage + rec.ist_off);
  const int* ipref = reinterpret_cast<const int*>(stage + rec.ipref_off);
  const long long nsub = rec.nsub, nint = rec.nint;
  const int P = sd.bpm;
  uint64_t* cand = reinterpret_cast<uint64_t*>(work + rec.cand_off);
  int* link = reinterpret_cast<int*>(work + rec.link_off);
  long long* lcnt = reinterpret_cast<long long*>(work + rec.lcnt_off);
  long long* cnt0 = reinterpret_cast<long long*>(work + rec.cnt0_off);
  uint64_t* fin = reinterpret_cast<uint64_t*>(work + rec.s_off);
  long long* cnt = reinterpret_cast<long long*>(work + rec.cnt_off);
  int16_t* coef = reinterpret_cast<int16_t*>(work + rec.coef_off);

  // 1. candidates: every subsequence from its first bit in every block phase (an interval's first subsequence: exact start)
  for (long long i = tid; i < nsub * P; i += blockDim.x) {
    const long long t = i / P;
    const int p = (int)(i % P);
    const SubGeom g = sub_geom(ist, ipref, nint, t);
    if (g.first && p > 0) { cand[i] = kNone; continue; }
    long long nb;
    cand[i] = sub_step(sd, sd.tab, data, g.end, g.limit, pack(State{g.start, p, 0}), &nb, !g.first);
    if (g.first) cnt0[t] = nb;
  }
  __syncthreads();
  // 2. links: the exact decode of subsequence t from each candidate of t-1
  for (long long i = tid; i < nsub * P; i += blockDim.x) {
    const long long t = i / P;
    const SubGeom g = sub_geom(ist, ipref, nint, t);
    link[i] = -1;
    if (g.first || cand[i - P] == kNone) continue;
    const uint64_t e = sub_step(sd, sd.tab, data, g.end, g.limit, cand[i - P], &lcnt[i]);
    for (int q = 0; q < P; q++)
      if (cand[t * P + q] == e) { link[i] = q; break; }
  }
  __syncthreads();
  // 3. the walk, one thread per restart interval
  long long serial = 0;
  for (long long j = tid; j < nint; j += blockDim.x)
    walk_interval(sd, sd.tab, data, ist[j], ist[j + 1], kSubBits, ipref[j], ipref[j + 1], cand, link, lcnt, cnt0, fin, cnt, &serial);
  sh[tid] = serial;
  __syncthreads();
  if (tid == 0) {
    long long tot = 0;
    for (int u = 0; u < (int)blockDim.x; u++) tot += sh[u];
    status[2 * nimg + img] = (int)(tot < INT_MAX ? tot : INT_MAX);
  }
  __syncthreads();
  // 4. block offsets, then per-interval checks: an error state, the block count, a block cut at the end, > 7 padding bits
  const long long total = cta_exclusive_scan(cnt, nsub, sh);
  int bad = 0;
  for (long long j = tid; j < nint; j += blockDim.x) {
    const long long t0 = ipref[j], t1 = ipref[j + 1];
    const long long got = (t1 < nsub ? cnt[t1] : total) - cnt[t0];
    const uint64_t e = fin[t1 - 1];
    if (e == kErrState) { bad |= kStEntropy; continue; }
    const State st = unpack(e);
    if (got != interval_blocks(sd, j) || st.k != 0 || ist[j + 1] - st.pos >= 8) bad |= kStEntropy;
  }
  if (__syncthreads_or(bad)) {
    if (tid == 0) status[img] = kStEntropy;
    return;
  }
  // 5. zero the coefficients, then write them from the exact states
  {
    const long long n16 = total_blocks(sd) * 64 * 2 / 16;
    int4* z = reinterpret_cast<int4*>(coef);
    for (long long i = tid; i < n16; i += blockDim.x) z[i] = make_int4(0, 0, 0, 0);
  }
  __syncthreads();
  for (long long t = tid; t < nsub; t += blockDim.x) {
    const SubGeom g = sub_geom(ist, ipref, nint, t);
    State st = g.first ? State{g.start, 0, 0} : unpack(fin[t - 1]);
    int err = 0;
    decode_run<true>(sd, sd.tab, data, g.end, g.limit, &st, &err, coef, cnt[t]);
  }
  __syncthreads();
  // 6. DC prediction: segmented prefix sums per component, in int64, flagged when they leave int32 (libjpeg raises there)
  int ovf = 0;
  for (int c = 0; c < sd.ncomp; c++) {
    const long long ne = comp_blocks(sd, c);
    const long long chunk = (ne + blockDim.x - 1) / blockDim.x, lo = tid * chunk, hi = lo + chunk < ne ? lo + chunk : ne;
    long long s = 0;
    bool r = false;
    for (long long e = lo; e < hi; e++) {
      bool rs;
      const long long i = block_of(sd, c, e, &rs);
      if (rs) { s = 0; r = true; }
      s += coef[i * 64];
    }
    sh[tid] = s;
    shr[tid] = r;
    __syncthreads();
    if (tid == 0) {
      long long carry = 0;
      for (int u = 0; u < (int)blockDim.x; u++) { const long long x = sh[u]; sh[u] = carry; carry = shr[u] ? x : carry + x; }
    }
    __syncthreads();
    s = sh[tid];
    for (long long e = lo; e < hi; e++) {
      bool rs;
      const long long i = block_of(sd, c, e, &rs);
      if (rs) s = 0;
      s += coef[i * 64];
      if (s > INT_MAX || s < INT_MIN) ovf = 1;
      coef[i * 64] = (int16_t)s;
    }
    __syncthreads();
  }
  ovf = __syncthreads_or(ovf);
  if (tid == 0) status[img] = ovf ? kStOverflow : 0;
}

__global__ void __launch_bounds__(kIdctBlocksPerCta * 8) idct_kernel(const uint8_t* __restrict__ stage, uint8_t* __restrict__ work,
                                                                     const int* __restrict__ status, int* __restrict__ range) {
  __shared__ int ws[kIdctBlocksPerCta][64];
  const int img = blockIdx.y;
  const ImgRec& rec = reinterpret_cast<const ImgRec*>(stage)[img];
  if (status[img]) return;
  const Desc& d = rec.d;
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const long long blk = (long long)blockIdx.x * kIdctBlocksPerCta + lb;
  const bool live = blk < total_blocks(d);
  int flag = 0;
  const int16_t* coef = reinterpret_cast<const int16_t*>(work + rec.coef_off) + blk * 64;
  int c = 0;
  if (live) {
    c = d.blk_comp[blk % d.bpm];
    idct_pass1(coef, d.quant[d.comp[c].tq], lane, ws[lb], &flag);
  }
  __syncthreads();
  if (live) {
    const long long m = blk / d.bpm;
    const int b = (int)(blk % d.bpm);
    const Comp& k = d.comp[c];
    const long long bx = (m % d.mcux) * k.h + d.blk_dx[b], by = (m / d.mcux) * k.v + d.blk_dy[b];
    const long long pitch = (long long)k.bw * 8;
    uint8_t row[8];
    idct_pass2(ws[lb], lane, row, &flag);
    uint8_t* dst = work + rec.plane_off[c] + (by * 8 + lane) * pitch + bx * 8;
    *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(row);
  }
  if (__syncthreads_or(flag) && threadIdx.x == 0) atomicOr(range + img, kStRange);
}

__global__ void __launch_bounds__(256) color_kernel(const uint8_t* __restrict__ stage, const uint8_t* __restrict__ work,
                                                    const int* __restrict__ status, const int* __restrict__ range) {
  const int img = blockIdx.y;
  const ImgRec& rec = reinterpret_cast<const ImgRec*>(stage)[img];
  if (status[img] | range[img]) return;
  const Desc& d = rec.d;
  const long long npix = (long long)d.w * d.h;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / d.w), x = (int)(p % d.w);
    uint8_t* o = rec.out + p * 3;
    const int yv = work[rec.plane_off[0] + (long long)y * d.comp[0].bw * 8 + x];
    if (d.ncomp == 1) {
      o[0] = o[1] = o[2] = (uint8_t)yv;
    } else {
      const int cb = upsample(d, 1, work + rec.plane_off[1], d.comp[1].bw * 8, x, y);
      const int cr = upsample(d, 2, work + rec.plane_off[2], d.comp[2].bw * 8, x, y);
      ycc_to_rgb(yv, cb, cr, o);
    }
  }
}
}  // namespace

// -------------------------------------------------------------------------------------------------------------- host
// sizes: stage = records + payloads + interval tables, work = per image workspace (all 16-B aligned)
static int jpeg_sizes(const ssp_jpeg_item* items, int n, long long* stage, long long* work, std::vector<Desc>* descs) {
  if (!items || n < 0) return fail_msg(SSP_ERR_ARG, "jpeg: bad argument (null items or n < 0)");
  long long st = align16((long long)n * sizeof(ImgRec)), wk = 0;
  if (descs) descs->resize(n);
  Desc tmp;
  for (int i = 0; i < n; i++) {
    if (!items[i].data || items[i].size < 0) return fail_msg(SSP_ERR_ARG, "jpeg: bad item (null data or size < 0)");
    Desc& d = descs ? (*descs)[i] : tmp;
    if (parse(static_cast<const uint8_t*>(items[i].data), items[i].size, d) != kOk)
      return fail_msg(SSP_ERR_ARG, "jpeg: item is not decodable on the GPU (ssp_jpeg_parse declines it)");
    st += align16(d.seg_len + 8) + 2 * align16((n_intervals(d) + 1) * 4);
    wk += image_work(d, nsub_bound(d), nullptr, 0);
  }
  *stage = st; *work = wk;
  return SSP_OK;
}

}  // namespace ssp

using namespace ssp;

extern "C" {
int ssp_jpeg_parse(const void* data, long long size, ssp_jpeg_info* info) {
  if (!data || size < 0 || !info) return fail_msg(SSP_ERR_ARG, "jpeg_parse: bad argument (null pointer or size < 0)");
  static thread_local Desc d;
  const int rc = parse(static_cast<const uint8_t*>(data), size, d);
  memset(info, 0, sizeof(*info));
  info->width = d.w; info->height = d.h; info->components = d.ncomp;
  info->h_samp = d.comp[0].h; info->v_samp = d.comp[0].v; info->restart_interval = d.ri;
  return rc;
}

const char* ssp_jpeg_decline_reason(int code) { return code >= 0 && code < kNumDecline ? kDeclineText[code] : "unknown code"; }

long long ssp_jpeg_stage_bytes(const ssp_jpeg_item* items, int n) {
  long long s, w;
  const int rc = jpeg_sizes(items, n, &s, &w, nullptr);
  return rc ? rc : s;
}
long long ssp_jpeg_work_bytes(const ssp_jpeg_item* items, int n) {
  long long s, w;
  const int rc = jpeg_sizes(items, n, &s, &w, nullptr);
  return rc ? rc : w;
}

int ssp_jpeg_batch_plan(const ssp_jpeg_item* items, int n, void* stage_host, long long stage_bytes, long long* dims) {
  if (!stage_host || !dims) return fail_msg(SSP_ERR_ARG, "jpeg_batch_plan: bad argument (null pointer)");
  std::vector<Desc> descs;
  long long need_s, need_w;
  const int rc = jpeg_sizes(items, n, &need_s, &need_w, &descs);
  if (rc) return rc;
  if (stage_bytes < need_s) return fail_msg(SSP_ERR_ARG, "jpeg_batch_plan: staging buffer smaller than ssp_jpeg_stage_bytes()");
  for (int i = 0; i < n; i++)
    if (!items[i].out) return fail_msg(SSP_ERR_ARG, "jpeg_batch_plan: null output pointer");
  uint8_t* base = static_cast<uint8_t*>(stage_host);
  ImgRec* recs = reinterpret_cast<ImgRec*>(base);
  long long at = align16((long long)n * sizeof(ImgRec)), wat = 0, max_blocks = 0, max_pix = 0;
  for (int i = 0; i < n; i++) {
    ImgRec& r = recs[i];
    memset(&r, 0, sizeof(r));
    r.d = descs[i];
    const Desc& d = r.d;
    r.nint = n_intervals(d);
    r.out = static_cast<uint8_t*>(items[i].out);
    r.data_off = at;
    at += align16(d.seg_len + 8);
    r.ist_off = at;
    at += align16((r.nint + 1) * 4);
    r.ipref_off = at;
    at += align16((r.nint + 1) * 4);
    uint32_t* ist = reinterpret_cast<uint32_t*>(base + r.ist_off);
    int* ipref = reinterpret_cast<int*>(base + r.ipref_off);
    long long len = 0;
    r.pre_status = unstuff(static_cast<const uint8_t*>(items[i].data) + d.seg_off, d.seg_len, d, base + r.data_off, &len, ist);
    long long nsub = 0;
    ipref[0] = 0;
    if (!r.pre_status)
      for (long long j = 0; j < r.nint; j++) {
        const long long bits = ist[j + 1] - ist[j];
        nsub += bits ? (bits + kSubBits - 1) / kSubBits : 1;
        ipref[j + 1] = (int)nsub;
      }
    r.nsub = nsub;
    wat += image_work(d, nsub_bound(d), &r, wat);                // offsets from the start of `work`
    if (total_blocks(d) > max_blocks) max_blocks = total_blocks(d);
    if ((long long)d.w * d.h > max_pix) max_pix = (long long)d.w * d.h;
  }
  dims[0] = max_blocks; dims[1] = max_pix; dims[2] = need_w; dims[3] = at;
  return SSP_OK;
}

int ssp_jpeg_batch_run(const void* stage_dev, int n, const long long* dims, void* work, long long work_bytes, int* status, void* stream) {
  const cudaStream_t s = (cudaStream_t)stream;
  if (n < 0 || !dims) return fail_msg(SSP_ERR_ARG, "jpeg_batch_run: bad argument (n < 0 or null dims)");
  if (n == 0) return SSP_OK;
  if (!stage_dev || !work || !status) return fail_msg(SSP_ERR_ARG, "jpeg_batch_run: bad argument (null pointer)");
  if (n > 65535) return fail_msg(SSP_ERR_ARG, "jpeg_batch_run: more than 65535 images");
  if (work_bytes < dims[2]) return fail_msg(SSP_ERR_ARG, "jpeg_batch_run: work buffer smaller than ssp_jpeg_work_bytes()");
  const uint8_t* st = static_cast<const uint8_t*>(stage_dev);
  uint8_t* wk = static_cast<uint8_t*>(work);
  entropy_kernel<<<n, kEntropyThreads, 0, s>>>(st, wk, status, n);
  SSP_CHECK_LAUNCH();
  const long long gx = (dims[0] + kIdctBlocksPerCta - 1) / kIdctBlocksPerCta;
  idct_kernel<<<dim3((unsigned)gx, (unsigned)n), kIdctBlocksPerCta * 8, 0, s>>>(st, wk, status, status + n);
  SSP_CHECK_LAUNCH();
  const long long px = (dims[1] + 255) / 256;
  color_kernel<<<dim3((unsigned)(px < 4096 ? px : 4096), (unsigned)n), 256, 0, s>>>(st, wk, status, status + n);
  SSP_CHECK_LAUNCH();
  return SSP_OK;
}
}  // extern "C"
