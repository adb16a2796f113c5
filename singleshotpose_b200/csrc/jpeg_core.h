// Baseline JPEG decode rules, restated from ITU-T T.81 and libjpeg-turbo's published algorithms so that the output is
// byte-identical to what Pillow (built on libjpeg-turbo, default ISLOW IDCT and fancy upsampling) returns for
// Image.open(f).convert('RGB').  Compiled by nvcc into csrc/jpeg.cu and by g++ into tests/helpers/jpeg_host.cpp: both run the
// same phase functions, so the CPU suite checks the kernels' arithmetic against the installed Pillow bit for bit.
//
// Pipeline: parse (host) -> entropy decode into int16 coefficients in scan (MCU) order with DC differences -> per-component DC
// prefix sums (reset at each restart interval) -> dequantise + ISLOW IDCT into component planes -> fancy upsampling + YCbCr->RGB.
//
// Anything the GPU path cannot reproduce exactly is either declined at parse time (a reason code) or flagged per image at run
// time (a status bit); the caller decodes those images with Pillow.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define JHD __host__ __device__ __forceinline__
#else
#define JHD inline
#endif

namespace ssp_jpeg {

constexpr int kMaxComp = 3;
constexpr int kMaxBlocksPerMcu = 6;   // luma 2x2 + two 1x1 chroma
constexpr int kMaxTables = 4;         // distinct Huffman tables one scan may use here
constexpr int kLookBits = 9;          // fast Huffman lookup width
constexpr int kMaxDim = 65500;        // libjpeg's JPEG_MAX_DIMENSION

// status bits (per image, written by the decode)
constexpr int kStEntropy = 1;         // the entropy-coded segment is not a clean stream
constexpr int kStRange = 2;           // a block leaves the range where libjpeg-turbo's SIMD and C IDCT agree
constexpr int kStStructure = 4;       // restart markers missing, extra or out of sequence, or a marker inside the scan
constexpr int kStOverflow = 8;        // a DC prediction leaves int32 (libjpeg raises)

// decline codes of parse (0 = the GPU path takes the file)
enum Decline : int {
  kOk = 0, kNotJpeg, kTruncated, kProgressive, kArithmetic, kLossless, kPrecision, kCmyk, kRgbTransform, kComponents,
  kSampling, kMultiScan, kDnl, kNoEoi, kBadTable, kTooManyTables, kBadMarker, kTooLarge, kNumDecline
};
static const char* const kDeclineText[kNumDecline] = {
  "ok", "not a JPEG (no SOI)", "header truncated", "progressive", "arithmetic coding", "lossless or hierarchical",
  "not 8-bit precision", "CMYK/YCCK", "RGB-coded (Adobe transform 0 or 'RGB' component IDs)", "component count not 1 or 3",
  "sampling factors not supported", "multi-scan sequential", "height defined by DNL", "missing EOI",
  "bad quantisation or Huffman table", "more than 4 Huffman tables in the scan", "unsupported marker or segment",
  "image too large"};

struct HuffTable {
  uint16_t lut[1 << kLookBits];   // (length << 8) | symbol for codes of <= kLookBits bits; 0 = longer code
  int32_t maxcode[18];            // largest code of each length, -1 when none (T.81 F.2.2.3)
  int32_t valoff[17];             // huffval index of a code of length l = valoff[l] + code
  uint8_t huffval[256];
  uint8_t pad[4];
};

struct Comp {
  int h, v;          // sampling factors (1x1 for chroma and for a single-component image)
  int tq, dc, ac;    // quantisation table, compact Huffman table slots
  int bw, bh;        // plane size in blocks (MCU grid * sampling)
  int dw, dh;        // downsampled size in samples (libjpeg's downsampled_width / height)
};

// Everything the device needs about one image; filled by parse(), positions filled by the batch plan.
struct Desc {
  int w, h, ncomp, hmax, vmax;
  int mcux, mcuy, bpm;            // MCU grid, blocks per MCU
  int ri;                         // restart interval in MCUs (0: none)
  int ycc;                        // 3 components: YCbCr (1) -- the only 3-component colour space taken
  int blk_comp[kMaxBlocksPerMcu], blk_dx[kMaxBlocksPerMcu], blk_dy[kMaxBlocksPerMcu];
  Comp comp[kMaxComp];
  int ntab;
  long long seg_off, seg_len;     // entropy-coded segment in the file: bytes [seg_off, seg_off + seg_len)
  uint16_t quant[4][64];          // natural order
  HuffTable tab[kMaxTables];
};

JHD long long total_mcus(const Desc& d) { return (long long)d.mcux * d.mcuy; }
JHD long long total_blocks(const Desc& d) { return total_mcus(d) * d.bpm; }
JHD long long n_intervals(const Desc& d) { return d.ri ? (total_mcus(d) + d.ri - 1) / d.ri : 1; }
JHD long long interval_blocks(const Desc& d, long long j) {
  if (!d.ri) return total_blocks(d);
  const long long m = total_mcus(d) - j * d.ri;
  return (m < d.ri ? m : d.ri) * d.bpm;
}

#define SSP_JPEG_NATURAL {                                                                                              \
  0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, \
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
static const uint8_t kNatural[64] = SSP_JPEG_NATURAL;   // zigzag index -> natural (row-major) index
#ifdef __CUDACC__
__constant__ uint8_t kNaturalDev[64] = SSP_JPEG_NATURAL;
#endif
JHD int natural(int k) {
#ifdef __CUDA_ARCH__
  return kNaturalDev[k];
#else
  return kNatural[k];
#endif
}

// ------------------------------------------------------------------------------------------------ header parse (host)
// Canonical codes from BITS / HUFFVAL (T.81 Annex C); false for a table libjpeg rejects (over-full, or a DC symbol > 15).
inline bool build_table(const uint8_t bits[17], const uint8_t* vals, int nvals, bool dc, HuffTable& t) {
  memset(&t, 0, sizeof(t));
  memcpy(t.huffval, vals, nvals);
  int code = 0, p = 0;
  for (int l = 1; l <= 16; l++) {
    t.maxcode[l] = -1;
    if (bits[l]) {
      t.valoff[l] = p - code;
      for (int i = 0; i < bits[l]; i++, p++, code++)
        if (l <= kLookBits) {
          const int lo = code << (kLookBits - l), cnt = 1 << (kLookBits - l);
          for (int j = 0; j < cnt; j++) t.lut[lo + j] = (uint16_t)((l << 8) | vals[p]);
        }
      t.maxcode[l] = code - 1;
    }
    if (code >= (1 << l)) return false;          // no code may be all ones
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  if (dc)
    for (int i = 0; i < nvals; i++)
      if (vals[i] > 15) return false;
  return true;
}

inline int rd16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Parses SOI .. SOS and checks that the file ends with EOI.  Returns a Decline code; on kOk `d` is complete except positions.
inline int parse(const uint8_t* f, long long n, Desc& d) {
  memset(&d, 0, sizeof(d));
  if (n < 4 || f[0] != 0xFF || f[1] != 0xD8) return kNotJpeg;
  struct Raw { uint8_t bits[17]; uint8_t vals[256]; int nvals; bool set; } raw[2][4];
  bool qset[4] = {false, false, false, false};
  for (auto& a : raw) for (auto& r : a) r.set = false;
  int ids[kMaxComp] = {0, 0, 0}, hs[4] = {0}, vs[4] = {0}, tqs[4] = {0};
  bool sof = false, jfif = false, adobe = false;
  int transform = -1;
  long long p = 2;
  for (;;) {
    if (p >= n) return kTruncated;
    if (f[p] != 0xFF) return kBadMarker;
    while (p < n && f[p] == 0xFF) p++;           // fill bytes
    if (p >= n) return kTruncated;
    const int m = f[p++];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return kBadMarker;
    if (p + 2 > n) return kTruncated;
    const int len = rd16(f + p);
    if (len < 2) return kBadMarker;
    if (p + len > n) return kTruncated;
    const uint8_t* s = f + p + 2;
    const int sl = len - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (sof) return kBadMarker;
      sof = true;
      if (sl < 6) return kBadMarker;
      if (s[0] != 8) return kPrecision;
      d.h = rd16(s + 1); d.w = rd16(s + 3); d.ncomp = s[5];
      if (d.h == 0) return kDnl;
      if (d.w == 0) return kBadMarker;
      if (d.w > kMaxDim || d.h > kMaxDim) return kTooLarge;
      if (d.ncomp != 1 && d.ncomp != 3) return d.ncomp == 4 ? kCmyk : kComponents;
      if (sl < 6 + 3 * d.ncomp) return kBadMarker;
      for (int c = 0; c < d.ncomp; c++) {
        ids[c] = s[6 + 3 * c]; hs[c] = s[7 + 3 * c] >> 4; vs[c] = s[7 + 3 * c] & 15; tqs[c] = s[8 + 3 * c];
        if (hs[c] < 1 || hs[c] > 4 || vs[c] < 1 || vs[c] > 4 || tqs[c] > 3) return kBadMarker;
      }
    } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
      return m == 0xC2 ? kProgressive : (m == 0xCA ? kArithmetic : kLossless);
    } else if (m == 0xC3 || m == 0xC5 || m == 0xC7 || m == 0xCB || m == 0xCF || m == 0xDE || m == 0xDF) {
      return (m == 0xCB || m == 0xCF) ? kArithmetic : kLossless;
    } else if (m == 0xC9 || m == 0xCC) {
      return kArithmetic;
    } else if (m == 0xDB) {
      for (int q = 0; q < sl;) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        if (pq != 0) return kPrecision;          // 16-bit tables: outside what this decoder restates
        if (tq > 3 || q + 65 > sl) return kBadTable;
        for (int k = 0; k < 64; k++) d.quant[tq][kNatural[k]] = s[q + 1 + k];
        qset[tq] = true;
        q += 65;
      }
    } else if (m == 0xC4) {
      for (int q = 0; q < sl;) {
        const int tc = s[q] >> 4, th = s[q] & 15;
        if (tc > 1 || th > 3 || q + 17 > sl) return kBadTable;
        Raw& r = raw[tc][th];
        r.bits[0] = 0;
        int cnt = 0;
        for (int i = 1; i <= 16; i++) { r.bits[i] = s[q + i]; cnt += r.bits[i]; }
        if (cnt > 256 || q + 17 + cnt > sl) return kBadTable;
        memcpy(r.vals, s + q + 17, cnt);
        r.nvals = cnt; r.set = true;
        q += 17 + cnt;
      }
    } else if (m == 0xDD) {
      if (sl < 2) return kBadMarker;
      d.ri = rd16(s);
    } else if (m == 0xDC) {
      return kDnl;
    } else if (m == 0xE0) {                      // libjpeg examines at most the first 14 bytes
      if (sl >= 14 && s[0] == 'J' && s[1] == 'F' && s[2] == 'I' && s[3] == 'F' && s[4] == 0) jfif = true;
    } else if (m == 0xEE) {
      if (sl >= 12 && s[0] == 'A' && s[1] == 'd' && s[2] == 'o' && s[3] == 'b' && s[4] == 'e') { adobe = true; transform = s[11]; }
    } else if (m == 0xDA) {
      if (!sof) return kBadMarker;
      if (sl < 1) return kBadMarker;
      const int ns = s[0];
      if (sl < 1 + 2 * ns + 3) return kBadMarker;
      if (ns != d.ncomp) return kMultiScan;
      const int ss = s[1 + 2 * ns], se = s[2 + 2 * ns], ah = s[3 + 2 * ns] >> 4, al = s[3 + 2 * ns] & 15;
      if (ss != 0 || se != 63 || ah != 0 || al != 0) return kBadMarker;
      int slot_of[2][4];
      for (auto& a : slot_of) for (int& x : a) x = -1;
      d.ntab = 0;
      for (int i = 0; i < ns; i++) {
        const int cid = s[1 + 2 * i], td = s[2 + 2 * i] >> 4, ta = s[2 + 2 * i] & 15;
        if (cid != ids[i] || td > 3 || ta > 3) return kBadMarker;   // scan order = frame order (single interleaved scan)
        const int want[2] = {td, ta};
        int slot[2];
        for (int cls = 0; cls < 2; cls++) {
          int& sl2 = slot_of[cls][want[cls]];
          if (sl2 < 0) {
            const Raw& r = raw[cls][want[cls]];
            if (!r.set) return kBadTable;
            if (d.ntab == kMaxTables) return kTooManyTables;
            if (!build_table(r.bits, r.vals, r.nvals, cls == 0, d.tab[d.ntab])) return kBadTable;
            sl2 = d.ntab++;
          }
          slot[cls] = sl2;
        }
        d.comp[i].dc = slot[0]; d.comp[i].ac = slot[1];
      }
      for (int c = 0; c < d.ncomp; c++)
        if (!qset[tqs[c]]) return kBadTable;
      d.seg_off = p + len;
      break;
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {
      // other APPn and COM: skipped, as libjpeg does
    } else {
      return kBadMarker;
    }
    p += len;
  }
  if (n < d.seg_off + 2 || f[n - 2] != 0xFF || f[n - 1] != 0xD9) return kNoEoi;
  d.seg_len = n - 2 - d.seg_off;
  // colour space: libjpeg's default_decompress_parms
  if (d.ncomp == 3) {
    int cs_ycc;
    if (jfif) cs_ycc = 1;
    else if (adobe) cs_ycc = transform != 0;
    else cs_ycc = !(ids[0] == 82 && ids[1] == 71 && ids[2] == 66);
    if (!cs_ycc) return kRgbTransform;
    d.ycc = 1;
    if (!((hs[0] == 1 || hs[0] == 2) && (vs[0] == 1 || vs[0] == 2))) return kSampling;
    if (hs[1] != 1 || vs[1] != 1 || hs[2] != 1 || vs[2] != 1) return kSampling;
    d.hmax = hs[0]; d.vmax = vs[0];
    d.mcux = (d.w + 8 * d.hmax - 1) / (8 * d.hmax);
    d.mcuy = (d.h + 8 * d.vmax - 1) / (8 * d.vmax);
    int b = 0;
    for (int c = 0; c < 3; c++) {
      d.comp[c].h = hs[c]; d.comp[c].v = vs[c];
      for (int y = 0; y < vs[c]; y++)
        for (int x = 0; x < hs[c]; x++, b++) { d.blk_comp[b] = c; d.blk_dx[b] = x; d.blk_dy[b] = y; }
    }
    d.bpm = b;
  } else {                                       // one component: non-interleaved, one block per MCU
    d.hmax = d.vmax = 1;
    d.mcux = (d.w + 7) / 8; d.mcuy = (d.h + 7) / 8;
    d.comp[0].h = d.comp[0].v = 1;
    d.bpm = 1;
  }
  for (int c = 0; c < d.ncomp; c++) {
    Comp& k = d.comp[c];
    k.tq = tqs[c];
    k.bw = d.mcux * k.h; k.bh = d.mcuy * k.v;
    k.dw = (int)(((long long)d.w * k.h + d.hmax - 1) / d.hmax);
    k.dh = (int)(((long long)d.h * k.v + d.vmax - 1) / d.vmax);
  }
  if (total_blocks(d) > (1LL << 28)) return kTooLarge;
  return kOk;
}

// ------------------------------------------------------------------------------------------------ entropy decode
// The entropy-coded data is handed to the decoder without its stuffed zero bytes and restart markers (the batch plan copies it
// so), as one bit string per image; restart interval j occupies bits [istart[j], istart[j+1]).  `data` must be readable
// 8 bytes past the end.
//
// Decoder state between codewords: bit position, block of the MCU, zigzag index (0: a DC difference comes next).  Packed in
// 64 bits so that two states compare in one operation; kErrState is the state after an invalid stream.
struct State { uint32_t pos; int b, k; };
constexpr uint64_t kErrState = ~0ull;
JHD uint64_t pack(const State& s) { return ((uint64_t)s.pos << 32) | ((uint64_t)s.b << 8) | (uint64_t)s.k; }
JHD State unpack(uint64_t v) { return State{(uint32_t)(v >> 32), (int)((v >> 8) & 0xff), (int)(v & 0xff)}; }

// Host: copies the entropy-coded segment s[0..n) to dst without stuffed zero bytes and restart markers; ist[j] = first bit of
// interval j, ist[nint] = end.  dst needs n + 8 bytes.  Returns 0 or kStStructure: a marker other than the expected RSTn, or a
// restart count that does not match the image (libjpeg resynchronises there; such files go to Pillow).
inline int unstuff(const uint8_t* s, long long n, const Desc& d, uint8_t* dst, long long* out_len, uint32_t* ist) {
  const long long nint = n_intervals(d);
  long long o = 0, j = 0, i = 0;
  ist[0] = 0;
  while (i < n) {
    const uint8_t* ff = static_cast<const uint8_t*>(memchr(s + i, 0xFF, (size_t)(n - i)));
    const long long stop = ff ? ff - s : n;
    memcpy(dst + o, s + i, (size_t)(stop - i));
    o += stop - i;
    i = stop;
    if (i >= n) break;
    if (i + 1 >= n) return kStStructure;
    const uint8_t m = s[i + 1];
    if (m == 0x00) {
      dst[o++] = 0xFF;
    } else if (m >= 0xD0 && m <= 0xD7 && d.ri && m - 0xD0 == (int)(j % 8) && j + 1 < nint) {
      ist[++j] = (uint32_t)(o * 8);
    } else {
      return kStStructure;
    }
    i += 2;
  }
  if (j + 1 != nint || o * 8 > 0xF0000000LL) return kStStructure;
  ist[nint] = (uint32_t)(o * 8);
  memset(dst + o, 0, 8);                      // the bit reader looks up to 8 bytes ahead
  *out_len = o;
  return 0;
}

JHD uint32_t peek32(const uint8_t* data, uint32_t pos) {
  const uint8_t* p = data + (pos >> 3);
  const uint64_t w = ((uint64_t)p[0] << 32) | ((uint64_t)p[1] << 24) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 8) | p[4];
  return (uint32_t)(w >> (8 - (pos & 7)));
}

JHD int extend(int v, int s) { return s == 0 ? 0 : (v < (1 << (s - 1)) ? v - (1 << s) + 1 : v); }

// Decodes codewords from *st while st->pos < end, never reading a codeword that does not end by `limit` (the end of the
// restart interval).  Returns the number of blocks completed; *st becomes the state at the first codeword boundary >= end,
// or at the point where the next codeword does not fit (the interval's padding); *err = 1 for an invalid code or a coefficient
// index past 63.  With `resync` (a speculative decode from a guessed state) such an error is instead taken as a sign of a wrong
// guess: the decode restarts one bit further on with a new guess (the same block of the MCU, DC next).  With kWrite, writes each coefficient of
// block `blk0 + (blocks completed)` (AC at its natural index, the DC difference at index 0).
template <bool kWrite>
JHD long long decode_run(const Desc& d, const HuffTable* tab, const uint8_t* data, uint32_t end, uint32_t limit, State* st,
                         int* err, int16_t* coef, long long blk0, bool resync = false) {
  uint32_t pos = st->pos;
  int b = st->b, k = st->k;
  const int b0 = b;                              // a speculative decode keeps its guessed block phase when it resynchronises
  long long done = 0;
  while (pos < end) {
    const uint32_t w = peek32(data, pos);
    const int c = d.blk_comp[b];
    const HuffTable& t = tab[k == 0 ? d.comp[c].dc : d.comp[c].ac];
    int len, sym;
    const uint16_t e = t.lut[w >> (32 - kLookBits)];
    if (e) {
      len = e >> 8; sym = e & 0xff;
    } else {
      len = kLookBits + 1;
      while (len <= 16 && (int32_t)(w >> (32 - len)) > t.maxcode[len]) len++;
      if (len > 16) {                           // no code: past the interval's end it is its padding, else corrupt data
        if ((uint64_t)pos + 16 > limit) break;
        if (resync) { pos++; b = b0; k = 0; continue; }
        *err = 1;
        break;
      }
      sym = t.huffval[(t.valoff[len] + (int32_t)(w >> (32 - len))) & 0xff];
    }
    const int s = sym & 15, r = sym >> 4;
    const int nb = (k == 0) ? sym : s;           // DC: the symbol is the magnitude category (<= 15, parse checks)
    if ((uint64_t)pos + len + nb > limit) break; // does not fit: the interval's padding
    const int v = nb ? extend((int)((w << len) >> (32 - nb)), nb) : 0;
    pos += len + nb;
    if (k == 0) {
      if (kWrite) coef[(blk0 + done) * 64] = (int16_t)v;
      k = 1;
    } else if (s) {
      k += r;
      if (k > 63) {
        if (resync) { b = b0; k = 0; continue; }
        *err = 1;
        break;
      }
      if (kWrite) coef[(blk0 + done) * 64 + natural(k)] = (int16_t)v;
      k++;
    } else if (r == 15) {
      k += 16;
      if (k > 64) {
        if (resync) { b = b0; k = 0; continue; }
        *err = 1;
        break;
      }
    } else {
      k = 64;                                    // EOB
    }
    if (k == 64) {
      k = 0; done++;
      if (++b == d.bpm) b = 0;
    }
  }
  st->pos = pos; st->b = b; st->k = k;
  return done;
}

// One subsequence of the self-synchronising decode: from state `in` (kErrState propagates) decode until the first codeword
// boundary at or after `end`.  This is the function the sync rounds iterate: out = f(in).  `guess`: `in` is a guess (the first
// pass), so errors resynchronise instead of ending in kErrState; a wrong guess only costs rounds, it is never relied on.
JHD uint64_t sub_step(const Desc& d, const HuffTable* tab, const uint8_t* data, uint32_t end, uint32_t limit, uint64_t in,
                      long long* nblk, bool guess = false) {
  *nblk = 0;
  if (in == kErrState) return kErrState;
  State st = unpack(in);
  int err = 0;
  *nblk = decode_run<false>(d, tab, data, end, limit, &st, &err, nullptr, 0, guess);
  return err ? kErrState : pack(st);
}

// Phase recovery of the self-synchronising decode.  A speculative decode from a guessed state rejoins the true decode only if,
// once their codeword boundaries agree, they also agree on the block of the MCU (each block has its own tables).  So every
// subsequence t is decoded speculatively from each block phase p: cand[t][p] is the end state from (first bit, block p, DC next)
// (the first subsequence of an interval has the exact start: only p = 0, the others are kNone).  link[t][p] = q when the exact
// decode of subsequence t from cand[t-1][p] ends in cand[t][q] (-1 when it ends in none), lcnt[t][p] its block count.
// walk_interval then follows the chain: while the true state of subsequence t-1 is a candidate, the true state of t is read
// from the link; otherwise subsequence t is decoded from it.  Every state it writes is the exact decoder's state, because each
// link was established by an exact decode from that very state -- fast synchronisation saves decodes, it is never assumed.
constexpr uint64_t kNone = ~1ull;                // never a packed state (b would be 255, k 254)
JHD uint32_t sub_end(uint32_t istart, uint32_t limit, int sub_bits, long long u) {
  const uint64_t e = (uint64_t)istart + (uint64_t)(u + 1) * sub_bits;
  return e < limit ? (uint32_t)e : limit;
}
JHD void walk_interval(const Desc& d, const HuffTable* tab, const uint8_t* data, uint32_t istart, uint32_t limit, int sub_bits,
                       long long t0, long long t1, const uint64_t* cand, const int* link, const long long* lcnt,
                       const long long* cnt0, uint64_t* S, long long* cnt, long long* decodes) {
  const int P = d.bpm;
  int q = 0;
  S[t0] = cand[t0 * P];
  cnt[t0] = cnt0[t0];
  for (long long t = t0 + 1; t < t1; t++) {
    if (q >= 0 && link[t * P + q] >= 0) {
      cnt[t] = lcnt[t * P + q];
      q = link[t * P + q];
      S[t] = cand[t * P + q];
      continue;
    }
    (*decodes)++;
    S[t] = sub_step(d, tab, data, sub_end(istart, limit, sub_bits, t - t0), limit, S[t - 1], &cnt[t]);
    q = -1;
    for (int p = 0; p < P; p++)
      if (cand[t * P + p] == S[t]) { q = p; break; }
  }
}

// Per-component DC prediction: the decoded value of a component's block is the running sum of its DC differences, reset to 0
// at every restart interval.  Element e of component c (scan order) is block block_of(d, c, e).
JHD long long comp_blocks(const Desc& d, int c) { return total_mcus(d) * d.comp[c].h * d.comp[c].v; }
JHD long long block_of(const Desc& d, int c, long long e, bool* reset) {
  const int per = d.comp[c].h * d.comp[c].v;
  int off = 0;
  for (int b = 0; b < d.bpm && d.blk_comp[b] != c; b++) off++;
  const long long m = e / per;
  const int within = (int)(e % per);
  *reset = within == 0 && (d.ri ? m % d.ri == 0 : m == 0);
  return m * d.bpm + off + within;
}

// ------------------------------------------------------------------------------------------------ IDCT (jidctint ISLOW)
// C semantics with 64-bit intermediates (libjpeg's JLONG on LP64).  libjpeg-turbo's x86 SIMD ISLOW works in 16-bit lanes;
// it agrees with this whenever every dequantised coefficient and every pass-1 value fits int16 and every output lies in
// [-512, 511] (where the C range-limit table is monotonic).  Otherwise *range_flag is set and the image goes to Pillow.
constexpr int kConstBits = 13, kPass1Bits = 2;
JHD long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

template <class Get, class Put>
JHD void idct_1d(Get in, Put out, int shift) {
  long long z2 = in(2), z3 = in(6);
  long long z1 = (z2 + z3) * 4433;                          // FIX(0.541196100)
  long long tmp2 = z1 + z3 * -15137;                        // FIX(1.847759065)
  long long tmp3 = z1 + z2 * 6270;                          // FIX(0.765366865)
  z2 = in(0); z3 = in(4);
  long long tmp0 = (z2 + z3) * (1LL << kConstBits);
  long long tmp1 = (z2 - z3) * (1LL << kConstBits);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in(7); tmp1 = in(5); tmp2 = in(3); tmp3 = in(1);
  z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * 9633;                    // FIX(1.175875602)
  tmp0 = tmp0 * 2446; tmp1 = tmp1 * 16819; tmp2 = tmp2 * 25172; tmp3 = tmp3 * 12299;
  z1 = z1 * -7373; z2 = z2 * -20995; z3 = z3 * -16069; z4 = z4 * -3196;
  z3 += z5; z4 += z5;
  tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
  out(0, descale(tmp10 + tmp3, shift)); out(7, descale(tmp10 - tmp3, shift));
  out(1, descale(tmp11 + tmp2, shift)); out(6, descale(tmp11 - tmp2, shift));
  out(2, descale(tmp12 + tmp1, shift)); out(5, descale(tmp12 - tmp1, shift));
  out(3, descale(tmp13 + tmp0, shift)); out(4, descale(tmp13 - tmp0, shift));
}

JHD bool fits16(long long v) { return v >= -32768 && v <= 32767; }

// libjpeg's post-IDCT range limit: table[(v) & 1023] with CENTERJSAMPLE added
JHD uint8_t range_limit_idct(long long v) {
  const int i = (int)(v & 1023);
  if (i < 128) return (uint8_t)(i + 128);
  if (i < 512) return 255;
  if (i < 896) return 0;
  return (uint8_t)(i - 896);
}

// Pass 1 on column `col` of block `blk` (natural order) into ws[8][8] (ws[row][col]).
JHD void idct_pass1(const int16_t* blk, const uint16_t* q, int col, int* ws, int* flag) {
  long long deq[8];
  for (int r = 0; r < 8; r++) {
    deq[r] = (long long)blk[r * 8 + col] * q[r * 8 + col];
    if (!fits16(deq[r])) *flag = 1;
  }
  idct_1d([&](int r) { return deq[r]; },
          [&](int r, long long v) { if (!fits16(v)) *flag = 1; ws[r * 8 + col] = (int)v; }, kConstBits - kPass1Bits);
}

// Pass 2 on row `row` of ws into out[0..7].
JHD void idct_pass2(const int* ws, int row, uint8_t* out, int* flag) {
  const int* w = ws + row * 8;
  idct_1d([&](int c) { return (long long)w[c]; },
          [&](int c, long long v) { if (v < -512 || v > 511) *flag = 1; out[c] = range_limit_idct(v); },
          kConstBits + kPass1Bits + 3);
}

// ------------------------------------------------------------------------------------------------ upsampling + colour
// Sample of component c (plane pitch `pitch`) that libjpeg-turbo's default upsampler produces at output pixel (x, y).
// h2v1 / h2v2 fancy filters need a downsampled width > 2 (otherwise libjpeg replicates); h1v2 is always fancy.  Context
// columns and rows are clamped to the real downsampled size: libjpeg replicates the edge column / the first and last real row.
JHD int upsample(const Desc& d, int c, const uint8_t* plane, int pitch, int x, int y) {
  const Comp& k = d.comp[c];
  const int fh = d.hmax / k.h, fv = d.vmax / k.v;           // 1 or 2
  if (fh == 1 && fv == 1) return plane[(long long)y * pitch + x];
  const int cx = x / fh, cy = y / fv;
  if (fh == 2 && k.dw <= 2) {                                // box replication (h2v1_upsample / h2v2_upsample)
    return plane[(long long)cy * pitch + cx];
  }
  auto at = [&](int xx, int yy) -> int {
    xx = xx < 0 ? 0 : (xx >= k.dw ? k.dw - 1 : xx);
    yy = yy < 0 ? 0 : (yy >= k.dh ? k.dh - 1 : yy);
    return plane[(long long)yy * pitch + xx];
  };
  if (fv == 1) {                                             // h2v1
    const int near = at(cx, cy) * 3;
    return (x & 1) ? (near + at(cx + 1, cy) + 2) >> 2 : (near + at(cx - 1, cy) + 1) >> 2;
  }
  const int ny = (y & 1) ? cy + 1 : cy - 1;                  // the next-nearest row: above for even rows, below for odd
  if (fh == 1) {                                             // h1v2
    const int sum = at(cx, cy) * 3 + at(cx, ny);
    return (sum + ((y & 1) ? 2 : 1)) >> 2;
  }
  const int sum = at(cx, cy) * 3 + at(cx, ny);               // h2v2: vertical 3:1 column sums, then horizontal
  if (x & 1) return (sum * 3 + at(cx + 1, cy) * 3 + at(cx + 1, ny) + 7) >> 4;
  return (sum * 3 + at(cx - 1, cy) * 3 + at(cx - 1, ny) + 8) >> 4;
}

// jdcolor's ycc_rgb_convert: SCALEBITS 16 fixed point tables, range-limited
JHD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
JHD void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
  const long long half = 1LL << 15;
  const long long xcb = cb - 128, xcr = cr - 128;
  const int r_off = (int)((91881 * xcr + half) >> 16);           // FIX(1.40200)
  const int b_off = (int)((116130 * xcb + half) >> 16);          // FIX(1.77200)
  const int g_off = (int)((-22554 * xcb + half + -46802 * xcr) >> 16);   // -FIX(0.34414), -FIX(0.71414)
  rgb[0] = clamp255(y + r_off);
  rgb[1] = clamp255(y + g_off);
  rgb[2] = clamp255(y + b_off);
}

}  // namespace ssp_jpeg
