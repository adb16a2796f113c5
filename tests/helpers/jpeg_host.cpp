// Host harness of the JPEG decode rules of jpeg_core.h, driven the way entropy_kernel / idct_kernel / color_kernel (jpeg.cu)
// drive them, with plain loops: the same unstuffing, the same subsequence geometry, the same candidates, links and walk,
// the same block offsets and checks, the same IDCT and colour functions.  The subsequence length is a parameter, so a
// tiny one forces many candidate links and serial decodes.  Test infrastructure: built by tests/test_jpeg_cpu.py into a temporary .so (also with
// -fsanitize=address,undefined); never loaded by the product.
#include <limits.h>

#include <vector>

#include "../../singleshotpose_b200/csrc/jpeg_core.h"

using namespace ssp_jpeg;

extern "C" {
// info[6] = w, h, components, luma h, luma v, restart interval.  Returns the decline code (0: decodable).
int h_parse(const uint8_t* f, long long n, int* info) {
  static Desc d;
  const int rc = parse(f, n, d);
  info[0] = d.w; info[1] = d.h; info[2] = d.ncomp; info[3] = d.comp[0].h; info[4] = d.comp[0].v; info[5] = d.ri;
  return rc;
}

const char* h_reason(int code) { return code >= 0 && code < kNumDecline ? kDeclineText[code] : "unknown code"; }

// Decodes f into out (h*w*3, RGB).  Returns -(decline code) when parse declines, else the status word (0 = out written).
// stats[2] = subsequences the walk had to decode serially (no candidate link), subsequences.
int h_decode(const uint8_t* f, long long n, int sub_bits, uint8_t* out, long long* stats) {
  static Desc d;
  const int rc = parse(f, n, d);
  if (rc) return -rc;
  const long long nint = n_intervals(d);
  std::vector<uint8_t> data(d.seg_len + 8);
  std::vector<uint32_t> ist(nint + 1);
  long long len = 0;
  const int pre = unstuff(f + d.seg_off, d.seg_len, d, data.data(), &len, ist.data());
  if (pre) return pre;
  std::vector<long long> ipref(nint + 1, 0);
  for (long long j = 0; j < nint; j++) {
    const long long bits = ist[j + 1] - ist[j];
    ipref[j + 1] = ipref[j] + (bits ? (bits + sub_bits - 1) / sub_bits : 1);
  }
  const long long nsub = ipref[nint];
  std::vector<uint32_t> start(nsub), end(nsub), limit(nsub);
  std::vector<char> first(nsub);
  for (long long j = 0; j < nint; j++)
    for (long long t = ipref[j]; t < ipref[j + 1]; t++) {
      start[t] = ist[j] + (uint32_t)((t - ipref[j]) * sub_bits);
      limit[t] = ist[j + 1];
      end[t] = start[t] + sub_bits < limit[t] ? start[t] + sub_bits : limit[t];
      first[t] = t == ipref[j];
    }
  // candidates from every block phase, links between neighbouring candidates, then the walk (jpeg_core.h walk_interval)
  const int P = d.bpm;
  std::vector<uint64_t> cand(nsub * P, kNone), fin(nsub);
  std::vector<int> link(nsub * P, -1);
  std::vector<long long> lcnt(nsub * P, 0), cnt0(nsub, 0), cnt(nsub);
  for (long long t = 0; t < nsub; t++)
    for (int p = 0; p < (first[t] ? 1 : P); p++) {
      long long nb;
      cand[t * P + p] = sub_step(d, d.tab, data.data(), end[t], limit[t], pack(State{start[t], p, 0}), &nb, !first[t]);
      if (first[t]) cnt0[t] = nb;
    }
  for (long long t = 0; t < nsub; t++)
    for (int p = 0; p < P && !first[t]; p++) {
      if (cand[(t - 1) * P + p] == kNone) continue;
      const uint64_t e = sub_step(d, d.tab, data.data(), end[t], limit[t], cand[(t - 1) * P + p], &lcnt[t * P + p]);
      for (int q = 0; q < P; q++)
        if (cand[t * P + q] == e) { link[t * P + p] = q; break; }
    }
  long long decodes = 0;
  for (long long j = 0; j < nint; j++)
    walk_interval(d, d.tab, data.data(), ist[j], ist[j + 1], sub_bits, ipref[j], ipref[j + 1], cand.data(), link.data(), lcnt.data(),
                  cnt0.data(), fin.data(), cnt.data(), &decodes);
  stats[0] = decodes; stats[1] = nsub;
  long long total = 0;
  for (long long t = 0; t < nsub; t++) { const long long x = cnt[t]; cnt[t] = total; total += x; }
  for (long long j = 0; j < nint; j++) {
    const long long t0 = ipref[j], t1 = ipref[j + 1];
    const long long got = (t1 < nsub ? cnt[t1] : total) - cnt[t0];
    const uint64_t e = fin[t1 - 1];
    if (e == kErrState) return kStEntropy;
    const State st = unpack(e);
    if (got != interval_blocks(d, j) || st.k != 0 || ist[j + 1] - st.pos >= 8) return kStEntropy;
  }
  std::vector<int16_t> coef(total_blocks(d) * 64, 0);
  for (long long t = 0; t < nsub; t++) {
    State st = first[t] ? State{start[t], 0, 0} : unpack(fin[t - 1]);
    int err = 0;
    decode_run<true>(d, d.tab, data.data(), end[t], limit[t], &st, &err, coef.data(), cnt[t]);
  }
  for (int c = 0; c < d.ncomp; c++) {
    long long s = 0;
    for (long long e = 0; e < comp_blocks(d, c); e++) {
      bool rs;
      const long long i = block_of(d, c, e, &rs);
      if (rs) s = 0;
      s += coef[i * 64];
      if (s > INT_MAX || s < INT_MIN) return kStOverflow;
      coef[i * 64] = (int16_t)s;
    }
  }
  std::vector<std::vector<uint8_t>> planes(d.ncomp);
  for (int c = 0; c < d.ncomp; c++) planes[c].assign((size_t)d.comp[c].bw * d.comp[c].bh * 64, 0);
  int flag = 0;
  for (long long blk = 0; blk < total_blocks(d); blk++) {
    const long long m = blk / d.bpm;
    const int b = (int)(blk % d.bpm), c = d.blk_comp[b];
    const Comp& k = d.comp[c];
    int ws[64];
    for (int col = 0; col < 8; col++) idct_pass1(coef.data() + blk * 64, d.quant[k.tq], col, ws, &flag);
    const long long bx = (m % d.mcux) * k.h + d.blk_dx[b], by = (m / d.mcux) * k.v + d.blk_dy[b];
    for (int row = 0; row < 8; row++) idct_pass2(ws, row, &planes[c][(by * 8 + row) * k.bw * 8 + bx * 8], &flag);
  }
  if (flag) return kStRange;
  for (int y = 0; y < d.h; y++)
    for (int x = 0; x < d.w; x++) {
      uint8_t* o = out + ((long long)y * d.w + x) * 3;
      const int yv = planes[0][(long long)y * d.comp[0].bw * 8 + x];
      if (d.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)yv;
      } else {
        ycc_to_rgb(yv, upsample(d, 1, planes[1].data(), d.comp[1].bw * 8, x, y), upsample(d, 2, planes[2].data(), d.comp[2].bw * 8, x, y), o);
      }
    }
  return 0;
}
}

#ifdef JPEG_HOST_MAIN
// Sanitizer driver (a sanitized library cannot be loaded into a plain Python): argv[1] lists one input path per line; for
// each, writes <path>.out = int32 status (h_decode's return) followed by the RGB bytes when the status is 0.
#include <stdio.h>
#include <stdlib.h>
#include <string>
int main(int argc, char** argv) {
  if (argc != 3) return 2;
  const int sub_bits = atoi(argv[2]);
  FILE* lst = fopen(argv[1], "r");
  if (!lst) return 2;
  char line[4096];
  while (fgets(line, sizeof(line), lst)) {
    std::string path(line);
    while (!path.empty() && (path.back() == '\n' || path.back() == '\r')) path.pop_back();
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return 3;
    std::vector<uint8_t> buf;
    uint8_t tmp[65536];
    size_t k;
    while ((k = fread(tmp, 1, sizeof(tmp), f)) > 0) buf.insert(buf.end(), tmp, tmp + k);
    fclose(f);
    int info[6];
    std::vector<uint8_t> out;
    if (h_parse(buf.data(), (long long)buf.size(), info) == 0) out.resize((size_t)info[0] * info[1] * 3);
    long long stats[2];
    const int rc = h_decode(buf.data(), (long long)buf.size(), sub_bits, out.data(), stats);
    FILE* o = fopen((path + ".out").c_str(), "wb");
    fwrite(&rc, 4, 1, o);
    if (rc == 0) fwrite(out.data(), 1, out.size(), o);
    fclose(o);
  }
  fclose(lst);
  return 0;
}
#endif
