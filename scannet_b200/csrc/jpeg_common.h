// The JPEG format and stb_image v2.08's arithmetic, shared by the host decoder (jpeg.cpp) and the device decoder (jpeg_gpu.cu)
// so that both read the same segments the same way and compute the same bytes.
// Huffman tables: layout and construction follow the lookups of stb_image v2.08 (/root/reference/SensReader/c++/src/sensorData/
// stb_image.h: stbi__build_huffman :1590-1632, stbi__build_fast_ac :1636-1660) so that both decoders take the same path through
// the same bits: a 9-bit lookahead `fast` table, canonical maxcode/mincode/valptr for longer codes, and for AC tables `fast_ac`,
// which folds a short code and a small coefficient into one lookup.  Plain data: a table set is memcpy'd to the device as is.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#ifdef __CUDACC__
#define SCN_JPEG_HD __host__ __device__ __forceinline__
#else
#define SCN_JPEG_HD inline
#endif

namespace scn_jpeg {

constexpr int kFastBits = 9;

// zig-zag order, padded so that a run past the end of a block lands on coefficient 63 (stb_image.h:1467-1481).  The initialiser
// also fills the device decoder's __constant__ copy.
#define SCN_JPEG_ZIG {0,1,8,16,9,2,3,10,17,24,32,25,18,11,4,5,12,19,26,33,40,48,41,34,27,20,13,6,7,14,21,28,35,42,49,56,57,50,43,36, \
                      29,22,15,23,30,37,44,51,58,59,52,45,38,31,39,46,53,60,61,54,47,55,62,63,                                    \
                      63,63,63,63,63,63,63,63,63,63,63,63,63,63,63}
static const uint8_t kZig[64 + 15] = SCN_JPEG_ZIG;

struct HuffTab {
  int32_t present;
  int32_t maxcode[18]; int32_t valptr[17]; int32_t mincode[17];
  uint8_t vals[256];
  uint16_t fast[1 << kFastBits];          // (symbol << 4) | length for codes of <= 9 bits, 0xFFFF = longer code
  int16_t fast_ac[1 << kFastBits];        // AC tables: (value << 8) | (run << 4) | (code+magnitude bits) when both fit in 9 bits, else 0

  void build_fast_ac() {
    for (int i = 0; i < (1 << kFastBits); ++i) {
      fast_ac[i] = 0;
      const uint16_t e = fast[i];
      if (e == 0xFFFF) continue;
      const int rs = e >> 4, len = e & 15, run = rs >> 4, mag = rs & 15;
      if (mag && len + mag <= kFastBits) {
        int k = ((i << len) & ((1 << kFastBits) - 1)) >> (kFastBits - mag);
        if (k < (1 << (mag - 1))) k -= (1 << mag) - 1;                       // extend
        if (k >= -128 && k <= 127) fast_ac[i] = (int16_t)((k * 256) + (run * 16) + (len + mag));
      }
    }
  }
  bool build(const uint8_t* counts, const uint8_t* symbols, int nsym) {
    int code = 0, k = 0;
    // validate before any table write (stb_image.h:1590-1615 rejects over-subscribed lengths before building its fast
    // table): an over-subscribed code would index far outside fast[]
    for (int l = 1, c = 0, tot = 0; l <= 16; ++l) {
      c += counts[l - 1]; tot += counts[l - 1];
      if (c > (1 << l) || tot > nsym || tot > 256) return false;
      c <<= 1;
    }
    for (int i = 0; i < (1 << kFastBits); ++i) fast[i] = 0xFFFF;
    memset(fast_ac, 0, sizeof(fast_ac));
    memset(vals, 0, sizeof(vals));
    for (int l = 1; l <= 16; ++l) {
      valptr[l] = k; mincode[l] = code;
      if (l <= kFastBits)
        for (int j = 0; j < counts[l - 1]; ++j) {
          const int c = (code + j) << (kFastBits - l);
          for (int f = 0; f < (1 << (kFastBits - l)); ++f) fast[c + f] = (uint16_t)((symbols[k + j] << 4) | l);
        }
      code += counts[l - 1]; k += counts[l - 1];
      if (code > (1 << l)) return false;
      maxcode[l] = counts[l - 1] ? code - 1 : -1;
      code <<= 1;
    }
    valptr[0] = 0; mincode[0] = 0; maxcode[0] = -1;
    maxcode[17] = 0x7FFFFFFF;
    memcpy(vals, symbols, (size_t)nsym);
    present = 1;
    return true;
  }
};

// ---- stb's numerics ------------------------------------------------------------------------------------------------------------
SCN_JPEG_HD int extend(int v, int t) { return v < (1 << (t - 1)) ? v - (1 << t) + 1 : v; }      // a t-bit magnitude as a coefficient
SCN_JPEG_HD int clamp8(int x) { return (unsigned)x > 255u ? (x < 0 ? 0 : 255) : x; }

// one pass of the integer "islow" IDCT with 12-bit constants (stb_image.h:1928-2027): declares t0-t3, x0-x3 and the rest; the
// caller adds its rounding bias to x0-x3 and shifts x +- t
#define F2F(x) ((int)(((x) * 4096 + 0.5)))
#define IDCT_1D(s0, s1, s2, s3, s4, s5, s6, s7)                                      \
  int t0, t1, t2, t3, p1, p2, p3, p4, p5, x0, x1, x2, x3;                            \
  p2 = s2; p3 = s6;                                                                  \
  p1 = (p2 + p3) * F2F(0.5411961f);                                                  \
  t2 = p1 + p3 * F2F(-1.847759065f);                                                 \
  t3 = p1 + p2 * F2F(0.765366865f);                                                  \
  p2 = s0; p3 = s4;                                                                  \
  t0 = (p2 + p3) << 12; t1 = (p2 - p3) << 12;                                        \
  x0 = t0 + t3; x3 = t0 - t3; x1 = t1 + t2; x2 = t1 - t2;                            \
  t0 = s7; t1 = s5; t2 = s3; t3 = s1;                                                \
  p3 = t0 + t2; p4 = t1 + t3; p1 = t0 + t3; p2 = t1 + t2;                            \
  p5 = (p3 + p4) * F2F(1.175875602f);                                                \
  t0 = t0 * F2F(0.298631336f); t1 = t1 * F2F(2.053119869f);                          \
  t2 = t2 * F2F(3.072711026f); t3 = t3 * F2F(1.501321110f);                          \
  p1 = p5 + p1 * F2F(-0.899976223f); p2 = p5 + p2 * F2F(-2.562915447f);              \
  p3 = p3 * F2F(-1.961570560f); p4 = p4 * F2F(-0.390180644f);                        \
  t3 += p1 + p4; t2 += p2 + p3; t1 += p2 + p4; t0 += p1 + p3;

// YCbCr -> RGB in 20-bit fixed point with the masked Cb term (stb_image.h:3091-3118), as r | g << 8 | b << 16
#define FIX20(x) (((int)((x) * 4096.0f + 0.5f)) << 8)
SCN_JPEG_HD unsigned ycc_to_rgb(int y, int cbv, int crv) {
  const int yf = (y << 20) + (1 << 19), cr = crv - 128, cb = cbv - 128;
  int r = yf + cr * FIX20(1.40200f);
  int g = yf + (cr * -FIX20(0.71414f)) + ((cb * -FIX20(0.34414f)) & 0xffff0000);
  int b = yf + cb * FIX20(1.77200f);
  r >>= 20; g >>= 20; b >>= 20;
  return (unsigned)clamp8(r) | ((unsigned)clamp8(g) << 8) | ((unsigned)clamp8(b) << 16);
}

// ---- marker parser -------------------------------------------------------------------------------------------------------------
// What parse_header found: a scan, the end of the stream, or why it refuses the stream (jpeg.cpp turns each refusal into its error)
enum Parse { kScan, kEnd, kTruncated, kBadLength, kDqt16, kBadDqt, kBadDht, kBadCodeLengths, kBadDri, kNot8Bit, kBadSof, kBadSize,
             kBadSofComponent, kSosBeforeSof, kBadSos, kBadSosComponent, kMissingTable };

struct FrameComp { int id, h, v, tq, td, ta; };      // td / ta: the Huffman tables the latest scan gave the component

// What the segments before a scan establish.  It persists from one scan to the next.
struct Header {
  uint32_t want_w, want_h;                            // the container's frame size: a frame header must agree with it
  uint8_t quant[4][64]; bool have_q[4];               // natural order
  HuffTab dc[4], ac[4];
  int restart = 0;                                    // DRI: MCUs per restart interval, 0 = none
  int sof = 0, n_sof = 0;                             // marker of the last frame header (C0, C1 or C2, 0 = none yet); how many came
  bool other_sof = false;                             // a frame header of another process (lossless, arithmetic ...): skipped
  int W = 0, H = 0, ncomp = 0, hmax = 1, vmax = 1;    // hmax / vmax: largest sampling factors of every frame header so far
  FrameComp comp[3] = {};
  Header(uint32_t w, uint32_t h) : want_w(w), want_h(h), quant(), have_q() { for (int i = 0; i < 4; ++i) dc[i].present = ac[i].present = 0; }
};

// A scan header: per SOS entry the component (index into Header::comp) and its DC / AC table ids; spectral selection and
// successive approximation (se = 63 in a sequential scan); the offset of the entropy-coded segment
struct Scan { int ns, comp[3], td[3], ta[3], ss, se, ah, al; size_t data; };

// Walks the markers from `pos` (after SOI, or after a scan's entropy-coded data) and applies DQT, DHT, DRI and frame headers to
// `h`, up to and including the next SOS (kScan: `scan` describes it) or EOI / the end of the data (kEnd).  Anything else refuses
// the stream.  The raw DQT / DHT segments are appended to `tables` when it is given: they tell table sets apart.
inline Parse parse_header(const uint8_t* d, size_t n, size_t pos, Header& h, Scan& scan, std::vector<uint8_t>* tables = nullptr) {
  for (;;) {
    while (pos < n && d[pos] != 0xFF) ++pos;
    while (pos < n && d[pos] == 0xFF) ++pos;
    if (pos >= n) return kEnd;
    const int m = d[pos++];
    if (m == 0xD9) return kEnd;
    if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
    if (pos + 2 > n) return kTruncated;
    const size_t len = ((size_t)d[pos] << 8) | d[pos + 1];
    if (len < 2 || pos + len > n) return kBadLength;
    const uint8_t* s = d + pos + 2; size_t sl = len - 2;
    if (tables && (m == 0xDB || m == 0xC4)) tables->insert(tables->end(), d + pos - 1, d + pos + len);
    if (m == 0xDB) {
      while (sl > 0) {
        const int pq = s[0] >> 4, tq = s[0] & 15;
        if (pq != 0) return kDqt16;
        if (tq > 3 || sl < 65) return kBadDqt;
        for (int i = 0; i < 64; ++i) h.quant[tq][kZig[i]] = s[1 + i];
        h.have_q[tq] = true; s += 65; sl -= 65;
      }
    } else if (m == 0xC4) {
      while (sl > 0) {
        if (sl < 17) return kBadDht;
        const int tc = s[0] >> 4, th = s[0] & 15; int tot = 0;
        for (int i = 0; i < 16; ++i) tot += s[1 + i];
        if (tc > 1 || th > 3 || tot > 256 || sl < (size_t)(17 + tot)) return kBadDht;
        HuffTab& t = tc ? h.ac[th] : h.dc[th];
        if (!t.build(s + 1, s + 17, tot)) return kBadCodeLengths;
        if (tc) t.build_fast_ac();
        s += 17 + tot; sl -= 17 + tot;
      }
    } else if (m == 0xDD) { if (sl < 2) return kBadDri; h.restart = (s[0] << 8) | s[1]; }
    else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
      if (sl < 6 || s[0] != 8) return kNot8Bit;
      h.H = (s[1] << 8) | s[2]; h.W = (s[3] << 8) | s[4]; h.ncomp = s[5];
      if ((h.ncomp != 1 && h.ncomp != 3) || sl < (size_t)(6 + 3 * h.ncomp) || h.W == 0 || h.H == 0) return kBadSof;
      // the container's header fixes the frame size: refuse before any plane is sized from in-stream values
      if ((uint32_t)h.W != h.want_w || (uint32_t)h.H != h.want_h) return kBadSize;
      for (int i = 0; i < h.ncomp; ++i) {
        FrameComp& c = h.comp[i];
        c.id = s[6 + 3 * i]; c.h = s[7 + 3 * i] >> 4; c.v = s[7 + 3 * i] & 15; c.tq = s[8 + 3 * i];
        if (!c.h || c.h > 4 || !c.v || c.v > 4 || c.tq > 3) return kBadSofComponent;
        h.hmax = std::max(h.hmax, c.h); h.vmax = std::max(h.vmax, c.v);
      }
      h.sof = m; ++h.n_sof;
    } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) h.other_sof = true;
    else if (m == 0xDA) {
      if (!h.sof) return kSosBeforeSof;
      const int ns = sl ? s[0] : 0;
      if (ns < 1 || ns > h.ncomp || sl < (size_t)(1 + 2 * ns + 3)) return kBadSos;
      scan.ns = ns;
      for (int i = 0; i < ns; ++i) {
        int which = -1;
        for (int c = 0; c < h.ncomp; ++c) if (h.comp[c].id == s[1 + 2 * i]) which = c;
        if (which < 0) return kBadSosComponent;
        FrameComp& c = h.comp[which];
        scan.comp[i] = which; scan.td[i] = c.td = s[2 + 2 * i] >> 4; scan.ta[i] = c.ta = s[2 + 2 * i] & 15;
        if (c.td > 3 || c.ta > 3 || !h.have_q[c.tq]) return kMissingTable;
      }
      // spectral selection / successive approximation (stb_image.h:2665-2702)
      scan.ss = s[1 + 2 * ns]; scan.se = s[2 + 2 * ns]; scan.ah = s[3 + 2 * ns] >> 4; scan.al = s[3 + 2 * ns] & 15;
      const bool progressive = h.sof == 0xC2;
      if (progressive ? scan.ss > 63 || scan.se > 63 || scan.ss > scan.se || scan.ah > 13 || scan.al > 13 : scan.ss || scan.ah || scan.al) return kBadSos;
      if (!progressive) scan.se = 63;
      const bool need_dc = !progressive || scan.ss == 0, need_ac = !progressive || scan.ss != 0;
      for (int i = 0; i < ns; ++i) {
        const FrameComp& c = h.comp[scan.comp[i]];
        if ((need_dc && !h.dc[c.td].present) || (need_ac && !h.ac[c.ta].present)) return kMissingTable;
      }
      scan.data = pos + len;
      return kScan;
    }
    pos += len;
  }
}

}  // namespace scn_jpeg

namespace scn {

int jpeg_decode_rgb8(const uint8_t* d, size_t n, uint32_t want_w, uint32_t want_h, uint8_t* out);        // jpeg.cpp

// A decoded colour frame (RGB8) registered to the depth image: out[p] = rgb[lut[p]], black where lut[p] < 0, for n_px pixels.
inline void rgb8_through_lut(const uint8_t* rgb, const int32_t* lut, size_t n_px, uint8_t* out) {
  for (size_t p = 0; p < n_px; ++p) {
    const int32_t q = lut[p]; uint8_t* o = out + 3 * p;
    if (q >= 0) { o[0] = rgb[3 * (size_t)q]; o[1] = rgb[3 * (size_t)q + 1]; o[2] = rgb[3 * (size_t)q + 2]; } else o[0] = o[1] = o[2] = 0;
  }
}

}  // namespace scn
