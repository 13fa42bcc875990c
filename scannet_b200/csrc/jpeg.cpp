// Baseline JPEG -> RGB8 for `.sens` colour frames (TYPE_JPEG), host side.
//
// The reference decodes colour through stb_image v2.08 (vendored third-party code at
// /root/reference/SensReader/c++/src/sensorData/stb_image.h, called from sensorData.h:609-616 with
// 3 requested channels).  JPEG decoding is only defined up to IDCT / up-sampling / colour-conversion
// rounding, so to return the SAME BYTES this decoder restates stb's published numerics:
//   * integer "islow" IDCT, 12-bit constants, column pass keeps 2 extra bits (stb_image.h:1928-2027)
//   * chroma up-sampling: h2 / v2 = (3*near + far + 2) >> 2, h2v2 = (9,3,3,1)/16 with +8 (stb_image.h:2871-2925),
//     any other ratio nearest-neighbour (:3046-3056); row pairing by the ystep state machine (:3209-3225)
//   * YCbCr -> RGB in 20-bit fixed point with the masked Cb term (stb_image.h:3091-3118)
//   * coefficients truncated to int16 after de-quantisation (:1735,1764)
// Structure (marker parser, canonical Huffman decoder, plane layout) is this repo's own.
// Supported: SOF0/SOF1 and progressive SOF2 (spectral selection + successive approximation, stb_image.h:1771-1913, 2582-2600),
// 8-bit, 1 or 3 components, interleaved and non-interleaved scans, restart markers.
#include <algorithm>
#if defined(__x86_64__)
#include <immintrin.h>
#endif
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <vector>

#include "jpeg_common.h"
#include "scn_common.h"

namespace {

using namespace scn_jpeg;

// decoding state of one component: planes (and progressive coefficients) sized from the frame header
struct Comp { int dc_pred = 0, x = 0, y = 0, w2 = 0, h2 = 0, coeff_w = 0; std::vector<uint8_t> data; std::vector<short> coeff; };

struct Bits {
  const uint8_t* p; size_t n, pos; uint32_t buf = 0; int cnt = 0; bool hit_marker = false;
  void fill() {
    while (cnt <= 24) {
      uint32_t b = 0;
      if (!hit_marker && pos < n) {
        b = p[pos];
        if (b == 0xFF) {
          const uint8_t nx = pos + 1 < n ? p[pos + 1] : 0xD9;
          if (nx == 0) pos += 2; else { hit_marker = true; b = 0; }
        } else ++pos;
      }
      buf |= b << (24 - cnt); cnt += 8;
    }
  }
  int get(int k) { if (k == 0) return 0; if (cnt < k) fill(); const int v = (int)(buf >> (32 - k)); buf <<= k; cnt -= k; return v; }
  int decode(const HuffTab& h) {
    if (cnt < 16) fill();
    const uint16_t e = h.fast[buf >> (32 - kFastBits)];
    if (e != 0xFFFF) { const int l = e & 15; buf <<= l; cnt -= l; return e >> 4; }
    int code = 0;
    for (int l = 1; l <= 16; ++l) {
      code = (code << 1) | (int)(buf >> 31); buf <<= 1; --cnt;
      if (h.maxcode[l] >= 0 && code <= h.maxcode[l] && code >= h.mincode[l]) return h.vals[h.valptr[l] + code - h.mincode[l]];
    }
    return -1;
  }
  void reset() { buf = 0; cnt = 0; hit_marker = false; }
};

// AVX2 clones of the two hot loops, picked at load time.  (SCN_NO_TARGET_CLONES: ThreadSanitizer builds — the ifunc
// resolver would run before the sanitizer runtime is up.)
#ifdef SCN_NO_TARGET_CLONES
#define SCN_CLONES
#else
#define SCN_CLONES __attribute__((target_clones("avx2", "default")))
#endif
// The same arithmetic, eight columns (then eight rows) at a time in 32-bit lanes: every add, multiply (low 32 bits) and shift
// is the scalar one, so the bytes are identical.  The column shortcut for all-zero AC terms is not needed: with only s0 set the
// general formula gives (s0 << 12 + 512) >> 10 == s0 << 2 as well.
#if defined(__x86_64__)
#define VMUL(a, c) _mm256_mullo_epi32(a, _mm256_set1_epi32(F2F(c)))
#define VADD(a, b) _mm256_add_epi32(a, b)
#define VSUB(a, b) _mm256_sub_epi32(a, b)
#define IDCT_1D_V(s0, s1, s2, s3, s4, s5, s6, s7)                                                  \
  __m256i t0, t1, t2, t3, p1, p2, p3, p4, p5, x0, x1, x2, x3;                                      \
  p2 = s2; p3 = s6;                                                                                \
  p1 = VMUL(VADD(p2, p3), 0.5411961f);                                                             \
  t2 = VADD(p1, VMUL(p3, -1.847759065f));                                                          \
  t3 = VADD(p1, VMUL(p2, 0.765366865f));                                                           \
  p2 = s0; p3 = s4;                                                                                \
  t0 = _mm256_slli_epi32(VADD(p2, p3), 12); t1 = _mm256_slli_epi32(VSUB(p2, p3), 12);              \
  x0 = VADD(t0, t3); x3 = VSUB(t0, t3); x1 = VADD(t1, t2); x2 = VSUB(t1, t2);                      \
  t0 = s7; t1 = s5; t2 = s3; t3 = s1;                                                              \
  p3 = VADD(t0, t2); p4 = VADD(t1, t3); p1 = VADD(t0, t3); p2 = VADD(t1, t2);                      \
  p5 = VMUL(VADD(p3, p4), 1.175875602f);                                                           \
  t0 = VMUL(t0, 0.298631336f); t1 = VMUL(t1, 2.053119869f);                                        \
  t2 = VMUL(t2, 3.072711026f); t3 = VMUL(t3, 1.501321110f);                                        \
  p1 = VADD(p5, VMUL(p1, -0.899976223f)); p2 = VADD(p5, VMUL(p2, -2.562915447f));                  \
  p3 = VMUL(p3, -1.961570560f); p4 = VMUL(p4, -0.390180644f);                                      \
  t3 = VADD(t3, VADD(p1, p4)); t2 = VADD(t2, VADD(p2, p3)); t1 = VADD(t1, VADD(p2, p4)); t0 = VADD(t0, VADD(p1, p3));

__attribute__((target("avx2"))) static inline void transpose8(__m256i (&r)[8]) {
  const __m256i a0 = _mm256_unpacklo_epi32(r[0], r[1]), a1 = _mm256_unpackhi_epi32(r[0], r[1]), a2 = _mm256_unpacklo_epi32(r[2], r[3]),
                a3 = _mm256_unpackhi_epi32(r[2], r[3]), a4 = _mm256_unpacklo_epi32(r[4], r[5]), a5 = _mm256_unpackhi_epi32(r[4], r[5]),
                a6 = _mm256_unpacklo_epi32(r[6], r[7]), a7 = _mm256_unpackhi_epi32(r[6], r[7]);
  const __m256i b0 = _mm256_unpacklo_epi64(a0, a2), b1 = _mm256_unpackhi_epi64(a0, a2), b2 = _mm256_unpacklo_epi64(a1, a3),
                b3 = _mm256_unpackhi_epi64(a1, a3), b4 = _mm256_unpacklo_epi64(a4, a6), b5 = _mm256_unpackhi_epi64(a4, a6),
                b6 = _mm256_unpacklo_epi64(a5, a7), b7 = _mm256_unpackhi_epi64(a5, a7);
  r[0] = _mm256_permute2x128_si256(b0, b4, 0x20); r[1] = _mm256_permute2x128_si256(b1, b5, 0x20);
  r[2] = _mm256_permute2x128_si256(b2, b6, 0x20); r[3] = _mm256_permute2x128_si256(b3, b7, 0x20);
  r[4] = _mm256_permute2x128_si256(b0, b4, 0x31); r[5] = _mm256_permute2x128_si256(b1, b5, 0x31);
  r[6] = _mm256_permute2x128_si256(b2, b6, 0x31); r[7] = _mm256_permute2x128_si256(b3, b7, 0x31);
}

__attribute__((target("avx2"))) static void idct8x8_avx2(uint8_t* out, int stride, const short* d) {
  __m256i v[8];
  for (int k = 0; k < 8; ++k) v[k] = _mm256_cvtepi16_epi32(_mm_loadu_si128((const __m128i*)(d + 8 * k)));
  {                                                             // columns: lane = column, v[k] = row k
    IDCT_1D_V(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7])
    const __m256i r512 = _mm256_set1_epi32(512);
    x0 = VADD(x0, r512); x1 = VADD(x1, r512); x2 = VADD(x2, r512); x3 = VADD(x3, r512);
    v[0] = _mm256_srai_epi32(VADD(x0, t3), 10); v[7] = _mm256_srai_epi32(VSUB(x0, t3), 10);
    v[1] = _mm256_srai_epi32(VADD(x1, t2), 10); v[6] = _mm256_srai_epi32(VSUB(x1, t2), 10);
    v[2] = _mm256_srai_epi32(VADD(x2, t1), 10); v[5] = _mm256_srai_epi32(VSUB(x2, t1), 10);
    v[3] = _mm256_srai_epi32(VADD(x3, t0), 10); v[4] = _mm256_srai_epi32(VSUB(x3, t0), 10);
  }
  transpose8(v);                                                // now v[c] = column c of the intermediate, lane = row
  {
    IDCT_1D_V(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7])
    const __m256i bias = _mm256_set1_epi32(65536 + (128 << 17));
    x0 = VADD(x0, bias); x1 = VADD(x1, bias); x2 = VADD(x2, bias); x3 = VADD(x3, bias);
    v[0] = _mm256_srai_epi32(VADD(x0, t3), 17); v[7] = _mm256_srai_epi32(VSUB(x0, t3), 17);
    v[1] = _mm256_srai_epi32(VADD(x1, t2), 17); v[6] = _mm256_srai_epi32(VSUB(x1, t2), 17);
    v[2] = _mm256_srai_epi32(VADD(x2, t1), 17); v[5] = _mm256_srai_epi32(VSUB(x2, t1), 17);
    v[3] = _mm256_srai_epi32(VADD(x3, t0), 17); v[4] = _mm256_srai_epi32(VSUB(x3, t0), 17);
  }
  transpose8(v);                                                // v[r] = output row r, lane = column
  for (int r = 0; r < 8; r += 2) {                              // saturating packs == clamp8
    const __m256i w16 = _mm256_packs_epi32(v[r], v[r + 1]);     // per 128-bit half: r[0..3] r+1[0..3] | r[4..7] r+1[4..7]
    const __m256i w8 = _mm256_packus_epi16(w16, w16);           // per half: r[0..3] r+1[0..3] (twice) | r[4..7] r+1[4..7] (twice)
    const uint32_t a_lo = (uint32_t)_mm256_extract_epi32(w8, 0), b_lo = (uint32_t)_mm256_extract_epi32(w8, 1);
    const uint32_t a_hi = (uint32_t)_mm256_extract_epi32(w8, 4), b_hi = (uint32_t)_mm256_extract_epi32(w8, 5);
    uint8_t* o0 = out + (size_t)r * stride; uint8_t* o1 = o0 + stride;
    memcpy(o0, &a_lo, 4); memcpy(o0 + 4, &a_hi, 4); memcpy(o1, &b_lo, 4); memcpy(o1 + 4, &b_hi, 4);
  }
}
#endif

inline bool use_avx2() {
#if defined(__x86_64__)
  static const bool simd = __builtin_cpu_supports("avx2") && !getenv("SCN_JPEG_SCALAR");      // the env switch exists for the A/B parity test
  return simd;
#else
  return false;
#endif
}
void idct8x8_scalar(uint8_t* out, int stride, const short* d);
void idct8x8(uint8_t* out, int stride, const short* d) {
#if defined(__x86_64__)
  if (use_avx2()) { idct8x8_avx2(out, stride, d); return; }
#endif
  idct8x8_scalar(out, stride, d);
}

void idct8x8_scalar(uint8_t* out, int stride, const short* d) {
  int val[64];
  for (int i = 0; i < 8; ++i) {
    const short* c = d + i; int* v = val + i;
    if (c[8] == 0 && c[16] == 0 && c[24] == 0 && c[32] == 0 && c[40] == 0 && c[48] == 0 && c[56] == 0) {
      const int dc = c[0] << 2;
      v[0] = v[8] = v[16] = v[24] = v[32] = v[40] = v[48] = v[56] = dc;
    } else {
      IDCT_1D(c[0], c[8], c[16], c[24], c[32], c[40], c[48], c[56])
      x0 += 512; x1 += 512; x2 += 512; x3 += 512;
      v[0] = (x0 + t3) >> 10; v[56] = (x0 - t3) >> 10; v[8] = (x1 + t2) >> 10; v[48] = (x1 - t2) >> 10;
      v[16] = (x2 + t1) >> 10; v[40] = (x2 - t1) >> 10; v[24] = (x3 + t0) >> 10; v[32] = (x3 - t0) >> 10;
    }
  }
  for (int i = 0; i < 8; ++i) {
    const int* v = val + 8 * i; uint8_t* o = out + (size_t)i * stride;
    IDCT_1D(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7])
    const int bias = 65536 + (128 << 17);
    x0 += bias; x1 += bias; x2 += bias; x3 += bias;
    o[0] = clamp8((x0 + t3) >> 17); o[7] = clamp8((x0 - t3) >> 17); o[1] = clamp8((x1 + t2) >> 17); o[6] = clamp8((x1 - t2) >> 17);
    o[2] = clamp8((x2 + t1) >> 17); o[5] = clamp8((x2 - t1) >> 17); o[3] = clamp8((x3 + t0) >> 17); o[4] = clamp8((x3 - t0) >> 17);
  }
}

const uint8_t* up_h2(uint8_t* out, const uint8_t* in, int w) {
  if (w == 1) { out[0] = out[1] = in[0]; return out; }
  out[0] = in[0]; out[1] = (uint8_t)((in[0] * 3 + in[1] + 2) >> 2);
  int i;
  for (i = 1; i < w - 1; ++i) { const int n = 3 * in[i] + 2; out[i * 2] = (uint8_t)((n + in[i - 1]) >> 2); out[i * 2 + 1] = (uint8_t)((n + in[i + 1]) >> 2); }
  out[i * 2] = (uint8_t)((in[w - 2] * 3 + in[w - 1] + 2) >> 2); out[i * 2 + 1] = in[w - 1];
  return out;
}
const uint8_t* up_v2(uint8_t* out, const uint8_t* nr, const uint8_t* fr, int w) {
  for (int i = 0; i < w; ++i) out[i] = (uint8_t)((3 * nr[i] + fr[i] + 2) >> 2);
  return out;
}
#if defined(__x86_64__)
// out[2j] = (3 t[j] + t[j-1] + 8) >> 4, out[2j+1] = (3 t[j] + t[j+1] + 8) >> 4 with t = 3*near + far, for 16 values of j at a time
// in 16-bit lanes (t <= 1020, sums <= 4088); the pair (even, odd) of one j is one little-endian 16-bit lane of the output.
__attribute__((target("avx2"))) static int up_hv2_avx2(uint8_t* out, const uint8_t* nr, const uint8_t* fr, int w) {
  int j = 1;
  const __m256i three = _mm256_set1_epi16(3), eight = _mm256_set1_epi16(8);
#define SCN_TVEC(k) _mm256_add_epi16(_mm256_mullo_epi16(_mm256_cvtepu8_epi16(_mm_loadu_si128((const __m128i*)(nr + (k)))), three), \
                                     _mm256_cvtepu8_epi16(_mm_loadu_si128((const __m128i*)(fr + (k)))))
  for (; j + 17 <= w; j += 16) {                                  // needs t[j-1 .. j+16]
    const __m256i t = SCN_TVEC(j), tm = SCN_TVEC(j - 1), tp = SCN_TVEC(j + 1);
    const __m256i t3 = _mm256_add_epi16(_mm256_mullo_epi16(t, three), eight);
    const __m256i ev = _mm256_srli_epi16(_mm256_add_epi16(t3, tm), 4), od = _mm256_srli_epi16(_mm256_add_epi16(t3, tp), 4);
    _mm256_storeu_si256((__m256i*)(out + 2 * j), _mm256_or_si256(ev, _mm256_slli_epi16(od, 8)));
  }
#undef SCN_TVEC
  return j;                                                       // first j not done
}
#endif
const uint8_t* up_hv2(uint8_t* out, const uint8_t* nr, const uint8_t* fr, int w) {
  if (w == 1) { out[0] = out[1] = (uint8_t)((3 * nr[0] + fr[0] + 2) >> 2); return out; }
  int t1 = 3 * nr[0] + fr[0], t0;
  out[0] = (uint8_t)((t1 + 2) >> 2);
  int i = 1;
#if defined(__x86_64__)
  if (use_avx2() && w >= 18) {
    out[1] = (uint8_t)((3 * t1 + (3 * nr[1] + fr[1]) + 8) >> 4);   // out[2*0+1], the odd sample of j = 0
    i = up_hv2_avx2(out, nr, fr, w);                              // wrote out[2 .. 2i-1]
    t1 = 3 * nr[i - 1] + fr[i - 1];
  }
#endif
  for (; i < w; ++i) { t0 = t1; t1 = 3 * nr[i] + fr[i]; out[i * 2 - 1] = (uint8_t)((3 * t0 + t1 + 8) >> 4); out[i * 2] = (uint8_t)((3 * t1 + t0 + 8) >> 4); }
  out[w * 2 - 1] = (uint8_t)((t1 + 2) >> 2);
  return out;
}
const uint8_t* up_generic(uint8_t* out, const uint8_t* in, int w, int hs) {
  for (int i = 0; i < w; ++i) for (int j = 0; j < hs; ++j) out[i * hs + j] = in[i];
  return out;
}

#if defined(__x86_64__)
// eight pixels per step in 32-bit lanes, the same fixed-point arithmetic; saturating packs == clamp8; a byte shuffle interleaves
__attribute__((target("avx2"))) static int ycc_row_to_rgb_avx2(uint8_t* o, const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int W) {
  const __m256i c128 = _mm256_set1_epi32(128), half = _mm256_set1_epi32(1 << 19), mask = _mm256_set1_epi32((int)0xffff0000);
  const __m256i k_r = _mm256_set1_epi32(FIX20(1.40200f)), k_g1 = _mm256_set1_epi32(-FIX20(0.71414f)), k_g2 = _mm256_set1_epi32(-FIX20(0.34414f)),
                k_b = _mm256_set1_epi32(FIX20(1.77200f));
  const __m256i shuf = _mm256_setr_epi8(0, 4, 8, 1, 5, 9, 2, 6, 10, 3, 7, 11, -1, -1, -1, -1, 0, 4, 8, 1, 5, 9, 2, 6, 10, 3, 7, 11, -1, -1, -1, -1);
  int i = 0;
  for (; i + 10 <= W; i += 8) {                                   // the two 16-byte stores cover 28 bytes from 3*i: stay inside the row
    const __m256i yy = _mm256_cvtepu8_epi32(_mm_loadl_epi64((const __m128i*)(y + i)));
    const __m256i b_ = _mm256_sub_epi32(_mm256_cvtepu8_epi32(_mm_loadl_epi64((const __m128i*)(cb + i))), c128);
    const __m256i r_ = _mm256_sub_epi32(_mm256_cvtepu8_epi32(_mm_loadl_epi64((const __m128i*)(cr + i))), c128);
    const __m256i yf = _mm256_add_epi32(_mm256_slli_epi32(yy, 20), half);
    const __m256i r = _mm256_srai_epi32(_mm256_add_epi32(yf, _mm256_mullo_epi32(r_, k_r)), 20);
    const __m256i g = _mm256_srai_epi32(_mm256_add_epi32(_mm256_add_epi32(yf, _mm256_mullo_epi32(r_, k_g1)), _mm256_and_si256(_mm256_mullo_epi32(b_, k_g2), mask)), 20);
    const __m256i b = _mm256_srai_epi32(_mm256_add_epi32(yf, _mm256_mullo_epi32(b_, k_b)), 20);
    const __m256i rg = _mm256_packs_epi32(r, g), bb = _mm256_packs_epi32(b, b);         // per half: r0-3 g0-3 | b0-3 b0-3
    const __m256i px = _mm256_shuffle_epi8(_mm256_packus_epi16(rg, bb), shuf);            // per half: r0 g0 b0 r1 g1 b1 ... b3 x x x x
    _mm_storeu_si128((__m128i*)(o + 3 * i), _mm256_castsi256_si128(px));
    _mm_storeu_si128((__m128i*)(o + 3 * i + 12), _mm256_extracti128_si256(px, 1));
  }
  return i;
}
#endif
void ycc_row_to_rgb(uint8_t* o, const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int W) {
  int i = 0;
#if defined(__x86_64__)
  if (use_avx2()) i = ycc_row_to_rgb_avx2(o, y, cb, cr, W);
#endif
  for (; i < W; ++i) { const unsigned c = ycc_to_rgb(y[i], cb[i], cr[i]); o[3 * i] = (uint8_t)c; o[3 * i + 1] = (uint8_t)(c >> 8); o[3 * i + 2] = (uint8_t)(c >> 16); }
}

}  // namespace

namespace scn {

// error code and text of each refusal of the marker parser, in the order of scn_jpeg::Parse from kTruncated on
static const struct { int code; const char* text; } kRefusal[] = {
    {SCN_ERR_FORMAT, "truncated JPEG"}, {SCN_ERR_FORMAT, "bad JPEG segment length"},
    {SCN_ERR_UNSUPPORTED, "16-bit quantisation tables are not supported (as in stb_image)"}, {SCN_ERR_FORMAT, "bad DQT"},
    {SCN_ERR_FORMAT, "bad DHT"}, {SCN_ERR_FORMAT, "bad code lengths"}, {SCN_ERR_FORMAT, "bad DRI"}, {SCN_ERR_UNSUPPORTED, "only 8-bit JPEG"},
    {SCN_ERR_FORMAT, "bad SOF"}, {SCN_ERR_FORMAT, nullptr /* kBadSize: formatted below */}, {SCN_ERR_FORMAT, "bad SOF component"},
    {SCN_ERR_FORMAT, "SOS before SOF"}, {SCN_ERR_FORMAT, "bad SOS"}, {SCN_ERR_FORMAT, "bad SOS component"},
    {SCN_ERR_FORMAT, "scan references a missing table"}};
static_assert(sizeof(kRefusal) / sizeof(kRefusal[0]) == kMissingTable - kTruncated + 1, "one entry per refusal");

int jpeg_decode_rgb8(const uint8_t* d, size_t n, uint32_t want_w, uint32_t want_h, uint8_t* out) {
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return fail(SCN_ERR_FORMAT, "not a JPEG (no SOI)");
  Header hd(want_w, want_h);
  Comp comp[3];
  // plane buffers are leased from the calling thread and handed back on every exit path: a decoder pool of 64 threads doing
  // a 460 KB allocation + page faults per frame serialised on the process's memory map (31 ms per 128-frame chunk instead of 7)
  static thread_local std::vector<uint8_t> tl_planes[3];
  struct PlaneLease {
    Comp* c; std::vector<uint8_t>* t; int n;
    PlaneLease(Comp* c_, std::vector<uint8_t>* t_, int n_) : c(c_), t(t_), n(n_) { for (int i = 0; i < n; ++i) c[i].data.swap(t[i]); }
    ~PlaneLease() { for (int i = 0; i < n; ++i) c[i].data.swap(t[i]); }
  } lease(comp, tl_planes, 3);
  int mcux = 0, mcuy = 0, sized_for = 0;             // sized_for: the frame header (by count) the planes were last sized for
  Scan sc;
  for (size_t pos = 2;;) {
    const Parse pr = parse_header(d, n, pos, hd, sc);
    if (pr == kBadSize) return fail(SCN_ERR_FORMAT, "JPEG is %dx%d, header says %ux%u", hd.W, hd.H, want_w, want_h);
    if (pr != kScan && pr != kEnd) return fail(kRefusal[pr - kTruncated].code, "%s", kRefusal[pr - kTruncated].text);
    const int ncomp = hd.ncomp, W = hd.W, H = hd.H, hmax = hd.hmax, vmax = hd.vmax;
    const bool progressive = hd.sof == 0xC2;
    if (hd.n_sof != sized_for) {                       // a new frame header: (re)size and clear the planes
      sized_for = hd.n_sof;
      mcux = (W + 8 * hmax - 1) / (8 * hmax); mcuy = (H + 8 * vmax - 1) / (8 * vmax);
      for (int i = 0; i < ncomp; ++i) {
        const FrameComp& f = hd.comp[i];
        comp[i].x = (W * f.h + hmax - 1) / hmax; comp[i].y = (H * f.v + vmax - 1) / vmax;
        comp[i].w2 = mcux * f.h * 8; comp[i].h2 = mcuy * f.v * 8;
        comp[i].data.assign((size_t)comp[i].w2 * comp[i].h2 + 15, 0);
        if (progressive) { comp[i].coeff_w = comp[i].w2 >> 3; comp[i].coeff.assign((size_t)comp[i].coeff_w * (comp[i].h2 >> 3) * 64, 0); }
      }
    }
    if (pr == kEnd) break;
    const int ns = sc.ns, spec_start = sc.ss, spec_end = sc.se, succ_high = sc.ah, succ_low = sc.al, restart = hd.restart;
    const int* order = sc.comp;
    Bits br{d, n, sc.data};
    for (int c = 0; c < ncomp; ++c) comp[c].dc_pred = 0;
    int todo = restart ? restart : 0x7fffffff;
    short blk[64];
    auto decode_block = [&](int kc, int bx, int by) -> bool {
      Comp& c = comp[kc]; const FrameComp& f = hd.comp[kc];
      memset(blk, 0, sizeof(blk));
      const int t = br.decode(hd.dc[f.td]);
      if (t < 0 || t > 16) return false;
      const int diff = t ? extend(br.get(t), t) : 0;
      c.dc_pred += diff;
      const uint8_t* q = hd.quant[f.tq];
      blk[0] = (short)(c.dc_pred * q[0]);
      const HuffTab& ha = hd.ac[f.ta];
      for (int k = 1; k < 64;) {
        if (br.cnt < 16) br.fill();
        const int fa = ha.fast_ac[br.buf >> (32 - kFastBits)];
        if (fa) {                                             // short code + small coefficient in one lookup
          k += (fa >> 4) & 15;
          const int used = fa & 15;
          br.buf <<= used; br.cnt -= used;
          const int z = kZig[k++];
          blk[z] = (short)((fa >> 8) * q[z]);
          continue;
        }
        const int rs = br.decode(ha);
        if (rs < 0) return false;
        const int sz = rs & 15, r = rs >> 4;
        if (sz == 0) { if (rs != 0xF0) break; k += 16; }
        else { k += r; const int z = kZig[k++]; blk[z] = (short)(extend(br.get(sz), sz) * q[z]); }
      }
      idct8x8(c.data.data() + (size_t)c.w2 * by * 8 + (size_t)bx * 8, c.w2, blk);
      return true;
    };
    int eob_run = 0;
    // progressive passes write into the persistent coefficient blocks (stb_image.h:1771-1913); same arithmetic, in shorts
    auto prog_dc = [&](int kc, short* data) -> bool {
      if (spec_end != 0) return false;                                     // "can't merge dc and ac"
      if (succ_high == 0) {
        memset(data, 0, 64 * sizeof(short));
        const int t = br.decode(hd.dc[hd.comp[kc].td]);
        if (t < 0 || t > 16) return false;
        const int diff = t ? extend(br.get(t), t) : 0;
        comp[kc].dc_pred += diff;
        data[0] = (short)(comp[kc].dc_pred << succ_low);
      } else if (br.get(1)) data[0] += (short)(1 << succ_low);
      return true;
    };
    auto prog_ac = [&](int kc, short* data) -> bool {
      if (spec_start == 0) return false;
      const HuffTab& ha = hd.ac[hd.comp[kc].ta];
      if (succ_high == 0) {
        const int shift = succ_low;
        if (eob_run) { --eob_run; return true; }
        int k = spec_start;
        do {
          if (br.cnt < 16) br.fill();
          const int fa = ha.fast_ac[br.buf >> (32 - kFastBits)];
          if (fa) {
            k += (fa >> 4) & 15;
            const int used = fa & 15;
            br.buf <<= used; br.cnt -= used;
            data[kZig[k++]] = (short)((fa >> 8) << shift);
          } else {
            const int rs = br.decode(ha);
            if (rs < 0) return false;
            const int sz = rs & 15, r = rs >> 4;
            if (sz == 0) {
              if (r < 15) { eob_run = 1 << r; if (r) eob_run += br.get(r); --eob_run; break; }
              k += 16;
            } else { k += r; data[kZig[k++]] = (short)(extend(br.get(sz), sz) << shift); }
          }
        } while (k <= spec_end);
      } else {
        const short bit = (short)(1 << succ_low);
        auto refine = [&](short* p) { if (br.get(1) && (*p & bit) == 0) { if (*p > 0) *p += bit; else *p -= bit; } };
        if (eob_run) {
          --eob_run;
          for (int k = spec_start; k <= spec_end; ++k) { short* p = &data[kZig[k]]; if (*p != 0) refine(p); }
        } else {
          int k = spec_start;
          do {
            const int rs = br.decode(ha);
            if (rs < 0) return false;
            int sz = rs & 15, r = rs >> 4;
            if (sz == 0) {
              if (r < 15) { eob_run = (1 << r) - 1; if (r) eob_run += br.get(r); r = 64; }
            } else {
              if (sz != 1) return false;
              sz = br.get(1) ? bit : -bit;
            }
            while (k <= spec_end) {
              short* p = &data[kZig[k++]];
              if (*p != 0) refine(p);
              else { if (r == 0) { *p = (short)sz; break; } --r; }
            }
          } while (k <= spec_end);
        }
      }
      return true;
    };
    auto handle_restart = [&]() {
      if (--todo <= 0) {
        eob_run = 0;
        // byte-align, expect RSTn
        br.reset();
        size_t q = br.pos;
        while (q + 1 < n && !(d[q] == 0xFF && d[q + 1] >= 0xD0 && d[q + 1] <= 0xD7)) { if (d[q] == 0xFF && d[q + 1] != 0 && d[q + 1] != 0xFF) return false; ++q; }
        if (q + 1 >= n) return false;
        br.pos = q + 2;
        for (int c = 0; c < ncomp; ++c) comp[c].dc_pred = 0;
        todo = restart ? restart : 0x7fffffff;
      }
      return true;
    };
    bool ended = false;
    auto one_block = [&](int kc, int bx, int by) -> bool {
      if (!progressive) return decode_block(kc, bx, by);
      short* data = comp[kc].coeff.data() + 64 * ((size_t)bx + (size_t)by * comp[kc].coeff_w);
      return (ns > 1 || spec_start == 0) ? prog_dc(kc, data) : prog_ac(kc, data);        // interleaved progressive scans are DC scans
    };
    if (ns == 1) {
      const Comp& c = comp[order[0]];
      const int bw = (c.x + 7) >> 3, bh = (c.y + 7) >> 3;
      for (int j = 0; j < bh && !ended; ++j) for (int i = 0; i < bw; ++i) {
        if (!one_block(order[0], i, j)) return fail(SCN_ERR_FORMAT, "bad huffman code");
        if (!handle_restart()) { ended = true; break; }
      }
    } else {
      for (int j = 0; j < mcuy && !ended; ++j) for (int i = 0; i < mcux; ++i) {
        for (int k = 0; k < ns; ++k) { const FrameComp& f = hd.comp[order[k]];
          for (int y = 0; y < f.v; ++y) for (int x = 0; x < f.h; ++x)
            if (!one_block(order[k], i * f.h + x, j * f.v + y)) return fail(SCN_ERR_FORMAT, "bad huffman code"); }
        if (!handle_restart()) { ended = true; break; }
      }
    }
    // continue the marker scan after the entropy-coded data
    pos = br.pos;
    while (pos + 1 < n && !(d[pos] == 0xFF && d[pos + 1] != 0 && !(d[pos + 1] >= 0xD0 && d[pos + 1] <= 0xD7) && d[pos + 1] != 0xFF)) ++pos;
  }
  if (!hd.sof) return fail(SCN_ERR_FORMAT, "no frame in JPEG");
  const int ncomp = hd.ncomp, W = hd.W, H = hd.H, hmax = hd.hmax, vmax = hd.vmax;
  if (hd.sof == 0xC2) {                                                       // stbi__jpeg_finish: dequantise (in shorts) + IDCT of every real block
    for (int k = 0; k < ncomp; ++k) {
      Comp& c = comp[k];
      if (!hd.have_q[hd.comp[k].tq]) return fail(SCN_ERR_FORMAT, "scan references a missing table");
      const uint8_t* q = hd.quant[hd.comp[k].tq];
      const int bw = (c.x + 7) >> 3, bh = (c.y + 7) >> 3;
      for (int j = 0; j < bh; ++j) for (int i = 0; i < bw; ++i) {
        short* data = c.coeff.data() + 64 * ((size_t)i + (size_t)j * c.coeff_w);
        for (int z = 0; z < 64; ++z) data[z] = (short)(data[z] * q[z]);
        idct8x8(c.data.data() + (size_t)c.w2 * j * 8 + (size_t)i * 8, c.w2, data);
      }
    }
  }
  // up-sample + colour convert, row by row (stb_image.h:3166-3250)
  struct Res { int hs, vs, ystep, wl, ypos; const uint8_t *l0, *l1; std::vector<uint8_t> buf; } rs[3];
  for (int k = 0; k < ncomp; ++k) {
    rs[k].hs = hmax / hd.comp[k].h; rs[k].vs = vmax / hd.comp[k].v; rs[k].ystep = rs[k].vs >> 1;
    rs[k].wl = (W + rs[k].hs - 1) / rs[k].hs; rs[k].ypos = 0; rs[k].l0 = rs[k].l1 = comp[k].data.data();
    rs[k].buf.assign((size_t)W + 16 + 8 * hmax, 0);
  }
  for (int j = 0; j < H; ++j) {
    const uint8_t* row[3];
    for (int k = 0; k < ncomp; ++k) {
      Res& r = rs[k];
      const bool bot = r.ystep >= (r.vs >> 1);
      const uint8_t* nr = bot ? r.l1 : r.l0; const uint8_t* fr = bot ? r.l0 : r.l1;
      if (r.hs == 1 && r.vs == 1) row[k] = nr;
      else if (r.hs == 1 && r.vs == 2) row[k] = up_v2(r.buf.data(), nr, fr, r.wl);
      else if (r.hs == 2 && r.vs == 1) row[k] = up_h2(r.buf.data(), nr, r.wl);
      else if (r.hs == 2 && r.vs == 2) row[k] = up_hv2(r.buf.data(), nr, fr, r.wl);
      else row[k] = up_generic(r.buf.data(), nr, r.wl, r.hs);
      if (++r.ystep >= r.vs) { r.ystep = 0; r.l0 = r.l1; if (++r.ypos < comp[k].y) r.l1 += comp[k].w2; }
    }
    uint8_t* o = out + (size_t)j * W * 3;
    if (ncomp == 3) ycc_row_to_rgb(o, row[0], row[1], row[2], W);
    else for (int i = 0; i < W; ++i) o[3 * i] = o[3 * i + 1] = o[3 * i + 2] = row[0][i];
  }
  return SCN_OK;
}

int zlib_inflate(const uint8_t* src, size_t n, std::vector<uint8_t>& out, size_t size_hint);   // sens.cpp

// PNG colour frames (TYPE_PNG, sensorData.h:346-351; decoded by stbi_load_from_memory with 3 requested channels,
// :609-616).  PNG is lossless, so any conforming decoder returns the reference's bytes; conversions to RGB follow
// stb_image v2.08 (grey replicated, alpha dropped, palette expanded; 16-bit PNGs are rejected there and here).
// Adam7-interlaced images are scattered pass by pass (stb_image.h:4310-4350).  At 1/2/4-bit depth stb v2.08 takes the
// "previous row" of the up/avg/paeth filters from uninitialised memory (:4003-4012); this decoder follows the PNG specification.
int png_decode_rgb8(const uint8_t* d, size_t n, uint32_t want_w, uint32_t want_h, uint8_t* out) {
  static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
  if (n < 8 || memcmp(d, sig, 8)) return fail(SCN_ERR_FORMAT, "not a PNG");
  auto be32 = [&](size_t o) { return ((uint32_t)d[o] << 24) | ((uint32_t)d[o + 1] << 16) | ((uint32_t)d[o + 2] << 8) | d[o + 3]; };
  uint32_t W = 0, H = 0; int depth = 0, ctype = 0, interlace = 0;
  std::vector<uint8_t> idat, pal;
  size_t pos = 8; bool have_hdr = false, done = false;
  while (!done && pos + 12 <= n) {
    const uint32_t len = be32(pos); const uint8_t* type = d + pos + 4;
    if (pos + 12 + (size_t)len > n) return fail(SCN_ERR_FORMAT, "truncated PNG chunk");
    const uint8_t* body = d + pos + 8;
    if (!memcmp(type, "IHDR", 4)) {
      if (len < 13) return fail(SCN_ERR_FORMAT, "bad IHDR");
      W = be32(pos + 8); H = be32(pos + 12); depth = body[8]; ctype = body[9]; interlace = body[12]; have_hdr = true;
    } else if (!memcmp(type, "PLTE", 4)) pal.assign(body, body + len);
    else if (!memcmp(type, "IDAT", 4)) idat.insert(idat.end(), body, body + len);
    else if (!memcmp(type, "IEND", 4)) done = true;
    pos += 12 + (size_t)len;
  }
  if (!have_hdr || idat.empty()) return fail(SCN_ERR_FORMAT, "PNG without IHDR/IDAT");
  if (W != want_w || H != want_h) return fail(SCN_ERR_FORMAT, "PNG is %ux%u, header says %ux%u", W, H, want_w, want_h);
  if (interlace > 1) return fail(SCN_ERR_FORMAT, "bad PNG interlace method");
  if (depth == 16) return fail(SCN_ERR_UNSUPPORTED, "PNG not supported: 1/2/4/8-bit only");          // as stb_image v2.08
  if (!(depth == 8 || ((ctype == 0 || ctype == 3) && (depth == 1 || depth == 2 || depth == 4)))) return fail(SCN_ERR_FORMAT, "bad PNG bit depth");
  const int ch = ctype == 0 ? 1 : ctype == 2 ? 3 : ctype == 3 ? 1 : ctype == 4 ? 2 : ctype == 6 ? 4 : 0;
  if (!ch) return fail(SCN_ERR_FORMAT, "bad PNG colour type");
  const size_t bpp = std::max<size_t>(1, (size_t)ch * depth / 8);
  auto pass_bytes = [&](uint32_t pw, uint32_t ph) { return pw && ph ? ((((size_t)pw * ch * depth + 7) >> 3) + 1) * ph : (size_t)0; };
  // Adam7 (stb_image.h:4310-4350): seven sub-images, each filtered like a small PNG, scattered on an 8x8 lattice
  static const uint32_t xorig[7] = {0, 4, 0, 2, 0, 1, 0}, yorig[7] = {0, 0, 4, 0, 2, 0, 1}, xspc[7] = {8, 8, 4, 4, 2, 2, 1}, yspc[7] = {8, 8, 8, 4, 4, 2, 2};
  size_t need = 0;
  if (interlace) { for (int p = 0; p < 7; ++p) need += pass_bytes((W - xorig[p] + xspc[p] - 1) / xspc[p], (H - yorig[p] + yspc[p] - 1) / yspc[p]); }
  else need = pass_bytes(W, H);
  std::vector<uint8_t> raw;
  if (zlib_inflate(idat.data(), idat.size(), raw, need) || raw.size() < need) return fail(SCN_ERR_FORMAT, "corrupt PNG data");
  // one (sub-)image: undo the row filters, expand to RGB8, write pixel (x, y) to (x0 + x*dx, y0 + y*dy)
  auto run_pass = [&](const uint8_t* src, uint32_t pw, uint32_t ph, uint32_t x0, uint32_t y0, uint32_t dx, uint32_t dy) -> int {
    const size_t stride = ((size_t)pw * ch * depth + 7) / 8;
    std::vector<uint8_t> prev(stride, 0), cur(stride);
    for (uint32_t y = 0; y < ph; ++y) {
      const uint8_t* line = src + (size_t)y * (stride + 1); const int ft = line[0];
      for (size_t i = 0; i < stride; ++i) {
        const int a = i >= bpp ? cur[i - bpp] : 0, b = prev[i], c = i >= bpp ? prev[i - bpp] : 0;
        int pr;
        switch (ft) {
          case 0: pr = 0; break; case 1: pr = a; break; case 2: pr = b; break; case 3: pr = (a + b) >> 1; break;
          case 4: { const int pp = a + b - c, pa = abs(pp - a), pb = abs(pp - b), pc = abs(pp - c); pr = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); } break;
          default: return fail(SCN_ERR_FORMAT, "bad PNG filter");
        }
        cur[i] = (uint8_t)(line[1 + i] + pr);
      }
      uint8_t* orow = out + (size_t)(y0 + y * dy) * W * 3;
      for (uint32_t x = 0; x < pw; ++x) {
        auto sample = [&](int k) -> int {                       // k-th channel of pixel x as an 8-bit value
          if (depth == 8) return cur[(size_t)x * ch + k];
          const size_t bit = (size_t)x * depth; const int v = (cur[bit >> 3] >> (8 - depth - (bit & 7))) & ((1 << depth) - 1);
          return ctype == 3 ? v : v * (255 / ((1 << depth) - 1));
        };
        uint8_t* o = orow + (size_t)(x0 + x * dx) * 3;
        if (ctype == 3) { const int idx = sample(0); for (int k = 0; k < 3; ++k) o[k] = (size_t)(3 * idx + k) < pal.size() ? pal[3 * idx + k] : 0; }
        else if (ch <= 2) { const uint8_t g = (uint8_t)sample(0); o[0] = o[1] = o[2] = g; }
        else for (int k = 0; k < 3; ++k) o[k] = (uint8_t)sample(k);
      }
      prev.swap(cur);
    }
    return SCN_OK;
  };
  if (!interlace) return run_pass(raw.data(), W, H, 0, 0, 1, 1);
  size_t off = 0;
  for (int p = 0; p < 7; ++p) {
    const uint32_t pw = (W - xorig[p] + xspc[p] - 1) / xspc[p], ph = (H - yorig[p] + yspc[p] - 1) / yspc[p];
    if (!pw || !ph) continue;
    if (int rc = run_pass(raw.data() + off, pw, ph, xorig[p], yorig[p], xspc[p], yspc[p])) return rc;
    off += pass_bytes(pw, ph);
  }
  return SCN_OK;
}

}  // namespace scn
