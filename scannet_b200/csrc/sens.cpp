// SensReader: the `.sens` v4 RGB-D container (host side, C++), mirroring ml::SensorData
// (/root/reference/SensReader/c++/src/sensorData.h:285-1936) behind the C ABI.
//
//   file layout            sensorData.h:1058-1074 (header), :733-754 (RGBDFrame), :786-833 (IMUFrame)
//   depth decode           :693-730  TYPE_RAW_USHORT / TYPE_ZLIB_USHORT (the reference inflates with
//                          stb's zlib decoder; any conforming inflate yields the same bytes — ours is below)
//   colour decode          :600-646  TYPE_RAW / JPEG / PNG (see jpeg.cpp)
//   writer                 :888-929 initDefault/addFrame, :648-691 compressDepth, :1101-1109 saveToFile
//   saveToImages / PGM     :1342-1466, savePoseFile :1706-1714, operator<< :1941-1955
// Errors never cross the boundary as exceptions: every entry point returns a status.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <limits>
#include <sstream>
#include <string>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#include "jpeg_common.h"
#include "scn_common.h"

namespace scn {
int png_decode_rgb8(const uint8_t* data, size_t n, uint32_t want_w, uint32_t want_h, uint8_t* out);    // jpeg.cpp
int zlib_inflate(const uint8_t* src, size_t n, std::vector<uint8_t>& out, size_t size_hint);
void zlib_deflate(const uint8_t* src, size_t n, std::vector<uint8_t>& out);
void png_encode_stb(const uint8_t* px, uint32_t w, uint32_t h, int n, std::vector<uint8_t>& out);
}  // namespace scn

// ------------------------------------------------------------------------------ inflate (RFC 1950/1951)
// Table-driven decoder: 64-bit bit reservoir, 10-bit first-level lookup per Huffman code (longer codes walk the
// canonical ranges), literals/matches written straight into a pre-sized output buffer.
namespace {

const uint16_t kLenBase[29] = {3,4,5,6,7,8,9,10,11,13,15,17,19,23,27,31,35,43,51,59,67,83,99,115,131,163,195,227,258};
const uint8_t kLenExtra[29] = {0,0,0,0,0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,4,4,4,4,5,5,5,5,0};
const uint16_t kDistBase[30] = {1,2,3,4,5,7,9,13,17,25,33,49,65,97,129,193,257,385,513,769,1025,1537,2049,3073,4097,6145,8193,12289,16385,24577};
const uint8_t kDistExtra[30] = {0,0,0,0,1,1,2,2,3,3,4,4,5,5,6,6,7,7,8,8,9,9,10,10,11,11,12,12,13,13};

#define LP(b, e) ((uint32_t)(b) | ((uint32_t)(e) << 16))
const uint32_t kLenPacked[29] = {LP(3,0),LP(4,0),LP(5,0),LP(6,0),LP(7,0),LP(8,0),LP(9,0),LP(10,0),LP(11,1),LP(13,1),LP(15,1),LP(17,1),LP(19,2),LP(23,2),LP(27,2),LP(31,2),
                                 LP(35,3),LP(43,3),LP(51,3),LP(59,3),LP(67,4),LP(83,4),LP(99,4),LP(115,4),LP(131,5),LP(163,5),LP(195,5),LP(227,5),LP(258,0)};
const uint32_t kDistPacked[30] = {LP(1,0),LP(2,0),LP(3,0),LP(4,0),LP(5,1),LP(7,1),LP(9,2),LP(13,2),LP(17,3),LP(25,3),LP(33,4),LP(49,4),LP(65,5),LP(97,5),LP(129,6),LP(193,6),
                                  LP(257,7),LP(385,7),LP(513,8),LP(769,8),LP(1025,9),LP(1537,9),LP(2049,10),LP(3073,10),LP(4097,11),LP(6145,11),LP(8193,12),LP(12289,12),
                                  LP(16385,13),LP(24577,13)};
#undef LP

struct BitIn {
  const uint8_t* p; const uint8_t* end; uint64_t buf = 0; int cnt = 0; int pad = 0; bool bad = false;
  BitIn(const uint8_t* d, size_t n) : p(d), end(d + n) {}
  // past the end zero bytes are fed (the look-ahead may legitimately run a few bytes over); a stream that actually
  // consumes them is truncated: `bad` is raised once more than one reservoir of padding has been supplied
  inline void fill() {
    if (end - p >= 8) {                                       // one unaligned 8-byte load tops the reservoir up to 56..63 bits
      uint64_t v; memcpy(&v, p, 8);
      buf |= v << cnt; p += (63 - cnt) >> 3; cnt |= 56;
      return;
    }
    while (cnt <= 56) { if (p < end) buf |= (uint64_t)(*p++) << cnt; else if (++pad > 16) bad = true; cnt += 8; }
  }
  inline uint32_t peek(int k) { if (cnt < k) fill(); return (uint32_t)(buf & ((1ull << k) - 1)); }
  inline void drop(int k) { buf >>= k; cnt -= k; }
  inline uint32_t bits(int k) { if (k == 0) return 0; const uint32_t v = peek(k); drop(k); return v; }
  inline size_t overrun() const { return cnt < 0 ? 1 : 0; }
};

constexpr int kFast = 10;
struct Huff {
  uint16_t fast[1 << kFast];            // (symbol << 4) | length, 0 = not in table
  uint16_t count[16]; uint16_t symbol[288]; int first_code[16], first_sym[16]; int max_len = 0;
  static inline uint32_t rev(uint32_t c, int n) { uint32_t r = 0; for (int i = 0; i < n; ++i) { r = (r << 1) | (c & 1); c >>= 1; } return r; }
  bool build(const uint8_t* len, int n) {
    memset(count, 0, sizeof(count)); memset(fast, 0, sizeof(fast)); max_len = 0;
    for (int i = 0; i < n; ++i) count[len[i]]++;
    count[0] = 0;
    int code = 0, k = 0; uint16_t offs[16]; int next_code[16];
    for (int l = 1; l < 16; ++l) {
      first_code[l] = code; first_sym[l] = k; offs[l] = (uint16_t)k; next_code[l] = code;
      if (count[l] > (1 << l)) return false;
      code = (code + count[l]) << 1; k += count[l];
      if (count[l]) max_len = l;
    }
    for (int i = 0; i < n; ++i) if (len[i]) {
      const int l = len[i];
      symbol[offs[l]++] = (uint16_t)i;
      const int c = next_code[l]++;
      if (l <= kFast) {                                        // deflate codes are packed LSB first: index by the reversed code
        const uint32_t r = rev((uint32_t)c, l);
        for (uint32_t j = r; j < (1u << kFast); j += (1u << l)) fast[j] = (uint16_t)((i << 4) | l);
      }
    }
    return true;
  }
  inline int decode(BitIn& br) const {
    const uint32_t look = br.peek(15);
    const uint16_t e = fast[look & ((1u << kFast) - 1)];
    if (e) { br.drop(e & 15); return e >> 4; }
    int code = 0;
    for (int l = 1; l <= max_len; ++l) {
      code = (code << 1) | (int)((look >> (l - 1)) & 1);
      const int idx = code - first_code[l];
      if (idx >= 0 && idx < count[l]) { br.drop(l); return symbol[first_sym[l] + idx]; }
    }
    return -1;
  }
};

}  // namespace

int scn::zlib_inflate(const uint8_t* src, size_t n, std::vector<uint8_t>& out, size_t size_hint) {
  out.clear();
  if (n < 6) return -1;
  if ((src[0] & 0x0F) != 8 || ((src[0] << 8) | src[1]) % 31 != 0 || (src[1] & 0x20)) return -1;
  BitIn br(src + 2, n - 2);
  out.resize((size_hint ? size_hint : std::max<size_t>(n * 4, 1 << 16)) + 320);
  size_t op = 0;
  auto ensure = [&](size_t extra) { if (op + extra > out.size()) out.resize(std::max(out.size() * 2, op + extra)); };
  static thread_local Huff lit, dist;
  for (;;) {
    const uint32_t final = br.bits(1), type = br.bits(2);
    if (type == 0) {
      br.drop(br.cnt & 7);                                  // to the byte boundary
      const uint32_t len = br.bits(16), nlen = br.bits(16);
      if ((len ^ 0xFFFF) != nlen) return -1;
      ensure(len);
      for (uint32_t i = 0; i < len; ++i) { out[op++] = (uint8_t)br.bits(8); }
      if (br.bad) return -1;
    } else if (type == 1 || type == 2) {
      uint8_t lens[320];
      if (type == 1) {
        int i = 0;
        for (; i < 144; ++i) lens[i] = 8; for (; i < 256; ++i) lens[i] = 9; for (; i < 280; ++i) lens[i] = 7; for (; i < 288; ++i) lens[i] = 8;
        lit.build(lens, 288);
        for (i = 0; i < 30; ++i) lens[i] = 5;
        dist.build(lens, 30);
      } else {
        const int nlen = (int)br.bits(5) + 257, ndist = (int)br.bits(5) + 1, ncode = (int)br.bits(4) + 4;
        if (nlen > 286 || ndist > 30) return -1;
        static const uint8_t order[19] = {16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15};
        uint8_t cl[19]; memset(cl, 0, sizeof(cl));
        for (int i = 0; i < ncode; ++i) cl[order[i]] = (uint8_t)br.bits(3);
        Huff clh; if (!clh.build(cl, 19)) return -1;
        int idx = 0;
        while (idx < nlen + ndist) {
          const int sym = clh.decode(br);
          if (sym < 0) return -1;
          if (sym < 16) lens[idx++] = (uint8_t)sym;
          else {
            int rep, val = 0;
            if (sym == 16) { if (idx == 0) return -1; val = lens[idx - 1]; rep = 3 + (int)br.bits(2); }
            else if (sym == 17) rep = 3 + (int)br.bits(3);
            else rep = 11 + (int)br.bits(7);
            if (idx + rep > nlen + ndist) return -1;
            while (rep--) lens[idx++] = (uint8_t)val;
          }
        }
        if (!lit.build(lens, nlen) || !dist.build(lens + nlen, ndist)) return -1;
      }
      for (;;) {
        if (op + 300 > out.size()) ensure(300);               // room for a literal or the longest match plus the copy overshoot
        const int sym = lit.decode(br);
        if (sym < 0) return -1;
        if (sym < 256) { out[op++] = (uint8_t)sym; }
        else if (sym == 256) break;
        else {
          const int li = sym - 257;
          if (li >= 29) return -1;
          if (br.cnt < 48) br.fill();                           // length extra (5) + distance code (15) + distance extra (13) in one reservoir
          const uint32_t le = kLenPacked[li];
          const size_t len = (le & 0xFFFF) + (uint32_t)(br.buf & ((1u << (le >> 16)) - 1)); br.drop((int)(le >> 16));
          const int ds = dist.decode(br);
          if (ds < 0 || ds >= 30) return -1;
          const uint32_t de = kDistPacked[ds];
          const size_t d = (de & 0xFFFF) + (uint32_t)(br.buf & ((1u << (de >> 16)) - 1)); br.drop((int)(de >> 16));
          if (d > op) return -1;
          uint8_t* dst = out.data() + op; const uint8_t* from = dst - d;
          if (d >= 8) {                                         // 8 bytes at a time; may write up to 7 bytes past the match (slack above)
            for (size_t i = 0; i < len; i += 8) { uint64_t v; memcpy(&v, from + i, 8); memcpy(dst + i, &v, 8); }
          } else for (size_t i = 0; i < len; ++i) dst[i] = from[i];
          op += len;
        }
        if (br.bad) return -1;
      }
    } else return -1;
    if (final) break;
  }
  out.resize(op);
  return 0;
}

// ------------------------------------------------------------------------------ deflate (fixed Huffman + LZ77 hash chains)
namespace {
struct BitWriter {
  std::vector<uint8_t>& o; uint32_t buf = 0; int cnt = 0;
  explicit BitWriter(std::vector<uint8_t>& out) : o(out) {}
  void put(uint32_t v, int k) { buf |= v << cnt; cnt += k; while (cnt >= 8) { o.push_back((uint8_t)buf); buf >>= 8; cnt -= 8; } }
  void put_rev(uint32_t code, int k) { uint32_t r = 0; for (int i = 0; i < k; ++i) r |= ((code >> i) & 1u) << (k - 1 - i); put(r, k); }
  void flush() { if (cnt) { o.push_back((uint8_t)buf); buf = 0; cnt = 0; } }
};
void put_litlen(BitWriter& bw, int sym) {
  if (sym < 144) bw.put_rev(0x30 + sym, 8);
  else if (sym < 256) bw.put_rev(0x190 + (sym - 144), 9);
  else if (sym < 280) bw.put_rev(sym - 256, 7);
  else bw.put_rev(0xC0 + (sym - 280), 8);
}
}  // namespace

// The reference compresses depth (and the PNGs of saveToImages) with stb_image_write v1.00's zlib writer
// (sensorData.h:667, sensorData/stb_image_write.h:721-824): one fixed-Huffman block, greedy LZ77 with a one-byte lazy check,
// 16384 hash buckets that keep the most recent `quality`..2*quality positions.  Every decision below is the same decision, so
// a stream written here is byte-identical to the reference writer's (tests/test_sens_cpu.py):
//   * a candidate is usable if it is less than 32768 back (32767 for the lazy check), the longest match wins and of equal
//     matches the most recently inserted one (>=), matches shorter than 3 are literals;
//   * only positions where a search started are inserted; a bucket that reached 2*quality drops its older half first;
//   * the last 3 bytes are literals.
void scn::zlib_deflate(const uint8_t* src, size_t n, std::vector<uint8_t>& out) {
  const int quality = 8;                                        // compressDepth / stbi_write_png_to_mem both pass 8
  out.clear();
  out.push_back(0x78); out.push_back(0x5E);
  BitWriter bw(out);
  bw.put(1, 1); bw.put(1, 2);                                   // final block, fixed Huffman
  constexpr uint32_t kBuckets = 16384;
  struct Bucket { int32_t pos[16]; int n = 0; };                // 2*quality slots
  std::vector<Bucket> table(kBuckets);
  auto hash3 = [&](size_t i) {
    uint32_t h = (uint32_t)src[i] + ((uint32_t)src[i + 1] << 8) + ((uint32_t)src[i + 2] << 16);
    h ^= h << 3; h += h >> 5; h ^= h << 4; h += h >> 17; h ^= h << 25; h += h >> 6;
    return h & (kBuckets - 1);
  };
  auto match_len = [&](size_t a, size_t b, size_t limit) {      // common prefix of src[a..] and src[b..], at most min(limit, 258)
    size_t l = 0; const size_t m = limit < 258 ? limit : 258;
    while (l < m && src[a + l] == src[b + l]) ++l;
    return (int)l;
  };
  const long N = (long)n;
  long i = 0;
  while (i < N - 3) {
    Bucket& bk = table[hash3((size_t)i)];
    int best = 3; long best_pos = -1;
    for (int j = 0; j < bk.n; ++j) {
      if ((long)bk.pos[j] > i - 32768) {
        const int d = match_len((size_t)bk.pos[j], (size_t)i, (size_t)(N - i));
        if (d >= best) { best = d; best_pos = bk.pos[j]; }
      }
    }
    if (bk.n == 2 * quality) { memmove(bk.pos, bk.pos + quality, sizeof(int32_t) * quality); bk.n = quality; }
    bk.pos[bk.n++] = (int32_t)i;
    if (best_pos >= 0) {                                        // a longer match starting one byte later turns this byte into a literal
      const Bucket& nb = table[hash3((size_t)i + 1)];
      for (int j = 0; j < nb.n; ++j) {
        if ((long)nb.pos[j] > i - 32767 && match_len((size_t)nb.pos[j], (size_t)i + 1, (size_t)(N - i - 1)) > best) { best_pos = -1; break; }
      }
    }
    if (best_pos >= 0) {
      const int dist = (int)(i - best_pos);
      int li = 0; while (li < 28 && best >= kLenBase[li + 1]) ++li;
      put_litlen(bw, 257 + li); if (kLenExtra[li]) bw.put((uint32_t)(best - kLenBase[li]), kLenExtra[li]);
      int di = 0; while (di < 29 && dist >= kDistBase[di + 1]) ++di;
      bw.put_rev((uint32_t)di, 5); if (kDistExtra[di]) bw.put((uint32_t)(dist - kDistBase[di]), kDistExtra[di]);
      i += best;
    } else { put_litlen(bw, src[i]); ++i; }
  }
  for (; i < N; ++i) put_litlen(bw, src[i]);
  put_litlen(bw, 256);
  bw.flush();
  uint32_t a = 1, b = 0;
  for (size_t k = 0; k < n; ++k) { a = (a + src[k]) % 65521u; b = (b + a) % 65521u; }
  const uint32_t ad = (b << 16) | a;
  out.push_back((uint8_t)(ad >> 24)); out.push_back((uint8_t)(ad >> 16)); out.push_back((uint8_t)(ad >> 8)); out.push_back((uint8_t)ad);
}

// PNG as stb_image_write v1.00 writes it (stb_image_write.h:851-941), which is what saveToImages produces for TYPE_RAW colour
// (sensorData.h:1432-1440 via compressColor): 8-bit, no interlace, per row the filter with the smallest sum of |signed byte|
// (first of equals; row 0 tries none / sub / none / half-of-left / sub under the labels 0..4), one IDAT, the zlib writer above.
void scn::png_encode_stb(const uint8_t* px, uint32_t w, uint32_t h, int n, std::vector<uint8_t>& out) {
  const size_t row = (size_t)w * n;
  std::vector<uint8_t> filt((row + 1) * h);
  std::vector<int8_t> line(row ? row : 1);
  auto paeth = [](int a, int b, int c) { const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c);
                                         return pa <= pb && pa <= pc ? a : (pb <= pc ? b : c); };
  for (uint32_t j = 0; j < h; ++j) {
    static const int later[5] = {0, 1, 2, 3, 4}, first[5] = {0, 1, 0, 5, 6};
    const int* map = j ? later : first;
    const uint8_t* z = px + row * j;
    auto apply = [&](int type) {
      for (size_t i = 0; i < row; ++i) {
        const int cur = z[i], left = i >= (size_t)n ? z[i - n] : 0;
        const int up = (type == 2 || type == 3 || type == 4) ? z[(long)i - (long)row] : 0;
        const int ul = (type == 4 && i >= (size_t)n) ? z[(long)i - (long)row - n] : 0;
        int v;
        switch (type) {
          case 0: v = cur; break;
          case 1: v = cur - left; break;
          case 2: v = cur - up; break;
          case 3: v = cur - ((left + up) >> 1); break;
          case 4: v = cur - paeth(left, up, ul); break;
          case 5: v = cur - (left >> 1); break;
          default: v = cur - left; break;                       // 6: paeth(left, 0, 0) == left
        }
        line[i] = (int8_t)(uint8_t)v;
      }
    };
    int best = 0; long bestval = 0x7fffffff;
    for (int k = 0; k < 5; ++k) {
      apply(map[k]);
      long est = 0; for (size_t i = 0; i < row; ++i) est += std::abs((int)line[i]);
      if (est < bestval) { bestval = est; best = k; }
    }
    apply(map[best]);
    filt[j * (row + 1)] = (uint8_t)best;
    memcpy(&filt[j * (row + 1) + 1], line.data(), row);
  }
  std::vector<uint8_t> z;
  zlib_deflate(filt.data(), filt.size(), z);
  static uint32_t crc_table[256]; static bool crc_ready = false;
  if (!crc_ready) { for (uint32_t i = 0; i < 256; ++i) { uint32_t c = i; for (int k = 0; k < 8; ++k) c = (c >> 1) ^ ((c & 1) ? 0xedb88320u : 0u); crc_table[i] = c; } crc_ready = true; }
  auto be32 = [&](uint32_t v) { out.push_back((uint8_t)(v >> 24)); out.push_back((uint8_t)(v >> 16)); out.push_back((uint8_t)(v >> 8)); out.push_back((uint8_t)v); };
  auto chunk = [&](const char* tag, const uint8_t* d, size_t len) {
    be32((uint32_t)len);
    const size_t c0 = out.size();
    out.insert(out.end(), tag, tag + 4); out.insert(out.end(), d, d + len);
    uint32_t crc = ~0u; for (size_t i = c0; i < out.size(); ++i) crc = (crc >> 8) ^ crc_table[out[i] ^ (crc & 0xff)];
    be32(~crc);
  };
  out.clear();
  static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
  out.insert(out.end(), sig, sig + 8);
  static const int ctype[5] = {-1, 0, 4, 2, 6};
  uint8_t ihdr[13] = {(uint8_t)(w >> 24), (uint8_t)(w >> 16), (uint8_t)(w >> 8), (uint8_t)w, (uint8_t)(h >> 24), (uint8_t)(h >> 16), (uint8_t)(h >> 8), (uint8_t)h,
                      8, (uint8_t)ctype[n], 0, 0, 0};
  chunk("IHDR", ihdr, 13); chunk("IDAT", z.data(), z.size()); chunk("IEND", nullptr, 0);
}

// ------------------------------------------------------------------------------ container
// a compressed payload: a view into the mapped file (reader) or owned bytes (writer)
struct scn_blob {
  const uint8_t* p = nullptr; size_t n = 0; std::vector<uint8_t> own;
  const uint8_t* data() const { return own.empty() ? p : own.data(); }
  size_t size() const { return own.empty() ? n : own.size(); }
  bool empty() const { return size() == 0; }
  void view(const uint8_t* q, size_t m) { own.clear(); p = q; n = m; }
  void assign(const uint8_t* a, const uint8_t* b) { p = nullptr; n = 0; own.assign(a, b); }
  std::vector<uint8_t>& owned() { p = nullptr; n = 0; return own; }
};
struct scn_sens_frame {
  float cam2world[16];
  uint64_t ts_color = 0, ts_depth = 0;
  scn_blob color, depth;                      // compressed payloads as stored in the file
};
struct scn_sens {
  uint32_t version = 4;
  std::string sensor_name = "Unknown";
  float color_intr[16], color_extr[16], depth_intr[16], depth_extr[16];
  int32_t color_comp = -1, depth_comp = -1;
  uint32_t cw = 0, ch = 0, dw = 0, dh = 0;
  float depth_shift = 1000.0f;
  std::vector<scn_sens_frame> frames;
  std::vector<std::vector<uint8_t>> imu;      // 128-byte records (sensorData.h:786-833), kept verbatim
  // the file an opened stream was read from: mapped read-only (the payloads above point into it; a scan is 0.4-3 GB and
  // copying every payload into its own vector cost as much as fusing the scan) or, where mmap is not possible, read whole
  const uint8_t* file = nullptr; size_t file_len = 0; bool mapped = false; std::vector<uint8_t> file_buf;
  ~scn_sens() { if (mapped && file) munmap(const_cast<uint8_t*>(file), file_len); }
};

namespace {
void identity16(float* m) { for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? 1.0f : 0.0f; }
// istream-like cursor over the mapped file: a read past the end fails and every later read fails too
struct MemIn {
  const uint8_t* p; uint64_t n, pos = 0; bool ok = true;
  MemIn(const uint8_t* p_, uint64_t n_) : p(p_), n(n_) {}
  void read(char* dst, uint64_t k) { if (!ok || k > n - pos) { ok = false; return; } memcpy(dst, p + pos, k); pos += k; }
  const uint8_t* take(uint64_t k) { if (!ok || k > n - pos) { ok = false; return nullptr; } const uint8_t* q = p + pos; pos += k; return q; }
  int64_t tellg() const { return ok ? (int64_t)pos : -1; }
  explicit operator bool() const { return ok; }
};
template <typename T> bool rd(MemIn& in, T& v) { in.read((char*)&v, sizeof(T)); return (bool)in; }
const uint64_t kMaxPayload = 1ull << 31;
}  // namespace

extern "C" {

int scn_sens_open(const char* path, scn_sens** out) {
  if (!path || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  const int fd = ::open(path, O_RDONLY);
  if (fd < 0) return scn::fail(SCN_ERR_IO, "could not open file %s", path);                 // sensorData.h:1253-1255
  struct stat stt;
  if (fstat(fd, &stt) != 0 || S_ISDIR(stt.st_mode)) { ::close(fd); return scn::fail(SCN_ERR_IO, "could not open file %s", path); }
  const uint64_t file_size = (uint64_t)std::max<off_t>(stt.st_size, 0);
  scn_sens* s = new scn_sens();
  if (file_size && !getenv("SCN_SENS_NO_MMAP")) {
    void* m = mmap(nullptr, file_size, PROT_READ, MAP_PRIVATE | MAP_POPULATE, fd, 0);
    if (m != MAP_FAILED) { s->file = (const uint8_t*)m; s->file_len = file_size; s->mapped = true; madvise(m, file_size, MADV_WILLNEED); }
  }
  if (!s->mapped && file_size) {                                 // no mmap (special file systems): read the file whole
    s->file_buf.resize(file_size);
    uint64_t got = 0;
    while (got < file_size) { const ssize_t r = ::read(fd, s->file_buf.data() + got, file_size - got); if (r <= 0) break; got += (uint64_t)r; }
    s->file_buf.resize(got); s->file = s->file_buf.data(); s->file_len = got;
  }
  ::close(fd);
  MemIn in(s->file, s->file_len);
  // every count / size field is checked against what the file can still hold before anything is allocated for it
  auto left = [&]() { const int64_t p = in.tellg(); return p < 0 ? (uint64_t)0 : file_size - std::min<uint64_t>(file_size, (uint64_t)p); };
  auto bail = [&](int code, const char* msg) { delete s; return scn::fail(code, "%s: %s", path, msg); };
  if (!rd(in, s->version)) return bail(SCN_ERR_FORMAT, "truncated header");
  if (s->version != 4) {                                                                     // :882-886
    const uint32_t v = s->version; delete s;
    return scn::fail(SCN_ERR_FORMAT, "Invalid file version -- found %u but expectd 4", v);
  }
  uint64_t slen = 0;
  if (!rd(in, slen) || slen > (1u << 20) || slen > left()) return bail(SCN_ERR_FORMAT, "bad sensor name length");
  s->sensor_name.resize(slen);
  in.read(&s->sensor_name[0], (std::streamsize)slen);
  in.read((char*)s->color_intr, 64); in.read((char*)s->color_extr, 64);
  in.read((char*)s->depth_intr, 64); in.read((char*)s->depth_extr, 64);
  rd(in, s->color_comp); rd(in, s->depth_comp);
  rd(in, s->cw); rd(in, s->ch); rd(in, s->dw); rd(in, s->dh); rd(in, s->depth_shift);
  uint64_t nf = 0;
  if (!rd(in, nf)) return bail(SCN_ERR_FORMAT, "truncated header");
  if (nf > (1ull << 32) || nf > left() / 96) return bail(SCN_ERR_FORMAT, "implausible frame count");          // 96 = pose + 2 stamps + 2 sizes
  s->frames.resize(nf);
  for (uint64_t i = 0; i < nf; ++i) {
    scn_sens_frame& f = s->frames[i];
    uint64_t cb = 0, db = 0;
    in.read((char*)f.cam2world, 64);
    if (!rd(in, f.ts_color) || !rd(in, f.ts_depth) || !rd(in, cb) || !rd(in, db)) return bail(SCN_ERR_FORMAT, "truncated frame header");
    if (cb > kMaxPayload || db > kMaxPayload) return bail(SCN_ERR_FORMAT, "implausible payload size");
    if (cb + db > left()) return bail(SCN_ERR_FORMAT, "truncated frame payload");
    const uint8_t* cp = in.take(cb); const uint8_t* dp = in.take(db);        // views into the mapped file
    if (!in) return bail(SCN_ERR_FORMAT, "truncated frame payload");
    f.color.view(cp, cb); f.depth.view(dp, db);
  }
  uint64_t ni = 0;
  if (rd(in, ni) && ni > 0) {
    if (ni >= (1ull << 32) || ni > left() / 128) return bail(SCN_ERR_FORMAT, "truncated IMU frames");
    s->imu.resize(ni);
    for (uint64_t i = 0; i < ni; ++i) { s->imu[i].resize(128); in.read((char*)s->imu[i].data(), 128); if (!in) return bail(SCN_ERR_FORMAT, "truncated IMU frames"); }
  }
  *out = s;
  return SCN_OK;
}

void scn_sens_close(scn_sens* s) { delete s; }

int scn_sens_info(const scn_sens* s, scn_sens_info_t* info) {
  if (!s || !info) return scn::fail(SCN_ERR_ARG, "null argument");
  memset(info, 0, sizeof(*info));
  info->version = s->version;
  info->color_width = s->cw; info->color_height = s->ch; info->depth_width = s->dw; info->depth_height = s->dh;
  info->color_compression = s->color_comp; info->depth_compression = s->depth_comp;
  info->depth_shift = s->depth_shift; info->n_frames = s->frames.size(); info->n_imu_frames = s->imu.size();
  memcpy(info->color_intrinsic, s->color_intr, 64); memcpy(info->color_extrinsic, s->color_extr, 64);
  memcpy(info->depth_intrinsic, s->depth_intr, 64); memcpy(info->depth_extrinsic, s->depth_extr, 64);
  snprintf(info->sensor_name, sizeof(info->sensor_name), "%s", s->sensor_name.c_str());
  return SCN_OK;
}

int scn_sens_frame_meta(const scn_sens* s, uint64_t i, float cam2world[16], uint64_t* tc, uint64_t* td, uint64_t* cb, uint64_t* db) {
  if (!s) return scn::fail(SCN_ERR_ARG, "null handle");
  if (i >= s->frames.size()) return scn::fail(SCN_ERR_ARG, "out of bounds");               // sensorData.h:944
  const scn_sens_frame& f = s->frames[i];
  if (cam2world) memcpy(cam2world, f.cam2world, 64);
  if (tc) *tc = f.ts_color; if (td) *td = f.ts_depth; if (cb) *cb = f.color.size(); if (db) *db = f.depth.size();
  return SCN_OK;
}

int scn_sens_frame_depth_u16(const scn_sens* s, uint64_t i, uint16_t* out) {
  if (!s || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (i >= s->frames.size()) return scn::fail(SCN_ERR_ARG, "out of bounds");
  const scn_sens_frame& f = s->frames[i];
  const size_t want = (size_t)s->dw * s->dh * 2;
  if (s->depth_comp == 0) {                                                                  // TYPE_RAW_USHORT :724-730
    if (f.depth.empty()) return scn::fail(SCN_ERR_FORMAT, "invalid data");
    memcpy(out, f.depth.data(), std::min(want, f.depth.size()));
    return SCN_OK;
  }
  if (s->depth_comp == 1) {                                                                  // TYPE_ZLIB_USHORT :703-709
    static thread_local std::vector<uint8_t> raw;                                            // reused: decode pools call this from many threads
    if (scn::zlib_inflate(f.depth.data(), f.depth.size(), raw, want)) return scn::fail(SCN_ERR_FORMAT, "frame %llu: corrupt zlib depth stream", (unsigned long long)i);
    if (raw.size() < want) return scn::fail(SCN_ERR_FORMAT, "frame %llu: depth stream holds %zu bytes, need %zu", (unsigned long long)i, raw.size(), want);
    memcpy(out, raw.data(), want);
    return SCN_OK;
  }
  if (s->depth_comp == 2) return scn::fail(SCN_ERR_UNSUPPORTED, "need UPLINK_COMPRESSION");  // :711-722
  return scn::fail(SCN_ERR_FORMAT, "invalid type");
}

int scn_sens_frame_color_rgb8(const scn_sens* s, uint64_t i, uint8_t* out) {
  if (!s || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (i >= s->frames.size()) return scn::fail(SCN_ERR_ARG, "out of bounds");
  const scn_sens_frame& f = s->frames[i];
  const size_t want = (size_t)s->cw * s->ch * 3;
  if (f.color.empty()) return scn::fail(SCN_ERR_FORMAT, "decompression error");
  if (s->color_comp == 0) { memcpy(out, f.color.data(), std::min(want, f.color.size())); return SCN_OK; }   // :638-645
  if (s->color_comp == 2) return scn::jpeg_decode_rgb8(f.color.data(), f.color.size(), s->cw, s->ch, out);
  if (s->color_comp == 1) return scn::png_decode_rgb8(f.color.data(), f.color.size(), s->cw, s->ch, out);
  return scn::fail(SCN_ERR_FORMAT, "invliad type");
}

int scn_sens_frame_payload(const scn_sens* s, uint64_t i, const uint8_t** color, const uint8_t** depth) {
  if (!s) return scn::fail(SCN_ERR_ARG, "null handle");
  if (i >= s->frames.size()) return scn::fail(SCN_ERR_ARG, "out of bounds");
  if (color) *color = s->frames[i].color.data();
  if (depth) *depth = s->frames[i].depth.data();
  return SCN_OK;
}

// ------------------------------------------------------------------------------ read-ahead cache (RGBDFrameCacheRead)
struct scn_sens_cache {
  struct Slot { std::vector<uint16_t> depth; std::vector<uint8_t> color; int rc = 0; std::string err; bool ready = false; };
  const scn_sens* s = nullptr;
  std::vector<Slot> slots;
  std::vector<std::thread> workers;
  std::mutex m; std::condition_variable cv_ready, cv_space;
  uint64_t next_claim = 0, next_out = 0; bool stop = false;
  void work() {
    for (;;) {
      uint64_t i;
      {
        std::unique_lock<std::mutex> l(m);
        cv_space.wait(l, [&]() { return stop || next_claim >= s->frames.size() || next_claim < next_out + slots.size(); });
        if (stop || next_claim >= s->frames.size()) return;
        i = next_claim++;
      }
      Slot& sl = slots[i % slots.size()];                      // free: the consumer has passed frame i - slots.size()
      sl.depth.resize((size_t)s->dw * s->dh); sl.color.resize((size_t)s->cw * s->ch * 3);
      int rc = scn_sens_frame_depth_u16(s, i, sl.depth.data());
      if (!rc && s->color_comp >= 0 && !s->frames[i].color.empty()) rc = scn_sens_frame_color_rgb8(s, i, sl.color.data());
      { std::lock_guard<std::mutex> l(m); sl.rc = rc; if (rc) sl.err = scn_last_error(); sl.ready = true; }
      cv_ready.notify_all();
    }
  }
};

int scn_sens_cache_create(const scn_sens* s, uint32_t cache_size, int n_threads, scn_sens_cache** out) {
  if (!s || !out || cache_size == 0) return scn::fail(SCN_ERR_ARG, "bad argument");
  scn_sens_cache* c = new scn_sens_cache();
  c->s = s; c->slots.resize(cache_size);
  unsigned nt = n_threads > 0 ? (unsigned)n_threads : std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
  nt = std::min<unsigned>(nt, cache_size);
  for (unsigned t = 0; t < nt; ++t) c->workers.emplace_back([c]() { c->work(); });
  *out = c;
  return SCN_OK;
}

int scn_sens_cache_next(scn_sens_cache* c, uint16_t* depth_out, uint8_t* color_out, uint64_t* ts_depth, uint64_t* ts_color) {
  if (!c) return scn::fail(SCN_ERR_ARG, "null handle");
  std::unique_lock<std::mutex> l(c->m);
  if (c->next_out >= c->s->frames.size()) return 0;
  const uint64_t i = c->next_out;
  scn_sens_cache::Slot& sl = c->slots[i % c->slots.size()];
  c->cv_ready.wait(l, [&]() { return sl.ready && i < c->next_claim; });
  const int rc = sl.rc;
  if (rc) scn::fail(rc, "%s", sl.err.c_str());
  else {
    if (depth_out) memcpy(depth_out, sl.depth.data(), sl.depth.size() * 2);
    if (color_out) memcpy(color_out, sl.color.data(), sl.color.size());
    if (ts_depth) *ts_depth = c->s->frames[i].ts_depth;
    if (ts_color) *ts_color = c->s->frames[i].ts_color;
  }
  sl.ready = false; ++c->next_out;
  l.unlock();
  c->cv_space.notify_all();
  return rc ? rc : 1;
}

void scn_sens_cache_destroy(scn_sens_cache* c) {
  if (!c) return;
  { std::lock_guard<std::mutex> l(c->m); c->stop = true; }
  c->cv_space.notify_all();
  for (auto& t : c->workers) t.join();
  delete c;
}

int scn_sens_set_pose(scn_sens* s, uint64_t i, const float cam2world[16]) {
  if (!s || !cam2world) return scn::fail(SCN_ERR_ARG, "null argument");
  if (i >= s->frames.size()) return scn::fail(SCN_ERR_ARG, "out of bounds");
  memcpy(s->frames[i].cam2world, cam2world, 64);
  return SCN_OK;
}

int scn_sens_save(const scn_sens* s, const char* path) {
  if (!s || !path) return scn::fail(SCN_ERR_ARG, "null argument");
  // a stream opened from a file points into its mapping: never truncate that file in place (pose write-back saves over the
  // input) - write beside it and rename
  const std::string tmp = s->mapped ? std::string(path) + ".tmp" + std::to_string((long long)getpid()) : std::string(path);
  std::ofstream out(tmp, std::ios::binary);
  if (!out) return scn::fail(SCN_ERR_IO, "Unable to open file for writing: %s", path);       // sensorData.h:1103-1105
  out.write((const char*)&s->version, 4);
  const uint64_t slen = s->sensor_name.size();
  out.write((const char*)&slen, 8); out.write(s->sensor_name.data(), (std::streamsize)slen);
  out.write((const char*)s->color_intr, 64); out.write((const char*)s->color_extr, 64);
  out.write((const char*)s->depth_intr, 64); out.write((const char*)s->depth_extr, 64);
  out.write((const char*)&s->color_comp, 4); out.write((const char*)&s->depth_comp, 4);
  out.write((const char*)&s->cw, 4); out.write((const char*)&s->ch, 4); out.write((const char*)&s->dw, 4); out.write((const char*)&s->dh, 4);
  out.write((const char*)&s->depth_shift, 4);
  const uint64_t nf = s->frames.size();
  out.write((const char*)&nf, 8);
  for (const scn_sens_frame& f : s->frames) {
    const uint64_t cb = f.color.size(), db = f.depth.size();
    out.write((const char*)f.cam2world, 64);
    out.write((const char*)&f.ts_color, 8); out.write((const char*)&f.ts_depth, 8);
    out.write((const char*)&cb, 8); out.write((const char*)&db, 8);
    out.write((const char*)f.color.data(), (std::streamsize)cb); out.write((const char*)f.depth.data(), (std::streamsize)db);
  }
  const uint64_t ni = s->imu.size();
  out.write((const char*)&ni, 8);
  for (const auto& r : s->imu) out.write((const char*)r.data(), 128);
  out.close();
  if (!out) { if (s->mapped) remove(tmp.c_str()); return scn::fail(SCN_ERR_IO, "write failed: %s", path); }
  if (s->mapped && rename(tmp.c_str(), path) != 0) { remove(tmp.c_str()); return scn::fail(SCN_ERR_IO, "Unable to open file for writing: %s", path); }
  return SCN_OK;
}

int scn_sens_create(uint32_t cw, uint32_t ch, uint32_t dw, uint32_t dh, const float color_intr[16], const float depth_intr[16],
                    int32_t color_comp, int32_t depth_comp, float depth_shift, const char* name, scn_sens** out) {
  if (!out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (color_comp < 0 || color_comp > 2 || depth_comp < 0 || depth_comp > 1) return scn::fail(SCN_ERR_UNSUPPORTED, "unknown compression type");
  scn_sens* s = new scn_sens();
  s->cw = cw; s->ch = ch; s->dw = dw; s->dh = dh; s->color_comp = color_comp; s->depth_comp = depth_comp;
  s->depth_shift = depth_shift; s->sensor_name = name ? name : "Unknown";
  identity16(s->color_extr); identity16(s->depth_extr); identity16(s->color_intr); identity16(s->depth_intr);
  if (color_intr) memcpy(s->color_intr, color_intr, 64);
  if (depth_intr) memcpy(s->depth_intr, depth_intr, 64);
  *out = s;
  return SCN_OK;
}

int scn_sens_add_frame(scn_sens* s, const uint8_t* color, uint64_t color_bytes, const uint16_t* depth, const float cam2world[16],
                       uint64_t ts_color, uint64_t ts_depth) {
  if (!s) return scn::fail(SCN_ERR_ARG, "null handle");
  scn_sens_frame f;
  if (cam2world) memcpy(f.cam2world, cam2world, 64); else identity16(f.cam2world);
  f.ts_color = ts_color; f.ts_depth = ts_depth;
  if (color) {
    if (s->color_comp == 0) color_bytes = (uint64_t)s->cw * s->ch * 3;
    f.color.assign(color, color + color_bytes);
  }
  if (depth) {
    const size_t raw = (size_t)s->dw * s->dh * 2;
    if (s->depth_comp == 0) f.depth.assign((const uint8_t*)depth, (const uint8_t*)depth + raw);
    else scn::zlib_deflate((const uint8_t*)depth, raw, f.depth.owned());
  }
  s->frames.push_back(std::move(f));
  return SCN_OK;
}

// operator<< (sensorData.h:1941-1955)
int64_t scn_sens_describe(const scn_sens* s, char* buf, uint64_t cap) {
  if (!s) return scn::fail(SCN_ERR_ARG, "null handle");
  std::ostringstream o;
  o << "CalibratedSensorData:\n";
  o << '\t' << "sensorData.m_versionNumber" << '=' << s->version << '\n';
  o << '\t' << "sensorData.m_sensorName" << '=' << s->sensor_name << '\n';
  o << '\t' << "sensorData.m_colorWidth" << '=' << s->cw << '\n';
  o << '\t' << "sensorData.m_colorHeight" << '=' << s->ch << '\n';
  o << '\t' << "sensorData.m_depthWidth" << '=' << s->dw << '\n';
  o << '\t' << "sensorData.m_depthHeight" << '=' << s->dh << '\n';
  o << '\t' << "sensorData.m_depthShift" << '=' << s->depth_shift << '\n';
  o << '\t' << "sensorData.m_frames.size()" << '=' << s->frames.size() << '\n';
  o << '\t' << "sensorData.m_IMUFrames.size()" << '=' << s->imu.size() << '\n';
  const std::string t = o.str();
  if (buf && cap) { const size_t n = std::min<size_t>(cap - 1, t.size()); memcpy(buf, t.data(), n); buf[n] = 0; }
  return (int64_t)t.size();
}

namespace {
std::string counter_name(const std::string& base, unsigned cur, const std::string& ending, unsigned digits) {   // StringCounter :1292-1339
  std::stringstream ss;
  ss << base;
  for (unsigned i = std::max(1u, (unsigned)ceilf(log10f((float)cur + 1))); i < digits; i++) ss << "0";
  ss << cur;
  ss << (ending[0] == '.' ? ending : "." + ending);
  return ss.str();
}
}  // namespace

int scn_sens_save_to_images(const scn_sens* s, const char* out_dir) {
  if (!s || !out_dir) return scn::fail(SCN_ERR_ARG, "null argument");
  const std::string folder = out_dir;
  struct stat sb;
  if (stat(folder.c_str(), &sb) != 0) mkdir(folder.c_str(), 0777);
  {
    std::ofstream m(folder + "/" + "_info.txt");
    if (!m) return scn::fail(SCN_ERR_IO, "cannot open file %s/_info.txt", out_dir);
    m << "m_versionNumber" << " = " << s->version << '\n';
    m << "m_sensorName" << " = " << s->sensor_name << '\n';
    m << "m_colorWidth" << " = " << s->cw << '\n';
    m << "m_colorHeight" << " = " << s->ch << '\n';
    m << "m_depthWidth" << " = " << s->dw << '\n';
    m << "m_depthHeight" << " = " << s->dh << '\n';
    m << "m_depthShift" << " = " << s->depth_shift << '\n';
    const char* names[4] = {"m_calibrationColorIntrinsic", "m_calibrationColorExtrinsic", "m_calibrationDepthIntrinsic", "m_calibrationDepthExtrinsic"};
    const float* mats[4] = {s->color_intr, s->color_extr, s->depth_intr, s->depth_extr};
    for (int k = 0; k < 4; ++k) { m << names[k] << " = "; for (int i = 0; i < 16; ++i) m << mats[k][i] << " "; m << "\n"; }
    m << "m_frames.size" << " = " << (uint64_t)s->frames.size() << "\n";
    if (!s->imu.empty()) std::cout << "warning sensor has imu frames; but writing is not implemented here" << std::endl;
  }
  if (s->frames.empty()) return SCN_OK;
  const std::string cend = s->color_comp == 2 ? "jpg" : "png";
  std::cout << std::endl;
  std::vector<uint16_t> depth((size_t)s->dw * s->dh);
  for (size_t i = 0; i < s->frames.size(); ++i) {
    std::cout << "\r[ processing frame " << std::to_string(i) << " of " << std::to_string(s->frames.size()) << " ]";
    const scn_sens_frame& f = s->frames[i];
    const std::string base = folder + "/" + "frame-";
    if (s->color_comp == 1 || s->color_comp == 2) {
      const std::string cf = counter_name(base, (unsigned)i, "color." + cend, 6);
      FILE* fp = fopen(cf.c_str(), "wb");
      if (!fp) return scn::fail(SCN_ERR_IO, "cannot open file %s", cf.c_str());
      fwrite(f.color.data(), 1, f.color.size(), fp); fclose(fp);
    } else if (s->color_comp == 0) {
      // TYPE_RAW colour is re-encoded as frame-XXXXXX.color.png (sensorData.h:1410-1440).  The reference does that through its
      // uplink codec (Windows builds); built without it, as here, it throws "need UPLINK_COMPRESSION" (:592).  We write the
      // PNG with the stb_image_write-compatible encoder above.
      const std::string cf = counter_name(base, (unsigned)i, "color.png", 6);
      if (f.color.size() < (size_t)s->cw * s->ch * 3) return scn::fail(SCN_ERR_FORMAT, "invalid data");
      std::vector<uint8_t> png;
      scn::png_encode_stb(f.color.data(), s->cw, s->ch, 3, png);
      FILE* fp = fopen(cf.c_str(), "wb");
      if (!fp) return scn::fail(SCN_ERR_IO, "cannot open file %s", cf.c_str());
      fwrite(png.data(), 1, png.size(), fp); fclose(fp);
    } else return scn::fail(SCN_ERR_FORMAT, "unknown format");
    int rc = scn_sens_frame_depth_u16(s, i, depth.data());
    if (rc) return rc;
    {                                                                                        // saveAsPGM :1342-1375
      std::ofstream of(counter_name(base, (unsigned)i, "depth.pgm", 6), std::ios::binary);
      std::stringstream ss;
      ss << "P5\n";
      ss << "# data values are 16-bit each; depth shift is " << s->depth_shift << "\n";
      ss << s->dw << " " << s->dh << "\n";
      ss << std::numeric_limits<unsigned short>::max() << "\n";
      of << ss.str();
      uint8_t* dc = (uint8_t*)depth.data();
      for (size_t k = 0; k < depth.size(); ++k) std::swap(dc[2 * k], dc[2 * k + 1]);
      of.write((const char*)depth.data(), (std::streamsize)(depth.size() * 2));
    }
    {                                                                                        // savePoseFile :1706-1714
      std::ofstream pf(counter_name(base, (unsigned)i, ".pose.txt", 6));
      const float* m = f.cam2world;
      pf << m[0] << " " << m[1] << " " << m[2] << " " << m[3] << "\n" << m[4] << " " << m[5] << " " << m[6] << " " << m[7] << "\n"
         << m[8] << " " << m[9] << " " << m[10] << " " << m[11] << "\n" << m[12] << " " << m[13] << " " << m[14] << " " << m[15];
    }
  }
  return SCN_OK;
}

// `sens <file.sens> [outDir]` (SensReader/c++/src/main.cpp:28-97)
int scn_sens_main(int argc, const char** argv) {
  std::string filename = "scene0001_00.sens", outDir = "./out/";
  if (argc >= 2) filename = argv[1];
  else { std::cout << "run ./sens <sensfilename>.sens"; std::cout << "type in filename manually: "; std::cin >> filename; }
  if (argc >= 3) outDir = argv[2];
  std::cout << "filename =\t" << filename << std::endl;
  std::cout << "outDir =\t" << outDir << std::endl;
  std::cout << "loading from file... ";
  scn_sens* s = nullptr;
  if (scn_sens_open(filename.c_str(), &s)) { std::cout << "Exception caught! " << scn_last_error() << std::endl; return EXIT_FAILURE; }
  std::cout << "done!" << std::endl;
  std::vector<char> buf(4096);
  scn_sens_describe(s, buf.data(), buf.size());
  std::cout << buf.data() << std::endl;
  if (scn_sens_save_to_images(s, outDir.c_str())) { std::cout << "Exception caught! " << scn_last_error() << std::endl; scn_sens_close(s); return EXIT_FAILURE; }
  if (!s->frames.empty()) {                         // processFrame(sd, 0): decode one frame of each stream (main.cpp:6-26,64)
    std::vector<uint16_t> d((size_t)s->dw * s->dh); std::vector<uint8_t> c((size_t)s->cw * s->ch * 3);
    scn_sens_frame_depth_u16(s, 0, d.data());
    scn_sens_frame_color_rgb8(s, 0, c.data());
  }
  std::cout << std::endl;
  std::cout << "All done :)" << std::endl;
  scn_sens_close(s);
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------ frame helpers of the scene drivers
int scn::posed_frames(const scn_sens* s, uint64_t f0, uint64_t f1, PosedFrames& out) {
  out.frames.clear(); out.poses.clear();
  for (uint64_t f = f0; f < f1; ++f) {
    float T[16];
    if (int rc = scn_sens_frame_meta(s, f, T, nullptr, nullptr, nullptr, nullptr)) return rc;
    if (T[0] == -INFINITY) continue;
    out.frames.push_back(f); out.poses.insert(out.poses.end(), T, T + 16);
  }
  return SCN_OK;
}

void scn::build_color_lut(const scn_sens_info_t& in, std::vector<int32_t>& lut) {
  const uint32_t W = in.depth_width, H = in.depth_height;
  lut.resize((size_t)W * H);
  const float fxd = in.depth_intrinsic[0], cxd = in.depth_intrinsic[2], fyd = in.depth_intrinsic[5], cyd = in.depth_intrinsic[6];
  const float fxc = in.color_intrinsic[0], cxc = in.color_intrinsic[2], fyc = in.color_intrinsic[5], cyc = in.color_intrinsic[6];
  for (uint32_t y = 0; y < H; ++y) for (uint32_t x = 0; x < W; ++x) {
    const float u = ((float)x - cxd) / fxd * fxc + cxc, v = ((float)y - cyd) / fyd * fyc + cyc;
    const long cx = lrintf(u), cy = lrintf(v);
    lut[(size_t)y * W + x] = (cx >= 0 && cy >= 0 && cx < (long)in.color_width && cy < (long)in.color_height) ? (int32_t)(cy * in.color_width + cx) : -1;
  }
}

int scn::sens_color_to_depth(const scn_sens* s, uint64_t frame, const int32_t* lut, size_t n_px, uint8_t* scratch, uint8_t* out) {
  if (int rc = scn_sens_frame_color_rgb8(s, frame, scratch)) return rc;
  rgb8_through_lut(scratch, lut, n_px, out);
  return SCN_OK;
}
