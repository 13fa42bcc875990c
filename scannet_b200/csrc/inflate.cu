// Depth decode on the GPU (SURVEY.md §8f-2): the TYPE_ZLIB_USHORT payloads of a .sens stream
// (SensReader/c++/src/sensorData.h:703-709, stbi_zlib_decode_malloc) are uploaded COMPRESSED and inflated in HBM, so raw
// depth never crosses PCIe and never touches a host core.
//
// A deflate stream has no internal synchronisation points, so the parallelism is across frames: ONE WARP PER FRAME.
// What bounds a single stream is latency, not bandwidth: ~115-170 k symbols per 640x480 frame, ~60 % of them LZ77 matches
// whose source bytes were written moments ago, at distances spread over the whole 32 KB window (measured on depth frames:
// only ~45 % within 8 KB).  Read back from global memory every match costs an L2 round trip.  So each
// warp keeps the 32 KB deflate window as a ring in SHARED memory: literals and
// matches are written to the ring and streamed to HBM (fire-and-forget stores), matches are copied ring -> ring by the
// whole warp (byte i of a match is window[o - dist + (i mod dist)], which only reads bytes that existed before the match,
// so the 32 lanes are independent even when the match overlaps itself), and the bit reader runs one 32-bit word ahead
// of the decoder so that input loads are off the dependent chain.  All 32 lanes run the same bit reader and Huffman
// decoder redundantly (same addresses -> broadcast loads, no divergence, no shuffles).  38.5 KB of shared memory per
// stream = 5 streams per SM (660 in flight on 132 SMs).
// Fixed-Huffman blocks (what stb's compressor - the one the ScanNet tools use - emits) and dynamic blocks go through the
// same 9-bit lookahead tables (canonical first-code/offset tables beyond 9 bits) kept in shared memory; stored blocks are
// copied.  The same source compiles for the host (one lane, no ring) so the decoder is unit-tested on the CPU against
// zlib streams of every block type.
#include <algorithm>
#include <chrono>
#include <thread>
#include <vector>

#include "scn_common.h"
#include "stage_pool.h"

#define SCN_HD __host__ __device__ __forceinline__

namespace {

template <int BITS>
struct HuffTabT {                    // canonical Huffman code, lengths 1..15
  uint16_t count[16];                // codes per length
  uint16_t first[16];                // first code of each length
  uint16_t offs[16];                 // index of that code's symbol in sym[]
  uint16_t sym[288];
  static constexpr int kBits = BITS;
  uint32_t fast[1 << BITS];          // BITS-bit lookahead (stream bit order) -> packed entry (below); kLongCode = longer code
};
// Packed table entry: everything the main loop needs from one shared-memory load.
//   bits 0-3 code length, 4-7 number of extra bits, 8-9 kind, 10-14 code length + extra bits, 16-31 value (literal byte /
//   length base / distance base / symbol)
enum { K_LIT = 0, K_BASE = 1, K_EOB = 2, K_BAD = 3 };
// literal/length codes of a noisy depth frame reach 11-12 bits (5.7 % of the symbols were longer than 9): 10-bit lookahead;
// the 30 distance codes rarely pass 8 bits.  6.8 KB of tables per stream keeps 26 streams per SM resident when the window
// lives in HBM (a scan of 3840 frames in one wave).
constexpr int kLitBits = 10, kDistBits = 8;
using LitTab = HuffTabT<kLitBits>;
using DistTab = HuffTabT<kDistBits>;
constexpr uint32_t kLongCode = K_BAD << 8;           // kind "bad" with code length 0: the code is longer than the lookahead
enum { M_PLAIN = 0, M_LITLEN = 1, M_DIST = 2 };     // what the symbols of a table mean
struct InflateScratch { LitTab lit; DistTab dist; uint8_t lens[320]; };
constexpr uint32_t kWin = 32768;                                   // deflate window = the shared-memory ring of the device decoder
struct InflateScratchDev { uint8_t ring[kWin]; InflateScratch s; };

// On the device the scratch lives in (dynamic) shared memory and is addressed directly; a generic pointer made the compiler
// re-derive the shared window for every symbol.
extern __shared__ __align__(16) unsigned char g_inflate_smem[];
#ifdef __CUDA_ARCH__
#define SCN_SCR(scr) (RING ? reinterpret_cast<InflateScratchDev*>(g_inflate_smem)->s : *reinterpret_cast<InflateScratch*>(g_inflate_smem))
#define SCN_RING (reinterpret_cast<InflateScratchDev*>(g_inflate_smem)->ring)
#else
#define SCN_SCR(scr) (*(scr))
#endif

struct BitIn { const uint8_t* p; uint32_t n, pos; uint64_t bb; int bc; int over; uint32_t ahead; int has_ahead; };   // streams and frames are far below 4 GB: 32-bit offsets halve the address arithmetic

// Guarantees more than 32 valid bits (every decode step needs at most 32: a length code + extra bits is 20, a distance
// code + extra bits 28, a stored-block header 32).  One aligned 32-bit load per four input bytes: the dependent chain of
// a single warp is what bounds the kernel, so fewer, wider loads matter.  Past the end the buffer is zero-filled and the
// shortfall remembered.
// `ahead` holds the aligned word at b.pos, loaded one refill early: the load's latency overlaps the symbols decoded in
// between (b.pos is advanced only when the word is consumed, so the stored-block path can still derive its source offset).
SCN_HD void bi_refill(BitIn& b) {
  while (b.bc <= 32) {
    if (b.has_ahead) {
      b.bb |= (uint64_t)b.ahead << b.bc; b.pos += 4; b.bc += 32;
      b.has_ahead = (b.pos + 4 <= b.n);
      if (b.has_ahead) b.ahead = *(const uint32_t*)(b.p + b.pos);
    }
    else if ((((size_t)(b.p + b.pos)) & 3) == 0 && b.pos + 4 <= b.n) { b.has_ahead = 1; b.ahead = *(const uint32_t*)(b.p + b.pos); }
    else if (b.pos < b.n) { b.bb |= (uint64_t)b.p[b.pos++] << b.bc; b.bc += 8; }
    else { b.over += 8; b.bc += 8; }
  }
}
SCN_HD void bi_restart(BitIn& b, uint32_t pos) { b.pos = pos; b.bb = 0; b.bc = 0; b.over = 0; b.has_ahead = 0; }
SCN_HD unsigned bi_peek(const BitIn& b, int n) { return (unsigned)(b.bb & ((1ull << n) - 1ull)); }
SCN_HD void bi_drop(BitIn& b, int n) { b.bb >>= n; b.bc -= n; }
SCN_HD unsigned bi_get(BitIn& b, int n) { const unsigned v = bi_peek(b, n); bi_drop(b, n); return v; }
SCN_HD bool bi_overrun(const BitIn& b) { return b.over > b.bc; }                        // consumed bits that were never in the input

SCN_HD unsigned rev_bits(unsigned v, int n) {
#ifdef __CUDA_ARCH__
  return __brev(v) >> (32 - n);
#else
  unsigned r = 0; for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1u); v >>= 1; } return r;
#endif
}

// RFC 1951 3.2.5 base values / extra bits, packed as (base << 4 | extra).  __constant__ on the device: a local array was
// compiled into an 80-instruction select tree per lookup (46 % of all executed instructions in the first profile).
#define SCN_LEN_TAB {3 << 4 | 0, 4 << 4 | 0, 5 << 4 | 0, 6 << 4 | 0, 7 << 4 | 0, 8 << 4 | 0, 9 << 4 | 0, 10 << 4 | 0, 11 << 4 | 1, 13 << 4 | 1, \
                     15 << 4 | 1, 17 << 4 | 1, 19 << 4 | 2, 23 << 4 | 2, 27 << 4 | 2, 31 << 4 | 2, 35 << 4 | 3, 43 << 4 | 3, 51 << 4 | 3, 59 << 4 | 3, \
                     67 << 4 | 4, 83 << 4 | 4, 99 << 4 | 4, 115 << 4 | 4, 131 << 4 | 5, 163 << 4 | 5, 195 << 4 | 5, 227 << 4 | 5, 258 << 4 | 0}
#define SCN_DIST_TAB {1 << 4 | 0, 2 << 4 | 0, 3 << 4 | 0, 4 << 4 | 0, 5 << 4 | 1, 7 << 4 | 1, 9 << 4 | 2, 13 << 4 | 2, 17 << 4 | 3, 25 << 4 | 3, \
                      33 << 4 | 4, 49 << 4 | 4, 65 << 4 | 5, 97 << 4 | 5, 129 << 4 | 6, 193 << 4 | 6, 257 << 4 | 7, 385 << 4 | 7, 513 << 4 | 8, 769 << 4 | 8, \
                      1025 << 4 | 9, 1537 << 4 | 9, 2049 << 4 | 10, 3073 << 4 | 10, 4097 << 4 | 11, 6145 << 4 | 11, 8193 << 4 | 12, 12289 << 4 | 12, \
                      16385 << 4 | 13, 24577 << 4 | 13}
__constant__ unsigned c_len_tab[29] = SCN_LEN_TAB;
__constant__ unsigned c_dist_tab[30] = SCN_DIST_TAB;
static const unsigned h_len_tab[29] = SCN_LEN_TAB;
static const unsigned h_dist_tab[30] = SCN_DIST_TAB;
SCN_HD unsigned len_code(unsigned i) {
#ifdef __CUDA_ARCH__
  return c_len_tab[i];
#else
  return h_len_tab[i];
#endif
}
SCN_HD unsigned dist_code(unsigned i) {
#ifdef __CUDA_ARCH__
  return c_dist_tab[i];
#else
  return h_dist_tab[i];
#endif
}

template <int LANES>
SCN_HD void lanes_sync() {
#ifdef __CUDA_ARCH__
  if (LANES > 1) __syncwarp();
#endif
}

SCN_HD uint32_t make_entry(int mode, unsigned sym, unsigned len) {
  if (mode == M_PLAIN) return len | (K_LIT << 8) | (len << 10) | (sym << 16);
  if (mode == M_LITLEN) {
    if (sym < 256u) return len | (K_LIT << 8) | (len << 10) | (sym << 16);
    if (sym == 256u) return len | (K_EOB << 8) | (len << 10);
    if (sym > 285u) return len | (K_BAD << 8) | (len << 10);
    const unsigned lc = len_code(sym - 257u);
    return len | ((lc & 15u) << 4) | (K_BASE << 8) | ((len + (lc & 15u)) << 10) | ((lc >> 4) << 16);
  }
  if (sym > 29u) return len | (K_BAD << 8) | (len << 10);
  const unsigned dc = dist_code(sym);
  return len | ((dc & 15u) << 4) | (K_BASE << 8) | ((len + (dc & 15u)) << 10) | ((dc >> 4) << 16);
}

// canonical code from code lengths + the 9-bit lookahead table (filled by all lanes together); returns false for an
// over-subscribed set (incomplete sets are allowed, as in zlib for a single distance code)
template <int LANES, class Tab>
SCN_HD bool huff_build(Tab& h, const uint8_t* lens, int n, int lane, int mode) {
  // counted privately by every lane (a read-modify-write on the shared table would race between lanes); the shared copies
  // below are then written with identical values by all of them
  uint16_t cnt[16];
  for (int i = 0; i < 16; ++i) cnt[i] = 0;
  for (int i = 0; i < n; ++i) cnt[lens[i]]++;
  cnt[0] = 0;
  int left = 1; unsigned code = 0, off = 0;
  h.count[0] = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - (int)cnt[l];
    if (left < 0) return false;
    code = (code + cnt[l - 1]) << 1;
    h.count[l] = cnt[l]; h.first[l] = (uint16_t)code; h.offs[l] = (uint16_t)off; off += cnt[l];
  }
  constexpr int kFastBits = Tab::kBits; constexpr uint32_t kFastSize = 1u << kFastBits;
  for (int j = lane; j < (int)kFastSize; j += LANES) h.fast[j] = kLongCode;
  lanes_sync<LANES>();
  uint16_t nexti[16], nextc[16];
  { unsigned c2 = 0, o2 = 0; for (int l = 1; l < 16; ++l) { c2 = (c2 + cnt[l - 1]) << 1; nextc[l] = (uint16_t)c2; nexti[l] = (uint16_t)o2; o2 += cnt[l]; } }
  for (int i = 0; i < n; ++i) {
    const int l = lens[i];
    if (!l) continue;
    const unsigned c = nextc[l]++;
    h.sym[nexti[l]++] = (uint16_t)i;
    if (l <= kFastBits) {
      const unsigned r = rev_bits(c, l);
      const uint32_t e = make_entry(mode, (unsigned)i, (unsigned)l);
      for (unsigned j = r + ((unsigned)lane << l); j < kFastSize; j += (unsigned)LANES << l) h.fast[j] = e;
    }
  }
  return true;
}
// decode one symbol into a packed entry whose code bits are already consumed (caller guarantees >= 15 bits in the buffer:
// bi_refill leaves > 32); an invalid code gives kind K_BAD
template <class Tab>
SCN_HD uint32_t huff_decode(BitIn& b, const Tab& h, int mode) {
  constexpr int kFastBits = Tab::kBits;
  const uint32_t e = h.fast[bi_peek(b, kFastBits)];
  if (e != kLongCode) { bi_drop(b, (int)(e & 15u)); return e; }
  const unsigned r = rev_bits(bi_peek(b, 15), 15);
  for (int l = kFastBits + 1; l < 16; ++l) {
    const unsigned c = (r >> (15 - l)) - h.first[l];
    if (c < h.count[l]) { bi_drop(b, l); return make_entry(mode, h.sym[h.offs[l] + c], (unsigned)l); }
  }
  return K_BAD << 8;
}

enum { INF_OK = 0, INF_BAD_HEADER = 1, INF_BAD_BLOCK = 2, INF_BAD_CODE = 3, INF_BAD_DIST = 4, INF_OUT_FULL = 5, INF_TRUNCATED = 6 };

#ifdef __CUDA_ARCH__
// ---- device-only symbol loop ---------------------------------------------------------------------------------------------------
// A stream is ONE dependent chain of ~115-170 k symbols per frame, so what matters is the number of dependent instructions
// per symbol.  The generic reader above (64-bit buffer, byte-wise refill loop) cost ~120 instructions per symbol; this one is
// 32-bit throughout: three consecutive input words live in registers (the third loaded one word early), a funnel shift
// extracts the next 32 bits at the current bit offset, one table entry carries code length, extra-bit count, kind and base
// value, and literals / match lengths / distances are each decoded from a single peek.
struct FastBits {
  const uint32_t* p; uint32_t nwords, wi, w0, w1, w2, off;
  __device__ __forceinline__ uint32_t ld(uint32_t i) const { return i < nwords ? __ldg(p + i) : 0u; }
  __device__ __forceinline__ void init(const uint8_t* base, uint32_t n, uint32_t bitpos) {
    p = reinterpret_cast<const uint32_t*>(base); nwords = (n + 3u) >> 2; wi = bitpos >> 5; off = bitpos & 31u;
    w0 = ld(wi); w1 = ld(wi + 1); w2 = ld(wi + 2);
  }
  __device__ __forceinline__ uint32_t peek() const { return __funnelshift_r(w0, w1, off); }
  __device__ __forceinline__ void drop(uint32_t k) {                                       // k <= 28
    off += k;
    if (off >= 32u) { off -= 32u; w0 = w1; w1 = w2; ++wi; w2 = ld(wi + 2); }
  }
  __device__ __forceinline__ uint32_t bitpos() const { return (wi << 5) + off; }
};
// shared memory through 32-bit addresses (the generic-pointer form made ptxas re-derive the shared window per access)
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v)); }
template <class Tab>
__device__ __forceinline__ uint32_t long_code(const Tab& h, uint32_t win, int mode) {     // codes longer than the lookahead
  constexpr int kFastBits = Tab::kBits;
  const unsigned r = __brev(win & 0x7FFFu) >> 17;
  for (int l = kFastBits + 1; l < 16; ++l) {
    const unsigned c = (r >> (15 - l)) - h.first[l];
    if (c < h.count[l]) return make_entry(mode, h.sym[h.offs[l] + c], (unsigned)l);
  }
  return K_BAD << 8;
}
// symbols of one Huffman block until its end-of-block code.  Returns INF_OK at EOB, INF_OUT_FULL when the frame is complete.
// RING: the window is the shared-memory ring (+ a copy of every byte streamed to HBM); !RING: the window is the output in HBM.
// ~20 instructions per literal, ~50 per match: one table load per code, the kind tested on single bits in the order
// literal / match / rest, code length + extra bits pre-added in the entry, shared memory addressed with 32-bit registers.
// A stream that ends early decodes the zero padding; every exit reports INF_TRUNCATED when the reader is past the end.
template <bool RING>
__device__ __forceinline__ int inflate_block_fast(FastBits& fb, const InflateScratch& S, uint8_t* ring, uint8_t* out_in, uint32_t& o_io, uint32_t cap_in,
                                                  int lane, uint32_t nbits) {
  // A zero ptxas cannot see through: without it the shared-memory window base (S2UR SR_CgaCtaId + ULEA) and the stream's
  // output pointer (two IMADs of blockIdx and the stride) are re-derived for every symbol instead of being kept in registers.
  __shared__ volatile uint32_t s_zero;
  s_zero = 0u;
  __syncwarp();
  const uint32_t z = s_zero;
  const uint32_t s_lit = (uint32_t)__cvta_generic_to_shared(S.lit.fast) + z, s_dist = (uint32_t)__cvta_generic_to_shared(S.dist.fast) + z;
  const uint32_t s_ring = (RING ? (uint32_t)__cvta_generic_to_shared(ring) : 0u) + z;
  uint8_t* const out = out_in + z;
  const uint32_t cap = cap_in + z;
  uint32_t o = o_io;
  int rc;
  for (;;) {
    uint32_t win = fb.peek();
    uint32_t e = lds32(s_lit + ((win << 2) & (((1u << kLitBits) - 1u) << 2)));
  dispatch:
    if ((e & 0x300u) == 0u) {                                                                    // literal (every lane stores the same byte to the same place)
      if (o >= cap) { rc = INF_OUT_FULL; break; }
      fb.drop(e & 15u);
      const uint32_t v = e >> 16;
      if (RING) sts8(s_ring + (o & (kWin - 1u)), v);
      out[o] = (uint8_t)v;
      ++o;
      continue;
    }
    if ((e & 0x200u) != 0u) {                                                                    // end of block, bad code, or a code longer than the lookahead
      if (e == kLongCode) { e = long_code(S.lit, win, M_LITLEN); if (e != kLongCode) goto dispatch; }
      if (((e >> 8) & 3u) == K_EOB) { fb.drop(e & 15u); rc = INF_OK; break; }
      rc = INF_BAD_CODE; break;
    }
    // match: length = base + extra bits, i.e. bits [code length, code length + extra) of the window
    uint32_t len = (e >> 16) + ((win & ~(0xFFFFFFFFu << ((e >> 10) & 31u))) >> (e & 15u));        // code + extra bits <= 20
    fb.drop((e >> 10) & 31u);
    win = fb.peek();
    uint32_t d = lds32(s_dist + ((win << 2) & (((1u << kDistBits) - 1u) << 2)));
    if ((d & 0x300u) != (K_BASE << 8)) {
      if (d == kLongCode) d = long_code(S.dist, win, M_DIST);
      if ((d & 0x300u) != (K_BASE << 8)) { rc = INF_BAD_CODE; break; }
    }
    const uint32_t dist = (d >> 16) + ((win & ~(0xFFFFFFFFu << ((d >> 10) & 31u))) >> (d & 15u));   // code + extra bits <= 28
    fb.drop((d >> 10) & 31u);
    if (dist > o) { rc = INF_BAD_DIST; break; }
    const bool full = o + len > cap;
    if (full) len = cap - o;                                                                     // the caller's frame is complete: write what fits and stop
    __syncwarp();                                                                                // earlier literals / matches are visible to every lane
    const uint32_t so = o - dist;
    if (dist >= len) {
      uint32_t i = (uint32_t)lane;
      if (i < len) {
        uint32_t v;
        if (RING) { v = lds8(s_ring + ((so + i) & (kWin - 1u))); sts8(s_ring + ((o + i) & (kWin - 1u)), v); } else v = out[so + i];
        out[o + i] = (uint8_t)v;
      }
      if (len > 32u) {
#pragma unroll 1
        for (i += 32u; i < len; i += 32u) {
          uint32_t v;
          if (RING) { v = lds8(s_ring + ((so + i) & (kWin - 1u))); sts8(s_ring + ((o + i) & (kWin - 1u)), v); } else v = out[so + i];
          out[o + i] = (uint8_t)v;
        }
      }
    } else {
#pragma unroll 1
      for (uint32_t i = (uint32_t)lane; i < len; i += 32u) {
        const uint32_t k = (dist & (dist - 1u)) == 0u ? (i & (dist - 1u)) : i % dist;
        uint32_t v;
        if (RING) { v = lds8(s_ring + ((so + k) & (kWin - 1u))); sts8(s_ring + ((o + i) & (kWin - 1u)), v); } else v = out[so + k];
        out[o + i] = (uint8_t)v;
      }
    }
    o += len;
    if (full) { rc = INF_OUT_FULL; break; }
  }
  o_io = o;
  __syncwarp();
  if (fb.bitpos() > nbits) rc = INF_TRUNCATED;
  return rc;
}
#endif

// Inflates one zlib stream.  Every lane executes this with identical arguments except `lane`; the output is written
// cooperatively.  Returns INF_* and the number of bytes produced.
template <int LANES, bool RING>
SCN_HD int inflate_zlib(const uint8_t* in, size_t n_in, uint8_t* out, size_t cap_in, int lane, InflateScratch* scr, size_t* produced) {
  *produced = 0;
  if (n_in < 2 || n_in > 0xFFFFFFF0ull || cap_in > 0xFFFFFFF0ull) return INF_BAD_HEADER;
  const uint32_t n = (uint32_t)n_in, cap = (uint32_t)cap_in;
  const unsigned cmf = in[0], flg = in[1];
  if ((cmf & 15u) != 8u || ((cmf << 8) | flg) % 31u != 0u || (flg & 32u)) return INF_BAD_HEADER;     // RFC 1950; preset dictionaries are not used
  BitIn b{in, n, 2, 0ull, 0, 0, 0u, 0};
  InflateScratch& S = SCN_SCR(scr);
  uint32_t o = 0;
  // device: every output byte goes to the shared-memory ring (what later matches read) and to HBM; host: straight to `out`
#ifdef __CUDA_ARCH__
  uint8_t* const ring = RING ? SCN_RING : nullptr;
#define SCN_PUT(idx, v) do { const uint8_t v_ = (v); if (RING) ring[(idx) & (kWin - 1u)] = v_; out[(idx)] = v_; } while (0)
#define SCN_WIN(idx) (RING ? ring[(idx) & (kWin - 1u)] : out[(idx)])
#else
#define SCN_PUT(idx, v) out[(idx)] = (v)
#define SCN_WIN(idx) out[(idx)]
#endif
  for (;;) {
    bi_refill(b);
    const unsigned last = bi_get(b, 1), type = bi_get(b, 2);
    if (type == 0) {                                             // stored
      bi_drop(b, b.bc & 7);
      bi_refill(b);
      const unsigned len = bi_get(b, 16), nlen = bi_get(b, 16);
      if ((len ^ 0xFFFFu) != nlen || bi_overrun(b)) return INF_BAD_BLOCK;
      // the bytes still in the bit buffer come first, then straight from the input
      const uint32_t src0 = b.pos - (uint32_t)((b.bc - b.over) / 8);   // (a word held in `ahead` has not advanced b.pos)
      if (src0 + len > n) return INF_TRUNCATED;
      const uint32_t take = o + len > cap ? cap - o : len;
      lanes_sync<LANES>();
      for (uint32_t i = (uint32_t)lane; i < take; i += LANES) SCN_PUT(o + i, in[src0 + i]);
      o += take;
      if (take < len) { lanes_sync<LANES>(); *produced = o; return INF_OUT_FULL; }
      bi_restart(b, src0 + len);
    } else if (type == 1 || type == 2) {
      if (type == 2) {
        bi_refill(b);
        const int hlit = (int)bi_get(b, 5) + 257, hdist = (int)bi_get(b, 5) + 1, hclen = (int)bi_get(b, 4) + 4;
        if (hlit > 286 || hdist > 30) return INF_BAD_BLOCK;
        const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        uint8_t cl[19];
        for (int i = 0; i < 19; ++i) cl[i] = 0;
        for (int i = 0; i < hclen; ++i) { bi_refill(b); cl[order[i]] = (uint8_t)bi_get(b, 3); }
        lanes_sync<LANES>();                                      // previous block's tables are dead for every lane
        if (!huff_build<LANES>(S.lit, cl, 19, lane, M_PLAIN)) return INF_BAD_BLOCK;  // code-length code lives in the lit table for a moment
        lanes_sync<LANES>();
        int idx = 0;
        uint8_t* lens = S.lens;
        uint8_t prev = 0, eob_len = 0;
        while (idx < hlit + hdist) {
          bi_refill(b);
          const uint32_t ce = huff_decode(b, S.lit, M_PLAIN);
          if (((ce >> 8) & 3u) != K_LIT) return INF_BAD_CODE;
          const int s = (int)(ce >> 16);
          // `prev` and `eob_len` live in registers: every lane writes the same bytes to the shared array, nobody reads it here
          if (s < 16) { if (idx == 256) eob_len = (uint8_t)s; lens[idx++] = prev = (uint8_t)s; continue; }
          int rep; uint8_t v = 0;
          if (s == 16) { if (idx == 0) return INF_BAD_BLOCK; v = prev; rep = 3 + (int)bi_get(b, 2); }
          else if (s == 17) rep = 3 + (int)bi_get(b, 3);
          else rep = 11 + (int)bi_get(b, 7);
          if (idx + rep > hlit + hdist) return INF_BAD_BLOCK;
          if (idx <= 256 && 256 < idx + rep) eob_len = v;
          prev = v;
          while (rep--) lens[idx++] = v;
        }
        if (eob_len == 0) return INF_BAD_BLOCK;
        lanes_sync<LANES>();
        if (!huff_build<LANES>(S.lit, lens, hlit, lane, M_LITLEN) || !huff_build<LANES>(S.dist, lens + hlit, hdist, lane, M_DIST)) return INF_BAD_BLOCK;
        lanes_sync<LANES>();
      } else {                                                    // fixed code (RFC 1951 3.2.6) through the same tables: every code is <= 9 bits
        uint8_t* lens = S.lens;
        lanes_sync<LANES>();
        for (int i = lane; i < 320; i += LANES) lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
        lanes_sync<LANES>();
        huff_build<LANES>(S.lit, lens, 288, lane, M_LITLEN); huff_build<LANES>(S.dist, lens + 288, 30, lane, M_DIST);
        lanes_sync<LANES>();
      }
#ifdef __CUDA_ARCH__
      if (LANES == 32 && (((size_t)in) & 3u) == 0u) {                 // the lean 32-bit symbol loop (streams are packed at 16-byte offsets)
        if (b.over > 0) return INF_TRUNCATED;
        FastBits fb;
        fb.init(in, n, 8u * b.pos - (uint32_t)b.bc);                 // bytes before b.pos are in the bit buffer, b.bc of their bits still unread
        const int frc = inflate_block_fast<RING>(fb, S, ring, out, o, cap, lane, 8u * n);
        if (frc != INF_OK) { lanes_sync<LANES>(); *produced = o; return frc; }
        const uint32_t bp = fb.bitpos();
        if (bp > 8u * n) return INF_TRUNCATED;
        bi_restart(b, bp >> 3); bi_refill(b); bi_drop(b, (int)(bp & 7u));
        if (last) break;
        continue;
      }
#endif
      for (;;) {
        bi_refill(b);
        const uint32_t e = huff_decode(b, S.lit, M_LITLEN);
        const unsigned kind = (e >> 8) & 3u;
        if (kind == K_LIT) {
          if (o >= cap) { lanes_sync<LANES>(); *produced = o; return bi_overrun(b) ? INF_TRUNCATED : INF_OUT_FULL; }   // (zero padding past a truncated stream decodes as literals)
          if (lane == 0) SCN_PUT(o, (uint8_t)(e >> 16));
          ++o;
          continue;
        }
        if (kind == K_EOB) break;
        if (kind == K_BAD) return bi_overrun(b) ? INF_TRUNCATED : INF_BAD_CODE;
        unsigned len = (e >> 16) + bi_get(b, (int)((e >> 4) & 15u));
        bi_refill(b);
        const uint32_t d = huff_decode(b, S.dist, M_DIST);
        if (((d >> 8) & 3u) != K_BASE) return bi_overrun(b) ? INF_TRUNCATED : INF_BAD_CODE;
        const unsigned dist = (d >> 16) + bi_get(b, (int)((d >> 4) & 15u));
        if (bi_overrun(b)) return INF_TRUNCATED;
        if (dist > o) return INF_BAD_DIST;
        const bool full = o + len > cap;
        if (full) len = (unsigned)(cap - o);                      // the caller's frame is complete: write what fits and stop
        lanes_sync<LANES>();                                      // earlier literals / matches are visible to every lane
        const uint32_t so = o - dist;
        if (dist >= len) { for (unsigned i = (unsigned)lane; i < len; i += LANES) SCN_PUT(o + i, SCN_WIN(so + i)); }
        else if ((dist & (dist - 1u)) == 0u) { for (unsigned i = (unsigned)lane; i < len; i += LANES) SCN_PUT(o + i, SCN_WIN(so + (i & (dist - 1u)))); }
        else { for (unsigned i = (unsigned)lane; i < len; i += LANES) SCN_PUT(o + i, SCN_WIN(so + i % dist)); }
        o += len;
        if (full) { lanes_sync<LANES>(); *produced = o; return INF_OUT_FULL; }
      }
      if (bi_overrun(b)) return INF_TRUNCATED;
    } else return INF_BAD_BLOCK;
    if (last) break;
  }
  lanes_sync<LANES>();
  *produced = o;
  return INF_OK;                                                  // the Adler-32 trailer is not checked (stb_image does not either)
#undef SCN_PUT
#undef SCN_WIN
}

// one warp per stream
template <bool RING>
__global__ void __launch_bounds__(32) k_inflate(const uint8_t* __restrict__ in, const unsigned long long* __restrict__ in_off, uint8_t* out,
                                                  size_t out_stride, size_t out_cap, unsigned n, int* __restrict__ status,
                                                  unsigned long long* __restrict__ produced) {
  const unsigned s = blockIdx.x;
  if (s >= n) return;
  size_t got = 0;
  const int rc = inflate_zlib<32, RING>(in + in_off[s], (size_t)(in_off[s + 1] - in_off[s]), out + (size_t)s * out_stride, out_cap, (int)threadIdx.x, nullptr, &got);
  if (threadIdx.x == 0) { status[s] = rc; produced[s] = got; }
}

const char* inf_msg(int rc) {
  switch (rc) {
    case INF_BAD_HEADER: return "bad zlib header"; case INF_BAD_BLOCK: return "bad deflate block"; case INF_BAD_CODE: return "invalid Huffman code";
    case INF_BAD_DIST: return "match distance before start of output"; case INF_OUT_FULL: return "stream longer than the frame"; case INF_TRUNCATED: return "truncated stream";
    default: return "ok";
  }
}

// cached staging, one per calling thread: two 64 MB pinned slices (cudaHostAlloc costs ~0.2 ms per MB, so the pinned part is
// bounded and reused), a device buffer for the packed streams, per-stream offsets / status / produced counts
constexpr size_t kSlice = size_t(64) << 20;
struct InflateStage {
  int device = 0;
  scn::PinnedPtr<uint8_t> h[2]; scn::EventPtr ev[2];
  scn::EventPtr tk[2];                               // timing events around the kernel
  scn::DBuf d; size_t cap = 0;
  scn::DBuf d_off, d_status, d_prod; size_t ncap = 0;   // unsigned long long, int, unsigned long long
  void release() {
    for (int i = 0; i < 2; ++i) { h[i].reset(); ev[i].reset(); tk[i].reset(); }
    d.reset(); d_off.reset(); d_status.reset(); d_prod.reset(); cap = ncap = 0;
  }
  bool ensure(size_t bytes, size_t n) {
    for (int i = 0; i < 2; ++i) if (!h[i]) {
      if (scn::create(h[i], kSlice) != cudaSuccess || scn::create(ev[i], cudaEventDisableTiming) != cudaSuccess ||
          scn::create(tk[i]) != cudaSuccess) { cudaGetLastError(); release(); return false; }
    }
    if (bytes > cap) {                               // a failed allocation calls release(), which zeroes cap and ncap
      const size_t want = bytes + (bytes >> 2) + 4096;
      if (!d.alloc(want)) { release(); return false; }
      cap = want;
    }
    if (n > ncap) {
      d_off.reset(); d_status.reset(); d_prod.reset();
      const size_t want = n + (n >> 2) + 64;
      if (!d_off.alloc((want + 1) * 8) || !d_status.alloc(want * 4) || !d_prod.alloc(want * 8)) { release(); return false; }
      ncap = want;
    }
    return true;
  }
};
scn::StagePool<InflateStage>& inflate_pool() { static auto* p = new scn::StagePool<InflateStage>(); return *p; }
struct InflateTimings { double pack_s = 0, kernel_ms = 0; int ring = 0; unsigned n = 0; };
thread_local InflateTimings g_last;

}  // namespace

extern "C" {

// Host build of the same decoder (lanes = 1): unit-test hook for the CPU suite.
int scn_inflate_host(const uint8_t* src, size_t n, uint8_t* out, size_t cap, size_t* produced) {
  if (!src || !out || !produced) return scn::fail(SCN_ERR_ARG, "null argument");
  std::vector<InflateScratch> scr(1);
  const int rc = inflate_zlib<1, false>(src, n, out, cap, 0, scr.data(), produced);
  return rc == INF_OK ? SCN_OK : scn::fail(SCN_ERR_FORMAT, "inflate: %s", inf_msg(rc));
}

// n zlib streams (host pointers) -> n frames of `frame_bytes` each at d_out (device).  Streams are packed back to back
// (16-byte aligned starts) through two pinned 64 MB slices filled by a few host threads and uploaded while the next slice
// is being filled, then inflated by one warp each in a single launch.  Every stream must produce at least frame_bytes (the
// first frame_bytes are kept, as the host path does).  `stream` = cudaStream_t (0 = default); returns after the kernel
// has completed.
int scn_inflate_batch_device(const uint8_t* const* src, const uint64_t* src_bytes, uint32_t n, uint64_t frame_bytes, void* d_out, void* stream) {
  if (!n) return SCN_OK;
  if (!src || !src_bytes || !d_out) return scn::fail(SCN_ERR_ARG, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const double t_call = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  std::vector<unsigned long long> off((size_t)n + 1);
  size_t tot = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (src_bytes[i] && !src[i]) return scn::fail(SCN_ERR_ARG, "null stream %u", i);
    if (src_bytes[i] + 16 > kSlice) return scn::fail(SCN_ERR_ARG, "stream %u: %llu bytes is larger than a staging slice", i, (unsigned long long)src_bytes[i]);
    off[i] = tot; tot += ((size_t)src_bytes[i] + 15) & ~size_t(15);
  }
  off[n] = tot;
  scn::StagePool<InflateStage>::Lease lease(inflate_pool());
  InflateStage& g = *lease;
  if (!g.ensure(tot + 16, n)) return scn::fail(SCN_ERR_CUDA, "scn_inflate_batch_device: allocation of %zu staging bytes failed", tot);
  cudaError_t e = cudaMemcpyAsync(g.d_off.as<unsigned long long>(), off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, st);
  const unsigned nt = std::max(1u, std::min(24u, std::thread::hardware_concurrency()));     // packing is a 2-3 GB memcpy per scan: spread it
  int slot = 0; bool used[2] = {false, false};
  for (uint32_t i0 = 0; i0 < n && e == cudaSuccess;) {
    uint32_t i1 = i0; while (i1 < n && off[i1 + 1] - off[i0] <= kSlice) ++i1;               // streams [i0, i1) fit one slice
    if (used[slot]) e = cudaEventSynchronize(g.ev[slot].get());                             // its previous upload has left the pinned slice
    if (e != cudaSuccess) break;
    uint8_t* hs = g.h[slot].get(); const size_t base = off[i0];
    auto fill = [&](unsigned t) {
      for (uint32_t i = i0 + t; i < i1; i += nt) {
        if (src_bytes[i]) memcpy(hs + (off[i] - base), src[i], (size_t)src_bytes[i]);
        memset(hs + (off[i] - base) + src_bytes[i], 0, (size_t)(off[i + 1] - off[i] - src_bytes[i]));   // padding is never decoded, but keep it defined
      }
    };
    if (i1 - i0 >= 4 * nt && nt > 1) { std::vector<std::thread> pool; for (unsigned t = 1; t < nt; ++t) pool.emplace_back(fill, t); fill(0); for (auto& th : pool) th.join(); }
    else for (unsigned t = 0; t < nt; ++t) fill(t);
    e = cudaMemcpyAsync(g.d.as<uint8_t>() + base, hs, (size_t)(off[i1] - base), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaEventRecord(g.ev[slot].get(), st);
    used[slot] = true; slot ^= 1; i0 = i1;
  }
  std::vector<int> status(n); std::vector<unsigned long long> prod(n);
  const double t_packed = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  // Window placement.  Shared-memory ring: ~2.5x lower latency per stream, but 38.5 KB per stream = 5 streams per SM; window in
  // HBM (matches read the output back through L2): 32 streams per SM.  Up to about two waves of ring streams the ring wins.
  static const int n_sm = []() { int d = 0, v = 132; if (cudaGetDevice(&d) == cudaSuccess) cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d); return v; }();
  const char* wenv = getenv("SCN_INFLATE_WINDOW");
  const bool use_ring = wenv ? !strcmp(wenv, "ring") : n <= (uint32_t)(5 * n_sm);      // at most one wave of ring streams
  if (e == cudaSuccess) {
    cudaEventRecord(g.tk[0].get(), st);
    if (use_ring) k_inflate<true><<<n, 32, sizeof(InflateScratchDev), st>>>(g.d.as<uint8_t>(), g.d_off.as<unsigned long long>(), (uint8_t*)d_out, (size_t)frame_bytes, (size_t)frame_bytes, n, g.d_status.as<int>(), g.d_prod.as<unsigned long long>());
    else k_inflate<false><<<n, 32, sizeof(InflateScratch), st>>>(g.d.as<uint8_t>(), g.d_off.as<unsigned long long>(), (uint8_t*)d_out, (size_t)frame_bytes, (size_t)frame_bytes, n, g.d_status.as<int>(), g.d_prod.as<unsigned long long>());
    cudaEventRecord(g.tk[1].get(), st);
    e = cudaMemcpyAsync(status.data(), g.d_status.as<int>(), (size_t)n * 4, cudaMemcpyDeviceToHost, st);
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(prod.data(), g.d_prod.as<unsigned long long>(), (size_t)n * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return scn::fail(SCN_ERR_CUDA, "scn_inflate_batch_device: %s", cudaGetErrorString(e));
  { float ms = 0; if (cudaEventElapsedTime(&ms, g.tk[0].get(), g.tk[1].get()) == cudaSuccess) g_last.kernel_ms = ms; g_last.pack_s = t_packed - t_call; g_last.ring = use_ring; g_last.n = n; }
  for (uint32_t i = 0; i < n; ++i) {
    if (status[i] != INF_OK && status[i] != INF_OUT_FULL) return scn::fail(SCN_ERR_FORMAT, "frame %u: corrupt zlib depth stream (%s)", i, inf_msg(status[i]));
    if (prod[i] < frame_bytes) return scn::fail(SCN_ERR_FORMAT, "frame %u: depth stream holds %llu bytes, need %llu", i, prod[i], (unsigned long long)frame_bytes);
  }
  return SCN_OK;
}

// timings of the last scn_inflate_batch_device call of this thread: host packing + upload issue (s), inflate kernel (ms, CUDA
// events), whether the shared-memory-window kernel ran, streams in the launch
void scn_inflate_release_staging_() { inflate_pool().trim(); }

int scn_inflate_last_timings(double* pack_s, double* kernel_ms, int* ring_window, uint32_t* n_streams) {
  if (pack_s) *pack_s = g_last.pack_s;
  if (kernel_ms) *kernel_ms = g_last.kernel_ms;
  if (ring_window) *ring_window = g_last.ring;
  if (n_streams) *n_streams = g_last.n;
  return SCN_OK;
}

// Frames [first, first+n) of an open .sens stream decoded straight into device memory (u16 depth, row-major, frame after
// frame).  TYPE_ZLIB_USHORT goes through the GPU inflate; TYPE_RAW_USHORT is a plain upload.
int scn_sens_decode_depth_device(const scn_sens* s, uint64_t first, uint32_t n, uint16_t* d_depth_out, void* stream) {
  if (!s || (!d_depth_out && n)) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_sens_info_t info;
  if (int rc = scn_sens_info(s, &info)) return rc;
  if (first + n > info.n_frames) return scn::fail(SCN_ERR_ARG, "out of bounds");
  std::vector<uint64_t> frames(n);
  for (uint32_t i = 0; i < n; ++i) frames[i] = first + i;
  return scn::sens_depth_to_device(s, frames.data(), n, d_depth_out, stream);
}

}  // extern "C"

int scn::sens_depth_to_device(const scn_sens* s, const uint64_t* frames, uint32_t n, uint16_t* d_out, void* stream) {
  scn_sens_info_t info;
  if (int rc = scn_sens_info(s, &info)) return rc;
  if (info.depth_compression == 2) return scn::fail(SCN_ERR_UNSUPPORTED, "need UPLINK_COMPRESSION");
  if (info.depth_compression != 0 && info.depth_compression != 1) return scn::fail(SCN_ERR_FORMAT, "invalid type");
  const uint64_t fb = (uint64_t)info.depth_width * info.depth_height * 2;
  std::vector<const uint8_t*> src(n); std::vector<uint64_t> len(n);
  for (uint32_t i = 0; i < n; ++i) {
    if (int rc = scn_sens_frame_payload(s, frames[i], nullptr, &src[i])) return rc;
    if (int rc = scn_sens_frame_meta(s, frames[i], nullptr, nullptr, nullptr, nullptr, &len[i])) return rc;
    if (info.depth_compression == 0 && len[i] < fb)
      return scn::fail(SCN_ERR_FORMAT, "frame %llu: raw depth payload of %llu bytes, need %llu", (unsigned long long)frames[i],
                       (unsigned long long)len[i], (unsigned long long)fb);
  }
  if (info.depth_compression == 1) return scn_inflate_batch_device(src.data(), len.data(), n, fb, d_out, stream);
  cudaStream_t st = (cudaStream_t)stream;
  for (uint32_t i = 0; i < n; ++i) SCN_CUDA_TRY(cudaMemcpyAsync((uint8_t*)d_out + (size_t)i * fb, src[i], fb, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}
