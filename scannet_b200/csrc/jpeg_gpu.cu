// Colour decode on the GPU (SURVEY.md §8a R4): the TYPE_JPEG payloads of a .sens stream
// (SensReader/c++/src/sensorData.h:609-616 -> stbi_load_from_memory, 3 channels) are uploaded COMPRESSED and decoded in HBM,
// byte-identical to stb_image v2.08 (the numerics restated in jpeg.cpp: de-quantisation truncated to int16
// stb_image.h:1735,1764; integer "islow" IDCT :1928-2027; chroma up-sampling :2871-2925 incl. its end-of-row quirk; 20-bit
// fixed-point YCbCr->RGB with the masked Cb term :3091-3118).
//
//   host    parse the markers of every frame (SOF / DQT / DHT / DRI / SOS), build the Huffman lookup tables once per distinct
//           table set (a stream normally has one), pack the payloads into pinned slices and upload them;
//   k_jpeg_entropy_idct   ONE WARP PER FRAME: the entropy-coded segment is a single bit-serial chain (there are no
//           synchronisation points without restart markers), so all 32 lanes run the same bit reader and Huffman decoder
//           redundantly (broadcast loads, no divergence); after each MCU (up to 6 blocks) the warp does the IDCT of all its
//           blocks at once out of shared memory - one lane per column, then one lane per row, 32 of the 48 columns / rows of
//           a 4:2:0 MCU per step, bank-conflict-free through padding - and stores the rows into the component planes in
//           HBM.  The parallelism is across frames: a scan is thousands of frames, ~14 KB of shared memory per warp;
//   k_jpeg_color          fully parallel: chroma up-sampling + YCbCr->RGB per output pixel, either the whole frame (RGB8) or only
//           the colour pixels the depth image needs (a depth-pixel -> colour-pixel map), so that a 1296x968 frame feeding a
//           640x480 integration never materialises at full resolution.
// Supported on the device: baseline / extended-sequential Huffman JPEG (SOF0 / SOF1), 8 bit, 1 or 3 components in ONE
// interleaved scan, luma sampling (hmax, vmax) in {1,2}^2 with 1x1 chroma, table ids 0-1, restart intervals.  Anything
// else (progressive, multi-scan, exotic sampling) and every frame the device flags as corrupt is decoded by the host
// decoder (jpeg.cpp) and uploaded - same bytes, same errors.
#include <algorithm>
#include <chrono>
#include <thread>
#include <vector>

#include "jpeg_common.h"
#include "scn_common.h"
#include "stage_pool.h"

namespace {

using namespace scn_jpeg;

struct TableSet { HuffTab dc[2], ac[2]; uint8_t quant[4][64]; uint8_t have_q[4]; uint8_t pad[12]; };
static_assert(sizeof(TableSet) % 16 == 0, "TableSet is copied to shared memory in 16-byte pieces");

struct FrameDesc {
  unsigned long long src_off;       // start of this frame's JPEG in the packed input buffer
  unsigned scan_start, n_bytes;     // entropy-coded data starts here; total payload bytes
  unsigned table_set;
  unsigned restart;
  unsigned mcux, mcuy;
  unsigned short W, H;
  unsigned char ncomp, hmax, vmax, supported;
  unsigned char ch[3], cv[3], tq[3], td[3], ta[3], pad_;
  unsigned w2[3], h2[3], cy[3];     // padded plane size, real chroma rows (stb clamps the far row to them)
  unsigned plane_off[3];            // byte offset of each plane inside the frame's plane buffer
  unsigned pad2_;
};
static_assert(sizeof(FrameDesc) % 8 == 0, "FrameDesc is copied word by word");

__constant__ unsigned char c_zig[64 + 15] = SCN_JPEG_ZIG;

// MSB-first bit reader over the entropy-coded segment, same bit stream as jpeg.cpp's `Bits` (byte stuffing removed, a marker
// stops the input: zero bits from then on) - but the stuffing is removed by the WHOLE WARP, 32 raw bytes per step (ballot +
// prefix count compaction into a 1 KB ring in shared memory), so the bit-serial chain only ever sees clean big-endian words:
// one funnel shift per peek, one shared-memory load per 32 bits.  The first version (byte-wise refill with the FF test on
// the dependent chain) cost ~600 cycles per symbol.
constexpr unsigned kCleanRing = 1024;
constexpr int kMaxMcuBlocks = 6;           // 4 luma (2x2) + 2 chroma: the largest MCU the device path accepts
struct CleanBits {
  const unsigned char* p; unsigned n;       // raw stream
  unsigned char* ring;                      // shared memory, kCleanRing bytes, 4-byte aligned
  unsigned raw_pos;                         // next raw byte to stage
  unsigned fill, used;                      // clean bytes staged / fetched so far (monotone)
  unsigned w0, w1, off;                     // the two big-endian words at the read position, bit offset into w0
  unsigned last_raw;                        // raw byte before raw_pos (an FF there makes a following 00 a stuffed byte)
  unsigned marker_pos; bool marker;         // a marker (FF xx, xx != 0) stopped the staging at marker_pos
  int lane;

  __device__ __forceinline__ void stage32() {          // all lanes: up to 32 raw bytes -> ring
    const unsigned r = raw_pos + (unsigned)lane;
    const bool valid = r < n;
    const unsigned b = valid ? (unsigned)__ldg(p + r) : 0x100u;
    unsigned nxt = __shfl_down_sync(0xffffffffu, b, 1);
    if (lane == 31) nxt = r + 1 < n ? (unsigned)__ldg(p + r + 1) : 0xD9u;
    if (valid && r + 1 >= n) nxt = 0xD9u;                // the host treats the byte after the last one as EOI
    unsigned prv = __shfl_up_sync(0xffffffffu, b, 1);
    if (lane == 0) prv = last_raw;
    const bool is_mark = valid && b == 0xFFu && nxt != 0u;
    const bool is_stuff = valid && b == 0u && prv == 0xFFu;
    const unsigned mm = __ballot_sync(0xffffffffu, is_mark);
    const unsigned first = mm ? (unsigned)__ffs(mm) - 1u : 32u;
    const unsigned nvalid = min(32u, n - raw_pos);
    const unsigned stop = min(first, nvalid);
    const bool emit = (unsigned)lane < stop && !is_stuff;
    const unsigned em = __ballot_sync(0xffffffffu, emit);
    if (emit) ring[(fill + __popc(em & ((1u << lane) - 1u))) & (kCleanRing - 1u)] = (unsigned char)b;
    fill += __popc(em);
    if (stop) last_raw = __shfl_sync(0xffffffffu, b, (int)stop - 1);
    raw_pos += stop;
    if (first < nvalid) { marker = true; marker_pos = raw_pos; }
    __syncwarp();
  }
  __device__ __forceinline__ void refill() {           // keep the ring ahead of the reader
    while (!marker && raw_pos < n && (int)(fill - used) <= (int)(kCleanRing - 64u)) stage32();
  }
  __device__ __forceinline__ unsigned fetch() {        // next 4 clean bytes, big endian; zeros past a marker / the end
    if ((int)(fill - used) < 4) refill();
    unsigned w;
    if ((int)(fill - used) >= 4) w = __byte_perm(*reinterpret_cast<const unsigned*>(ring + (used & (kCleanRing - 1u))), 0u, 0x0123);
    else {
      w = 0u;
      for (int i = 0; i < 4; ++i) if ((int)(fill - used) > i) w |= (unsigned)ring[(used + i) & (kCleanRing - 1u)] << (24 - 8 * i);
    }
    used += 4u;
    return w;
  }
  __device__ __forceinline__ void start(unsigned at) {
    raw_pos = at; fill = used = 0u; last_raw = 0u; marker = false; marker_pos = 0u; off = 0u;
    refill();
    w0 = fetch(); w1 = fetch();
  }
  __device__ __forceinline__ unsigned peek() const { return __funnelshift_l(w1, w0, off); }      // 32 bits at the read position
  __device__ __forceinline__ void consume(unsigned k) {                                           // k <= 16
    off += k;
    if (off >= 32u) { off -= 32u; w0 = w1; w1 = fetch(); }
  }
  __device__ __forceinline__ int get(int k) { if (k == 0) return 0; const int v = (int)(peek() >> (32 - k)); consume((unsigned)k); return v; }
  __device__ __forceinline__ int decode(const HuffTab& h) {
    const unsigned pk = peek();
    const unsigned e = h.fast[pk >> (32 - kFastBits)];
    if (e != 0xFFFFu) { consume(e & 15u); return (int)(e >> 4); }
    for (int l = 1; l <= 16; ++l) {                     // jpeg.cpp consumes these bits one at a time: same codes, same count
      const int code = (int)(pk >> (32 - l));
      if (h.maxcode[l] >= 0 && code <= h.maxcode[l] && code >= h.mincode[l]) { consume((unsigned)l); return h.vals[h.valptr[l] + code - h.mincode[l]]; }
    }
    consume(16u);
    return -1;
  }
  // restart interval boundary (jpeg.cpp: handle_restart).  Returns 1 = continue after RSTn, 0 = the scan ends here
  // (as the host decoder decides when no RSTn follows).
  __device__ __forceinline__ int restart() {
    while (!marker && raw_pos < n) { fill = used; stage32(); }                                   // discard up to the next marker
    if (!marker || marker_pos + 1 >= n) return 0;
    const unsigned m = __ldg(p + marker_pos + 1);
    if (m < 0xD0u || m > 0xD7u) return 0;
    start(marker_pos + 2u);
    return 1;
  }
  __device__ __forceinline__ unsigned end_pos() const { return marker ? marker_pos : raw_pos; }
};

enum { JST_OK = 0, JST_UNSUPPORTED = 1, JST_BAD_CODE = 2, JST_BAD_RESTART = 3 };

// one warp per frame
__global__ void __launch_bounds__(32)
k_jpeg_entropy_idct(const unsigned char* __restrict__ in, const FrameDesc* __restrict__ fd, const TableSet* __restrict__ sets,
                    unsigned char* __restrict__ planes, size_t plane_stride, int* __restrict__ status, unsigned* __restrict__ end_pos) {
  __shared__ __align__(16) TableSet S;
  // padded so that the 32 lanes of an IDCT pass (4 blocks x 8 columns / rows) hit 32 different banks: coefficient blocks 72
  // shorts apart, intermediate rows 9 ints apart
  __shared__ __align__(16) short s_blk[kMaxMcuBlocks][72];
  __shared__ int s_val[kMaxMcuBlocks][72];
  __shared__ unsigned s_bk[kMaxMcuBlocks];               // block b of an MCU: component | row << 8 | column << 16
  __shared__ __align__(16) FrameDesc s_fd;
  __shared__ __align__(16) unsigned char s_ring[kCleanRing];
  const int lane = threadIdx.x;
  {
    const unsigned* src = reinterpret_cast<const unsigned*>(fd + blockIdx.x);
    unsigned* dst = reinterpret_cast<unsigned*>(&s_fd);
    for (int i = lane; i < (int)(sizeof(FrameDesc) / 4); i += 32) dst[i] = src[i];
  }
  __syncwarp();
  const FrameDesc& f = s_fd;
  if (!f.supported) { if (lane == 0) { status[blockIdx.x] = JST_UNSUPPORTED; end_pos[blockIdx.x] = 0; } return; }
  {
    const uint4* src = reinterpret_cast<const uint4*>(sets + f.table_set);
    uint4* dst = reinterpret_cast<uint4*>(&S);
    for (int i = lane; i < (int)(sizeof(TableSet) / 16); i += 32) dst[i] = src[i];
  }
  const int ncomp = f.ncomp;
  int nb = 0;
  for (int k = 0; k < ncomp; ++k) for (int by = 0; by < f.cv[k]; ++by) for (int bx = 0; bx < f.ch[k]; ++bx) { if (lane == 0 && nb < kMaxMcuBlocks) s_bk[nb] = (unsigned)k | ((unsigned)by << 8) | ((unsigned)bx << 16); ++nb; }
  __syncwarp();
  if (nb > kMaxMcuBlocks) { if (lane == 0) { status[blockIdx.x] = JST_UNSUPPORTED; end_pos[blockIdx.x] = 0; } return; }   // (parse_frame only passes samplings with <= 6 blocks)
  const unsigned char* d = in + f.src_off;
  unsigned char* pl = planes + (size_t)blockIdx.x * plane_stride;
  CleanBits br;
  br.p = d; br.n = f.n_bytes; br.ring = s_ring; br.lane = lane;
  br.start(f.scan_start);
  int dc0 = 0, dc1 = 0, dc2 = 0;                         // DC predictors (selects, not an indexed array: that lives in local memory)
  int todo = f.restart ? (int)f.restart : 0x7fffffff;
  int rc = JST_OK;
  for (unsigned my = 0; my < f.mcuy && rc == JST_OK; ++my) {
    for (unsigned mx = 0; mx < f.mcux && rc == JST_OK; ++mx) {
      // ---- entropy decode of the MCU's blocks (jpeg.cpp: decode_block; stb_image.h:1719-1770), every lane the same
      for (int w = lane; w < nb * 36; w += 32) reinterpret_cast<unsigned*>(s_blk)[w] = 0u;
      __syncwarp();
      int b = 0;
      for (int k = 0; k < ncomp && rc == JST_OK; ++k) {
        const HuffTab& hd = S.dc[f.td[k]];
        const HuffTab& ha = S.ac[f.ta[k]];
        const unsigned char* q = S.quant[f.tq[k]];
        const int nbk = f.cv[k] * f.ch[k];
        for (int j = 0; j < nbk; ++j, ++b) {
          short* blk = s_blk[b];
          const int t = br.decode(hd);
          if (t < 0 || t > 16) { rc = JST_BAD_CODE; break; }
          const int diff = t ? extend(br.get(t), t) : 0;
          const int dc = (k == 0 ? dc0 : k == 1 ? dc1 : dc2) + diff;
          if (k == 0) dc0 = dc; else if (k == 1) dc1 = dc; else dc2 = dc;
          if (lane == 0) blk[0] = (short)(dc * q[0]);
          for (int kk = 1; kk < 64;) {
            const int fa = ha.fast_ac[br.peek() >> (32 - kFastBits)];
            if (fa) {                                             // short code + small coefficient in one lookup
              kk += (fa >> 4) & 15;
              br.consume((unsigned)(fa & 15));
              const int z = c_zig[kk++];
              if (lane == 0) blk[z] = (short)((fa >> 8) * q[z]);
              continue;
            }
            const int rs = br.decode(ha);
            if (rs < 0) { rc = JST_BAD_CODE; break; }
            const int sz = rs & 15, r = rs >> 4;
            if (sz == 0) { if (rs != 0xF0) break; kk += 16; }
            else { kk += r; const int z = c_zig[kk++]; const int v = extend(br.get(sz), sz); if (lane == 0) blk[z] = (short)(v * q[z]); }
          }
          if (rc != JST_OK) break;
        }
      }
      if (rc != JST_OK) break;                                     // (the host decoder takes over a frame flagged here: its planes are not used)
      __syncwarp();
      // ---- IDCT of all blocks of the MCU (jpeg.cpp: idct8x8_scalar; stb_image.h:1928-2027): one lane = one column, then one row
      for (int tsk = lane; tsk < nb * 8; tsk += 32) {
        const short* c = s_blk[tsk >> 3] + (tsk & 7); int* v = s_val[tsk >> 3] + (tsk & 7);
        IDCT_1D(c[0], c[8], c[16], c[24], c[32], c[40], c[48], c[56])
        x0 += 512; x1 += 512; x2 += 512; x3 += 512;
        v[0] = (x0 + t3) >> 10; v[63] = (x0 - t3) >> 10; v[9] = (x1 + t2) >> 10; v[54] = (x1 - t2) >> 10;
        v[18] = (x2 + t1) >> 10; v[45] = (x2 - t1) >> 10; v[27] = (x3 + t0) >> 10; v[36] = (x3 - t0) >> 10;
      }
      __syncwarp();
      for (int tsk = lane; tsk < nb * 8; tsk += 32) {
        const int row = tsk & 7;
        const int* v = s_val[tsk >> 3] + 9 * row;
        IDCT_1D(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7])
        const int bias = 65536 + (128 << 17);
        x0 += bias; x1 += bias; x2 += bias; x3 += bias;
        const unsigned lo = (unsigned)clamp8((x0 + t3) >> 17) | ((unsigned)clamp8((x1 + t2) >> 17) << 8) | ((unsigned)clamp8((x2 + t1) >> 17) << 16) | ((unsigned)clamp8((x3 + t0) >> 17) << 24);
        const unsigned hi = (unsigned)clamp8((x3 - t0) >> 17) | ((unsigned)clamp8((x2 - t1) >> 17) << 8) | ((unsigned)clamp8((x1 - t2) >> 17) << 16) | ((unsigned)clamp8((x0 - t3) >> 17) << 24);
        const unsigned bk = s_bk[tsk >> 3];
        const unsigned k = bk & 255u, by = (bk >> 8) & 255u, bx = bk >> 16;
        const size_t px = (size_t)f.plane_off[k] + (size_t)((my * f.cv[k] + by) * 8 + row) * f.w2[k] + (size_t)(mx * f.ch[k] + bx) * 8;
        *reinterpret_cast<uint2*>(pl + px) = make_uint2(lo, hi);
      }
      __syncwarp();
      // ---- restart interval (jpeg.cpp: handle_restart; stb_image.h:2451-2470)
      if (--todo <= 0) {
        if (!br.restart()) {                                       // no RSTn follows: the host decoder stops decoding here ("ended")
          rc = (my == f.mcuy - 1 && mx == f.mcux - 1) ? JST_OK : JST_BAD_RESTART;   // unfinished planes are the host decoder's business
          my = f.mcuy; break;
        }
        dc0 = dc1 = dc2 = 0;
        todo = f.restart ? (int)f.restart : 0x7fffffff;
      }
    }
  }
  if (lane == 0) { status[blockIdx.x] = rc; end_pos[blockIdx.x] = br.end_pos(); }
}

// ---- up-sampling + colour conversion, one thread per output pixel -----------------------------------------------------------------
__device__ __forceinline__ int chroma_at(const unsigned char* P, unsigned w2, unsigned rows, unsigned wl, int hs, int vs, int x, int y) {
  // rows of the chroma plane that stb pairs for output row y (jpeg.cpp: the ystep state machine, stb_image.h:3209-3225)
  if (hs == 1 && vs == 1) return P[(size_t)y * w2 + x];
  int rn, rf;
  if (vs == 2) { const int c = y >> 1; rn = c; rf = (y & 1) ? min(c + 1, (int)rows - 1) : max(c - 1, 0); }
  else { rn = rf = y; }
  const unsigned char* nr = P + (size_t)rn * w2; const unsigned char* fr = P + (size_t)rf * w2;
  if (hs == 1) return (3 * nr[x] + fr[x] + 2) >> 2;                                      // up_v2
  const int w = (int)wl;
  if (vs == 1) {                                                                          // up_h2 (incl. stb's last-pair quirk)
    if (w == 1) return nr[0];
    if (x == 0) return nr[0];
    if (x == 1) return (nr[0] * 3 + nr[1] + 2) >> 2;
    const int i = x >> 1;
    if (i == w - 1) return (x & 1) ? nr[w - 1] : (nr[w - 2] * 3 + nr[w - 1] + 2) >> 2;
    const int n3 = 3 * nr[i] + 2;
    return (x & 1) ? (n3 + nr[i + 1]) >> 2 : (n3 + nr[i - 1]) >> 2;
  }
  // up_hv2
  if (w == 1) return (3 * nr[0] + fr[0] + 2) >> 2;
  if (x == 0) return (3 * nr[0] + fr[0] + 2) >> 2;
  if (x == 2 * w - 1) return (3 * nr[w - 1] + fr[w - 1] + 2) >> 2;
  const int i = (x + 1) >> 1;                                                             // x = 2i-1 (odd) or 2i (even), 1 <= i <= w-1
  const int ta = 3 * nr[i - 1] + fr[i - 1], tb = 3 * nr[i] + fr[i];
  return (x & 1) ? (3 * ta + tb + 8) >> 4 : (3 * tb + ta + 8) >> 4;
}
// one colour pixel (x, y) of a decoded frame as r | g << 8 | b << 16 (jpeg.cpp: the per-row conversion; stb_image.h:3091-3118)
__device__ __forceinline__ unsigned pixel_rgb(const FrameDesc& f, const unsigned char* pl, int x, int y) {
  const int yy = pl[f.plane_off[0] + (size_t)y * f.w2[0] + x];
  if (f.ncomp == 1) return (unsigned)yy * 0x010101u;
  int cc[2];
#pragma unroll
  for (int k = 1; k <= 2; ++k) {
    // sampling factors are 1 or 2 (parse_frame admits nothing else): no integer divisions per pixel
    const int hs = (f.hmax == 2 && f.ch[k] == 1) ? 2 : 1, vs = (f.vmax == 2 && f.cv[k] == 1) ? 2 : 1;
    cc[k - 1] = chroma_at(pl + f.plane_off[k], f.w2[k], f.cy[k], (f.W + hs - 1) >> (hs - 1), hs, vs, x, y);
  }
  return ycc_to_rgb(yy, cc[0], cc[1]);
}
// grid: (ceil(out_px / 256), n frames).  lut == nullptr: out pixel p = colour pixel p (out_px = W*H); else out pixel p shows
// colour pixel lut[p] (-1 = none -> black), the depth-registered sampling of the fusion path.
__global__ void __launch_bounds__(256)
k_jpeg_color(const FrameDesc* __restrict__ fd, const unsigned char* __restrict__ planes, size_t plane_stride, const int* __restrict__ status,
             const int* __restrict__ lut, unsigned out_px, unsigned char* __restrict__ out) {
  const FrameDesc& f = fd[blockIdx.y];
  if (status[blockIdx.y] != JST_OK) return;                      // the host decoder fills this frame
  const unsigned p = blockIdx.x * 256u + threadIdx.x;
  if (p >= out_px) return;
  unsigned char* o = out + ((size_t)blockIdx.y * out_px + p) * 3;
  int q = lut ? lut[p] : (int)p;
  if (q < 0) { o[0] = o[1] = o[2] = 0; return; }
  const unsigned c = pixel_rgb(f, planes + (size_t)blockIdx.y * plane_stride, q % f.W, q / f.W);
  o[0] = (unsigned char)c; o[1] = (unsigned char)(c >> 8); o[2] = (unsigned char)(c >> 16);
}
// whole frames (no map), out_px a multiple of 4: one thread = 4 consecutive pixels = three 32-bit stores (the per-pixel kernel's
// three byte stores held it at ~340 GB/s).  grid: (ceil(out_px / 1024), n frames)
__global__ void __launch_bounds__(256)
k_jpeg_color4(const FrameDesc* __restrict__ fd, const unsigned char* __restrict__ planes, size_t plane_stride, const int* __restrict__ status,
              unsigned out_px, unsigned char* __restrict__ out) {
  const FrameDesc& f = fd[blockIdx.y];
  if (status[blockIdx.y] != JST_OK) return;
  const unsigned p0 = (blockIdx.x * 256u + threadIdx.x) * 4u;
  if (p0 >= out_px) return;
  const unsigned char* pl = planes + (size_t)blockIdx.y * plane_stride;
  int x = (int)(p0 % f.W), y = (int)(p0 / f.W);
  unsigned c[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c[i] = pixel_rgb(f, pl, x, y);
    if (++x == (int)f.W) { x = 0; ++y; }
  }
  unsigned* o = reinterpret_cast<unsigned*>(out + ((size_t)blockIdx.y * out_px + p0) * 3);     // 12-byte chunks of 4-byte aligned frames
  o[0] = c[0] | (c[1] << 24);
  o[1] = (c[1] >> 8) | (c[2] << 16);
  o[2] = (c[2] >> 16) | (c[3] << 8);
}

// ---- host: marker parsing ------------------------------------------------------------------------------------------------------
struct Parsed { FrameDesc d; std::vector<uint8_t> table_bytes; bool ok = false; };

// Parses up to the first SOS.  Fills d (supported = 0 when the device path does not handle the stream) and the raw DQT/DHT bytes
// that identify the table set.
void parse_frame(const uint8_t* d, size_t n, uint32_t want_w, uint32_t want_h, Parsed& out, TableSet& ts) {
  FrameDesc& f = out.d;
  memset(&f, 0, sizeof(f));
  memset(&ts, 0, sizeof(ts));
  out.table_bytes.clear();
  if (n < 4 || n > 0xFFFFFFF0ull || d[0] != 0xFF || d[1] != 0xD8) return;
  Header h(want_w, want_h); Scan sc;
  if (parse_header(d, n, 2, h, sc, &out.table_bytes) != kScan) return;
  // the device subset: one baseline / extended-sequential frame header (the parser has already refused Ss, Ah, Al != 0 in it)
  // and Huffman table ids 0-1
  if (h.n_sof != 1 || h.sof == 0xC2 || h.other_sof) return;
  for (int k = 2; k < 4; ++k) if (h.dc[k].present || h.ac[k].present) return;
  // sampling factors 1 or 2 and 1x1 chroma, so luma carries the full resolution.  A one-component frame is one non-interleaved
  // scan whatever its sampling factors say: one block per MCU, ceil(W / 8) blocks per row (T.81 A.2.2; jpeg.cpp and stb read it so)
  const int nc = h.ncomp;
  for (int i = 0; i < nc; ++i) {
    const FrameComp& c = h.comp[i];
    if (c.h > 2 || c.v > 2 || (i > 0 && (c.h != 1 || c.v != 1))) return;
    f.ch[i] = (unsigned char)(nc == 1 ? 1 : c.h); f.cv[i] = (unsigned char)(nc == 1 ? 1 : c.v); f.tq[i] = (unsigned char)c.tq;
  }
  // one interleaved scan listing the components in the frame header's order (what every encoder writes; compared by id, as the
  // stream names them), tables 0-1 present
  if (sc.ns != nc) return;
  for (int i = 0; i < nc; ++i) {
    const int td = sc.td[i], ta = sc.ta[i];
    if (h.comp[sc.comp[i]].id != h.comp[i].id || td > 1 || ta > 1 || !h.have_q[h.comp[i].tq] || !h.dc[td].present || !h.ac[ta].present) return;
    f.td[i] = (unsigned char)td; f.ta[i] = (unsigned char)ta;
  }
  const int W = h.W, H = h.H, hmax = f.ch[0], vmax = f.cv[0];
  f.W = (unsigned short)W; f.H = (unsigned short)H; f.ncomp = (unsigned char)nc; f.hmax = (unsigned char)hmax; f.vmax = (unsigned char)vmax;
  f.restart = (unsigned)h.restart; f.scan_start = (unsigned)sc.data; f.n_bytes = (unsigned)n;
  f.mcux = (unsigned)((W + 8 * hmax - 1) / (8 * hmax)); f.mcuy = (unsigned)((H + 8 * vmax - 1) / (8 * vmax));
  unsigned off = 0;
  for (int i = 0; i < nc; ++i) {
    f.w2[i] = f.mcux * f.ch[i] * 8; f.h2[i] = f.mcuy * f.cv[i] * 8;
    f.cy[i] = (unsigned)((H * f.cv[i] + vmax - 1) / vmax);
    f.plane_off[i] = off; off += (f.w2[i] * f.h2[i] + 15u) & ~15u;
  }
  for (int k = 0; k < 2; ++k) { if (h.dc[k].present) ts.dc[k] = h.dc[k]; if (h.ac[k].present) ts.ac[k] = h.ac[k]; }
  memcpy(ts.quant, h.quant, sizeof(ts.quant));
  for (int k = 0; k < 4; ++k) ts.have_q[k] = h.have_q[k];
  f.supported = 1; out.ok = true;
}

// After the device has consumed the scan: the host decoder would go on reading markers; anything but padding / EOI after
// the scan (another SOS, tables for it ...) means a multi-scan file, which the device path does not do.
bool tail_is_plain(const uint8_t* d, size_t n, size_t pos) {
  while (pos + 1 < n && !(d[pos] == 0xFF && d[pos + 1] != 0 && !(d[pos + 1] >= 0xD0 && d[pos + 1] <= 0xD7) && d[pos + 1] != 0xFF)) ++pos;
  if (pos + 1 >= n) return true;                                   // ran out of data without another marker: the host would stop too
  return d[pos + 1] == 0xD9;
}

constexpr size_t kJSlice = size_t(64) << 20;
struct JpegStage {
  int device = 0;
  scn::PinnedPtr<uint8_t> h[2]; scn::EventPtr ev[2];
  scn::EventPtr tk[3];                               // timing events: before the entropy kernel, between, after the colour kernel
  scn::DBuf d_in; size_t in_cap = 0;                 // uint8_t
  scn::DBuf d_planes; size_t planes_cap = 0;         // uint8_t
  scn::DBuf d_fd, d_status, d_end; size_t ncap = 0;  // FrameDesc, int, unsigned
  scn::DBuf d_sets; size_t sets_cap = 0;             // TableSet
  bool ensure(size_t in_bytes, size_t plane_bytes, size_t n, size_t nsets) {
    for (int i = 0; i < 2; ++i) if (!h[i]) {
      if (scn::create(h[i], kJSlice) != cudaSuccess || scn::create(ev[i], cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); return false; }
    }
    for (int i = 0; i < 3; ++i) if (!tk[i] && scn::create(tk[i]) != cudaSuccess) { cudaGetLastError(); return false; }
    auto grow = [](scn::DBuf& b, size_t* cap, size_t want) {
      if (want <= *cap) return true;
      *cap = 0;
      const size_t w = want + (want >> 2) + 4096;
      if (!b.alloc(w)) return false;
      *cap = w; return true;
    };
    if (!grow(d_in, &in_cap, in_bytes) || !grow(d_planes, &planes_cap, plane_bytes)) return false;
    if (n > ncap) {
      d_fd.reset(); d_status.reset(); d_end.reset(); ncap = 0;
      const size_t w = n + (n >> 2) + 64;
      if (!d_fd.alloc(w * sizeof(FrameDesc)) || !d_status.alloc(w * 4) || !d_end.alloc(w * 4)) return false;
      ncap = w;
    }
    size_t sc = sets_cap * sizeof(TableSet);
    if (!grow(d_sets, &sc, nsets * sizeof(TableSet))) return false;
    sets_cap = sc / sizeof(TableSet);
    return true;
  }
  void release() {
    for (int i = 0; i < 2; ++i) { h[i].reset(); ev[i].reset(); }
    for (int i = 0; i < 3; ++i) tk[i].reset();
    d_in.reset(); d_planes.reset(); d_fd.reset(); d_status.reset(); d_end.reset(); d_sets.reset();
    in_cap = planes_cap = ncap = sets_cap = 0;
  }
};
scn::StagePool<JpegStage>& jpeg_pool() { static auto* p = new scn::StagePool<JpegStage>(); return *p; }
struct JpegTimings { double host_s = 0, entropy_ms = 0, color_ms = 0; };
thread_local JpegTimings g_jlast;

}  // namespace

extern "C" {

// n baseline JPEG payloads (host pointers), every one `width` x `height`, decoded on the device.
//   d_lut == NULL : d_out receives n frames of width*height RGB8 (the bytes of scn_sens_frame_color_rgb8);
//   d_lut != NULL : device array of out_px ints, colour pixel index per output pixel (-1 = none -> black); d_out receives n
//                   frames of out_px RGB8 - the depth-registered colour the fusion path consumes.
// Frames the device path does not handle or flags as corrupt are decoded by the host decoder (same bytes, same errors) and
// uploaded; an undecodable frame fails the call like scn_sens_frame_color_rgb8 does.  n_on_device (optional) reports how many
// frames the device decoded.  Returns after the work on `stream` has completed.
int scn_jpeg_decode_batch_device(const uint8_t* const* src, const uint64_t* src_bytes, uint32_t n, uint32_t width, uint32_t height,
                                 const int32_t* d_lut, uint32_t out_px, void* d_out, void* stream, uint32_t* n_on_device) {
  if (n_on_device) *n_on_device = 0;
  if (!n) return SCN_OK;
  if (!src || !src_bytes || !d_out || !width || !height) return scn::fail(SCN_ERR_ARG, "null argument");
  if (!d_lut) out_px = width * height;
  cudaStream_t st = (cudaStream_t)stream;
  const double t_call = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  // 1. parse (a few host threads), collect distinct table sets
  std::vector<Parsed> P(n); std::vector<TableSet> ts_all(n);
  {
    const unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    auto work = [&](unsigned t) { for (uint32_t i = t; i < n; i += nt) parse_frame(src[i], (size_t)src_bytes[i], width, height, P[i], ts_all[i]); };
    if (n >= 4 * nt && nt > 1) { std::vector<std::thread> pool; for (unsigned t = 1; t < nt; ++t) pool.emplace_back(work, t); work(0); for (auto& th : pool) th.join(); }
    else for (unsigned t = 0; t < nt; ++t) work(t);
  }
  std::vector<TableSet> sets; std::vector<const std::vector<uint8_t>*> set_keys;
  size_t plane_stride = 0, in_total = 0;
  std::vector<unsigned long long> off(n + 1);
  for (uint32_t i = 0; i < n; ++i) {
    off[i] = in_total;
    if (!P[i].ok) continue;
    if (src_bytes[i] + 16 > kJSlice) { P[i].ok = false; P[i].d.supported = 0; continue; }
    unsigned id = 0;
    for (; id < set_keys.size(); ++id) if (*set_keys[id] == P[i].table_bytes) break;
    if (id == set_keys.size()) { set_keys.push_back(&P[i].table_bytes); sets.push_back(ts_all[i]); }
    P[i].d.table_set = id; P[i].d.src_off = in_total;
    in_total += ((size_t)src_bytes[i] + 15) & ~size_t(15);
    const FrameDesc& f = P[i].d;
    const size_t pb = (size_t)f.plane_off[f.ncomp - 1] + (((size_t)f.w2[f.ncomp - 1] * f.h2[f.ncomp - 1] + 15) & ~size_t(15));
    plane_stride = std::max(plane_stride, pb);
  }
  off[n] = in_total;
  scn::StagePool<JpegStage>::Lease lease(jpeg_pool());
  JpegStage& g = *lease;
  if (!g.ensure(in_total + 16, plane_stride * n + 16, n, std::max<size_t>(1, sets.size()))) return scn::fail(SCN_ERR_CUDA, "scn_jpeg_decode_batch_device: device staging allocation failed");
  std::vector<FrameDesc> fd(n);
  for (uint32_t i = 0; i < n; ++i) fd[i] = P[i].d;
  cudaError_t e = cudaMemcpyAsync(g.d_fd.as<FrameDesc>(), fd.data(), n * sizeof(FrameDesc), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && !sets.empty()) e = cudaMemcpyAsync(g.d_sets.as<TableSet>(), sets.data(), sets.size() * sizeof(TableSet), cudaMemcpyHostToDevice, st);
  // 2. pack + upload the supported payloads through the two pinned slices
  {
    const unsigned nt = std::max(1u, std::min(24u, std::thread::hardware_concurrency()));     // packing is a 2-3 GB memcpy per scan: spread it
    int slot = 0; bool used[2] = {false, false};
    for (uint32_t i0 = 0; i0 < n && e == cudaSuccess;) {
      uint32_t i1 = i0; while (i1 < n && off[i1 + 1] - off[i0] <= kJSlice) ++i1;
      if (used[slot]) e = cudaEventSynchronize(g.ev[slot].get());
      if (e != cudaSuccess) break;
      uint8_t* hs = g.h[slot].get(); const size_t base = off[i0];
      auto fill = [&](unsigned t) {
        for (uint32_t i = i0 + t; i < i1; i += nt) if (P[i].ok) {
          memcpy(hs + (off[i] - base), src[i], (size_t)src_bytes[i]);
          memset(hs + (off[i] - base) + src_bytes[i], 0, (size_t)(off[i + 1] - off[i] - src_bytes[i]));
        }
      };
      if (i1 - i0 >= 4 * nt && nt > 1) { std::vector<std::thread> pool; for (unsigned t = 1; t < nt; ++t) pool.emplace_back(fill, t); fill(0); for (auto& th : pool) th.join(); }
      else for (unsigned t = 0; t < nt; ++t) fill(t);
      if (off[i1] > base) e = cudaMemcpyAsync(g.d_in.as<uint8_t>() + base, hs, (size_t)(off[i1] - base), cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess) e = cudaEventRecord(g.ev[slot].get(), st);
      used[slot] = true; slot ^= 1; i0 = i1;
    }
  }
  // 3. decode
  std::vector<int> status(n, JST_UNSUPPORTED); std::vector<unsigned> endp(n, 0);
  const double t_packed = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
  if (e == cudaSuccess) {
    cudaEventRecord(g.tk[0].get(), st);
    k_jpeg_entropy_idct<<<n, 32, 0, st>>>(g.d_in.as<uint8_t>(), g.d_fd.as<FrameDesc>(), g.d_sets.as<TableSet>(), g.d_planes.as<uint8_t>(), plane_stride, g.d_status.as<int>(), g.d_end.as<unsigned>());
    cudaEventRecord(g.tk[1].get(), st);
    e = cudaMemcpyAsync(status.data(), g.d_status.as<int>(), (size_t)n * 4, cudaMemcpyDeviceToHost, st);
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(endp.data(), g.d_end.as<unsigned>(), (size_t)n * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  // multi-scan files: what follows the scan must be padding / EOI, else the host decoder takes the frame
  std::vector<uint32_t> redo;
  if (e == cudaSuccess) {
    bool changed = false;
    for (uint32_t i = 0; i < n; ++i) {
      if (status[i] == JST_OK && !tail_is_plain(src[i], (size_t)src_bytes[i], endp[i])) { status[i] = JST_UNSUPPORTED; changed = true; }
      if (status[i] != JST_OK) redo.push_back(i);
    }
    if (changed) e = cudaMemcpyAsync(g.d_status.as<int>(), status.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st);
  }
  if (e == cudaSuccess) {
    if (!d_lut && out_px % 4 == 0 && (reinterpret_cast<uintptr_t>(d_out) & 3) == 0)
      k_jpeg_color4<<<dim3((out_px + 1023) / 1024, n), 256, 0, st>>>(g.d_fd.as<FrameDesc>(), g.d_planes.as<uint8_t>(), plane_stride, g.d_status.as<int>(), out_px, (unsigned char*)d_out);
    else
      k_jpeg_color<<<dim3((out_px + 255) / 256, n), 256, 0, st>>>(g.d_fd.as<FrameDesc>(), g.d_planes.as<uint8_t>(), plane_stride, g.d_status.as<int>(), d_lut, out_px, (unsigned char*)d_out);
    cudaEventRecord(g.tk[2].get(), st);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    float ms = 0;
    if (e == cudaSuccess && cudaEventElapsedTime(&ms, g.tk[0].get(), g.tk[1].get()) == cudaSuccess) g_jlast.entropy_ms = ms;
    if (e == cudaSuccess && cudaEventElapsedTime(&ms, g.tk[1].get(), g.tk[2].get()) == cudaSuccess) g_jlast.color_ms = ms;
    g_jlast.host_s = t_packed - t_call;
  }
  if (e != cudaSuccess) return scn::fail(SCN_ERR_CUDA, "scn_jpeg_decode_batch_device: %s", cudaGetErrorString(e));
  if (n_on_device) *n_on_device = n - (uint32_t)redo.size();
  // 4. host decoder for the rest (same bytes), resampled through the map if there is one
  if (!redo.empty()) {
    std::vector<int32_t> lut;
    if (d_lut) { lut.resize(out_px); SCN_CUDA_TRY(cudaMemcpyAsync(lut.data(), d_lut, (size_t)out_px * 4, cudaMemcpyDeviceToHost, st)); SCN_CUDA_TRY(cudaStreamSynchronize(st)); }
    std::vector<uint8_t> full((size_t)width * height * 3), res;
    if (d_lut) res.resize((size_t)out_px * 3);
    for (uint32_t i : redo) {
      const int rc = scn::jpeg_decode_rgb8(src[i], (size_t)src_bytes[i], width, height, full.data());
      if (rc) return rc;
      const uint8_t* h = full.data();
      if (d_lut) { scn::rgb8_through_lut(full.data(), lut.data(), out_px, res.data()); h = res.data(); }
      SCN_CUDA_TRY(cudaMemcpyAsync((uint8_t*)d_out + (size_t)i * out_px * 3, h, (size_t)out_px * 3, cudaMemcpyHostToDevice, st));
      SCN_CUDA_TRY(cudaStreamSynchronize(st));
    }
  }
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

// timings of the last scn_jpeg_decode_batch_device call of this thread: host parse + pack + upload issue (s), entropy+IDCT kernel
// and colour kernel (ms, CUDA events)
void scn_jpeg_release_staging_() { jpeg_pool().trim(); }

int scn_jpeg_last_timings(double* host_s, double* entropy_ms, double* color_ms) {
  if (host_s) *host_s = g_jlast.host_s;
  if (entropy_ms) *entropy_ms = g_jlast.entropy_ms;
  if (color_ms) *color_ms = g_jlast.color_ms;
  return SCN_OK;
}

// Colour frames [first, first+n) of an open .sens stream decoded into device memory (RGB8).  TYPE_JPEG goes through the
// device decoder; raw and PNG colour (and any JPEG the device path declines) through the host decoder + upload.
int scn_sens_decode_color_device(const scn_sens* s, uint64_t first, uint32_t n, const int32_t* d_lut, uint32_t out_px, void* d_out,
                                 void* stream, uint32_t* n_on_device) {
  if (n_on_device) *n_on_device = 0;
  if (!s || (!d_out && n)) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_sens_info_t info;
  if (scn_sens_info(s, &info)) return SCN_ERR_ARG;
  if (first + n > info.n_frames) return scn::fail(SCN_ERR_ARG, "out of bounds");
  if (!d_lut) out_px = info.color_width * info.color_height;
  if (info.color_compression == 2) {
    std::vector<const uint8_t*> src(n); std::vector<uint64_t> len(n);
    for (uint32_t i = 0; i < n; ++i) {
      const uint8_t* c = nullptr; const uint8_t* d = nullptr; uint64_t cb = 0;
      if (scn_sens_frame_payload(s, first + i, &c, &d) || scn_sens_frame_meta(s, first + i, nullptr, nullptr, nullptr, &cb, nullptr)) return SCN_ERR_ARG;
      src[i] = c; len[i] = cb;
    }
    return scn_jpeg_decode_batch_device(src.data(), len.data(), n, info.color_width, info.color_height, d_lut, out_px, d_out, stream, n_on_device);
  }
  // raw / PNG: host decode, frame by frame
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<int32_t> lut;
  if (d_lut) { lut.resize(out_px); SCN_CUDA_TRY(cudaMemcpyAsync(lut.data(), d_lut, (size_t)out_px * 4, cudaMemcpyDeviceToHost, st)); SCN_CUDA_TRY(cudaStreamSynchronize(st)); }
  std::vector<uint8_t> full((size_t)info.color_width * info.color_height * 3), res((size_t)(d_lut ? out_px : 0) * 3);
  for (uint32_t i = 0; i < n; ++i) {
    const int rc = d_lut ? scn::sens_color_to_depth(s, first + i, lut.data(), out_px, full.data(), res.data())
                         : scn_sens_frame_color_rgb8(s, first + i, full.data());
    if (rc) return rc;
    const uint8_t* h = d_lut ? res.data() : full.data();
    SCN_CUDA_TRY(cudaMemcpyAsync((uint8_t*)d_out + (size_t)i * out_px * 3, h, (size_t)out_px * 3, cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
  }
  return SCN_OK;
}

}  // extern "C"
