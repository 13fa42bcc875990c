// Internal declarations shared by tsdf.cu (fusion) and mc.cu (meshing): device tables, key packing, hash,
// and the host-side handle.  Not part of the public ABI.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

#include "scn_common.h"

namespace scn_tsdf_detail {

constexpr int kMaxBatch = 32;
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr int kKeyBias = 1 << 20;
constexpr int kDdaMaxSteps = 48;

struct VolParams {
  float vs, trunc_base, trunc_scale, dmin, dmax, maxint, inv_range, ws15, inv_bs, depth_shift;
  int W, H, weight_max, const_w1;
  // pixel rounding / gather addressing of the integrate kernels (tsdf.cu: frame_column)
  float magic_x;             // 1.5*2^23 + jx: u + magic_x has round-half-even(u) + cx_raw in its raw bits
  unsigned cx_raw;           // raw bits of magic_x
  unsigned c_raw;            // (raw bits of 1.5*2^23) * W + cx_raw  (mod 2^32): raw gather index = pixel + c_raw, never wraps
  unsigned sentinel_raw;     // raw index of the per-frame NaN element (pixel W*H)
  unsigned Wm2, Hm2;         // W-2, H-2 (0 when the image is narrower than 3 pixels: the fast path is then never taken)
  unsigned wmax8;            // 8 * weight_max (byte offset into the (w, 1/(w+1)) table)
  int dm_stride;             // elements between consecutive frames of dm / rgbx: W*H + kDmPad
};
constexpr int kDmPad = 32;   // one NaN sentinel element per frame + padding to keep frames 128-byte aligned
struct FrameParams {
  float T[12];       // cam2world rows 0..2
  float Rt[9];       // world->cam rotation
  float tinv[3];     // world->cam translation
  float Avs[9];      // Rt * voxel_size
  float fx, fy, cx, cy;
  float ifx, ify;    // 1/fx, 1/fy (correctly rounded, host)
  int src;           // index of the frame inside the depth / rgb source buffers
  int has_rgb;
};
struct BatchParams {
  FrameParams f[kMaxBatch];
  int n;
};

struct Tables {
  unsigned long long* keys;
  int* vals;
  unsigned int* mask;             // view of the batch parity in flight (host passes mask_base + parity*cap)
  unsigned long long* block_keys;
  unsigned int* list;             // view of the batch parity in flight
  unsigned long long* counters;   // [0] heap_count [1],[2] list_count ping-pong [3] N_u [4] N_b [5] error flags
  uint2* heap;                    // 512 voxels per block
  unsigned int cap_mask;
  unsigned int max_blocks;
};

enum { C_HEAP = 0, C_LIST0 = 1, C_LIST1 = 2, C_NU = 3, C_NB = 4, C_ERR = 5, C_UNION = 6, C_WORK0 = 7, C_WORK1 = 8, C_DONE0 = 9, C_DONE1 = 10, C_COUNT = 16 };

// ------------------------------------------------------------------------------ device
__host__ __device__ __forceinline__ bool key_ok(int x, int y, int z) {
  return x >= -kKeyBias && x < kKeyBias && y >= -kKeyBias && y < kKeyBias && z >= -kKeyBias && z < kKeyBias;
}
__host__ __device__ __forceinline__ unsigned long long pack_key(int x, int y, int z) {
  return (unsigned long long)(unsigned)(x + kKeyBias) | ((unsigned long long)(unsigned)(y + kKeyBias) << 21) |
         ((unsigned long long)(unsigned)(z + kKeyBias) << 42);
}
__host__ __device__ __forceinline__ void unpack_key(unsigned long long k, int& x, int& y, int& z) {
  x = (int)(k & 0x1FFFFF) - kKeyBias;
  y = (int)((k >> 21) & 0x1FFFFF) - kKeyBias;
  z = (int)((k >> 42) & 0x1FFFFF) - kKeyBias;
}
// vec3i hash of mLib (external/mLib/include/core-util/sparseGrid3.h:14-17) + an avalanche so
// that the power-of-two table mask sees all bits.
__device__ __forceinline__ unsigned hash_key(unsigned long long k) {
  int x, y, z;
  unpack_key(k, x, y, z);
  unsigned h = ((unsigned)x * 73856093u) ^ ((unsigned)y * 19349669u) ^ ((unsigned)z * 83492791u);
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}


// read-only lookup: heap index of block (x,y,z) or -1
__device__ __forceinline__ int lookup_block(const Tables& tb, int x, int y, int z) {
  if (!key_ok(x, y, z)) return -1;
  const unsigned long long key = pack_key(x, y, z);
  unsigned slot = hash_key(key) & tb.cap_mask;
  for (unsigned probe = 0; probe <= tb.cap_mask; ++probe) {
    const unsigned long long k = tb.keys[slot];
    if (k == key) return tb.vals[slot];
    if (k == kEmptyKey) return -1;
    slot = (slot + 1) & tb.cap_mask;
  }
  return -1;
}

// ------------------------------------------------------------------------------ host (shared with freespace.cu)
// Per-frame constants of spec step C (TSDF §3, free space §6h): every product and sum is one binary32 operation in the
// oracles' order (volatile keeps the host compiler from reassociating or widening).
inline void make_frame_params(float vs, const float* T, const float* K, int src, bool has_rgb, FrameParams& fp) {
  for (int i = 0; i < 12; ++i) fp.T[i] = T[i];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) fp.Rt[3 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; ++i) {
    volatile float a = fp.Rt[3 * i + 0] * T[3];
    volatile float b = fp.Rt[3 * i + 1] * T[7];
    volatile float c = fp.Rt[3 * i + 2] * T[11];
    volatile float ab = a + b;
    fp.tinv[i] = -(ab + c);
  }
  for (int i = 0; i < 9; ++i) { volatile float v = fp.Rt[i] * vs; fp.Avs[i] = v; }
  fp.fx = K[0]; fp.cx = K[2]; fp.fy = K[5]; fp.cy = K[6];
  { volatile float a = 1.0f / fp.fx; volatile float b = 1.0f / fp.fy; fp.ifx = a; fp.ify = b; }
  fp.src = src; fp.has_rgb = has_rgb ? 1 : 0;
}

// Spec step A as a table: raw u16 -> metres (IEEE division, as the oracles) or NaN when outside [depth_min, depth_max]
inline void make_depth_lut(float depth_shift, float depth_min, float depth_max, std::vector<float>& lut) {
  lut.resize(65536);
  for (int r = 0; r < 65536; ++r) {
    volatile float q = r == 0 ? 0.0f : (float)r / depth_shift;
    const float m = q;
    lut[r] = (m >= depth_min && m <= depth_max) ? m : NAN;
  }
}

}  // namespace scn_tsdf_detail

struct scn_tsdf {
  scn_tsdf_params p{};
  int device = 0;
  int sm_count = 132;
  scn_tsdf_detail::VolParams vp{};
  scn_tsdf_detail::Tables tb{};                  // the buffers below as the kernels see them (filled once, after allocation)
  uint64_t cap = 0;
  scn::DBuf keys, vals, block_keys, counters, heap;
  scn::DBuf mask_base, list_base;                // 2 x cap, 2 x max_blocks: one set per batch parity
  scn::DBuf dm;
  scn::DBuf depth_lut;                           // raw u16 depth -> metres or NaN (spec step A + range test), 65536 entries
  scn::DBuf rgbx;                                // colour of the current batches repacked to one word per pixel (2 parities), allocated on first use
  scn::DBuf d_depth[2], d_rgb[2];                // H2D staging, double buffered
  scn::PinnedPtr<uint16_t> h_depth[2];           // pinned bounce buffers (pageable callers)
  scn::PinnedPtr<uint8_t> h_rgb[2];
  cudaStream_t stream = nullptr;                 // the caller's stream (scn_tsdf_set_stream), not owned
  scn::StreamPtr copy_stream, alloc_stream;
  scn::EventPtr ev_alloc_done[2], ev_integ_done[2], ev_input;
  bool parity_used[2] = {false, false};
  bool heap_zeroed = false;                      // the whole heap has been cleared once; later resets clear only the used prefix
  scn::EventPtr ev_copied[2], ev_consumed[2];
  bool buf_used[2] = {false, false};
  int parity = 0;
  uint64_t frames_integrated = 0, frames_skipped = 0, frame_bytes = 0, launches = 0;
  uint64_t chunk_seq = 0;
  bool profile = false;
  std::vector<scn::EventPtr> prof_events;        // 4 per batch: around k_alloc (allocation stream), around the integrate kernel
  size_t prof_used = 0;
  scn::DBuf filt_raw, filt_out;                  // bilateral pre-filter scratch: 2 parities x K frames each (lazy)
  float mc_thresh_factor = 10.0f;         // s_SDFMarchingCubeThreshFactor (zParametersScanNet.txt:48)
};

namespace scn_tsdf_detail {

// Host copy of the device counters; the caller first synchronises the streams that write them.  `blocks` is the heap
// count clamped to max_blocks: the allocator keeps counting past an exhausted heap.
struct Counters {
  unsigned long long c[C_COUNT];
  uint64_t blocks;
};
inline int read_counters(const scn_tsdf* t, Counters& out) {
  SCN_CUDA_TRY(cudaMemcpy(out.c, t->tb.counters, sizeof(out.c), cudaMemcpyDeviceToHost));
  out.blocks = std::min<uint64_t>(out.c[C_HEAP], t->tb.max_blocks);
  return SCN_OK;
}

}  // namespace scn_tsdf_detail

// filter.cu: u16 -> metres (-inf invalid) -> bilateral filter for the n frames of a batch, on the allocation stream
int scn_filter_batch(scn_tsdf* t, int n, const uint16_t* d_depth, const scn_tsdf_detail::BatchParams& bp, int parity, const float** out);
