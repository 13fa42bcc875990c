// Free-space occupancy grid on H100 (sm_90a): per-voxel counts of "seen free" and "seen occupied" over a dense lattice box,
// from depth frames with poses, then labels cropped to the labelled voxels (DESIGN.md §6h, "free-space spec v1").
//
// Stands in for the external FreeSpace.exe of the reference pipeline's `freespace` stage (<id>.sens -> <id>.grid,
// Server/config/scan_stages.json:43-47, Server/scan_processor.py:150-152); its source is not in the reference tree, so the
// numerical contract is this repository's own spec, whose scalar statement is oracle/freespace_oracle.c (test infrastructure,
// never linked here).  The projection is the TSDF's (spec step C, tsdf.cu), on the same voxel-centre convention.
//
// Data layout in HBM:
//   cnt[nvox]        uint2 {n_free, n_occ} per voxel of the envelope box, x fastest (8 B per voxel)
//   depth_lut[65536] f32 raw u16 -> metres, NaN for raw 0 or outside [depth_min, depth_max]
//   box[8]           u32 crop box of the labelled voxels in envelope indices (min x,y,z; max x,y,z) + free / occupied counts
//   pairs            u64 (brick, frame) pairs classified
//
// Kernels:
//   k_classify  grid-stride over the 8^3 bricks of the envelope; 64 threads = the (lx,ly) columns of one brick.  Warp 0 tests
//               the brick against every frame of the batch (one lane per frame, binary64, conservative: a skipped pair cannot
//               hold an observation) and the ballot is the brick's frame mask.  Each thread then holds its column's 16 counters
//               in registers while the frames of the mask are applied: one 8 B read and one 8 B write per voxel per batch.
//   k_box       label of every voxel; the labelled ones' indices reduced per warp, then atomicMin / atomicMax (exact, so the
//               box does not depend on the schedule), and the label counts
//   k_gather    labels (and counts) of the crop box
// The spec arithmetic uses explicit round-to-nearest intrinsics; the file is compiled with -fmad=false.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "scn_common.h"

#include "tsdf_internal.cuh"

using scn_tsdf_detail::BatchParams;
using scn_tsdf_detail::FrameParams;
using scn_tsdf_detail::kMaxBatch;

namespace {

constexpr float kZMin = 0.015625f;             // 2^-6 m: voxels closer to the camera plane are never observed (as the TSDF)
constexpr int64_t kMaxCoord = 1 << 23;         // lattice coordinates stay inside +-2^23: float(8b) is exact
constexpr uint64_t kMaxFramePx = 1ull << 24;

// Per-volume constants of the kernels
struct FsParams {
  float vs, band_base, band_scale, maxd;
  float Wf, Hf;
  unsigned W, H;
  int lo[3];
  unsigned dims[3];
  int blo[3];                // first brick of the envelope
  unsigned nb[3];            // bricks per axis
  unsigned long long n_bricks;
  double cull_r;             // bounding-sphere radius of a brick's voxel centres + margin (metres)
  double zfar;               // max_distance + band(max_distance): no observation lies farther along the view axis
};

// Per-frame cull planes in camera space (x or y against z), unit normals: a point seen inside the image +-1 px satisfies
// n . (x, z) >= 0 for the two u planes and n . (y, z) >= 0 for the two v planes
struct CullPlanes { double u[2][2], v[2][2]; };
struct FsBatch { CullPlanes c[kMaxBatch]; };

// ------------------------------------------------------------------------------ device
// One frame applied to one voxel (spec step C): z and the pixel, the depth, the band test
__device__ __forceinline__ void observe(float pcx, float pcy, float z, const float4 k, const FsParams& fs, const uint16_t* __restrict__ dep,
                                        const float* __restrict__ lut, unsigned& nf, unsigned& no) {
  if (!(z >= kZMin)) return;
  const float rz = __frcp_rn(z);
  const float u = __fmaf_rn(__fmul_rn(pcx, rz), k.x, k.z), v = __fmaf_rn(__fmul_rn(pcy, rz), k.y, k.w);
  const float ur = rintf(u), vr = rintf(v);                         // round half to even, exact; NaN fails the tests below
  if (!(ur >= 0.0f && ur < fs.Wf && vr >= 0.0f && vr < fs.Hf)) return;
  const float d = __ldg(lut + __ldg(dep + (unsigned)vr * fs.W + (unsigned)ur));
  if (!(d == d)) return;                                            // raw 0 or outside [depth_min, depth_max]
  const float s = __fsub_rn(d, z);
  const float band = __fmaf_rn(fs.band_scale, d, fs.band_base);
  if (s > band) { if (z < fs.maxd) ++nf; }
  else if (s > -band && d < fs.maxd) ++no;
}

// Conservative brick / frame test in binary64: the sphere around the brick's voxel centres against the near and far planes and
// the four side planes of the frustum widened by one pixel
__device__ __forceinline__ bool brick_visible(const FrameParams& fp, const CullPlanes& cp, const FsParams& fs, int bx, int by, int bz) {
  const double vs = fs.vs;
  const double c[3] = {(8.0 * bx + 3.5) * vs, (8.0 * by + 3.5) * vs, (8.0 * bz + 3.5) * vs};
  double q[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) q[i] = (double)fp.Rt[3 * i] * c[0] + (double)fp.Rt[3 * i + 1] * c[1] + (double)fp.Rt[3 * i + 2] * c[2] + (double)fp.tinv[i];
  // the binary32 projection of a voxel differs from this one by a few ulps of the coordinates involved
  const double r = fs.cull_r + 1e-5 * (fabs(c[0]) + fabs(c[1]) + fabs(c[2]) + fabs(q[0]) + fabs(q[1]) + fabs(q[2]));
  return q[2] + r >= (double)kZMin && q[2] - r < fs.zfar &&
         cp.u[0][0] * q[0] + cp.u[0][1] * q[2] >= -r && cp.u[1][0] * q[0] + cp.u[1][1] * q[2] >= -r &&
         cp.v[0][0] * q[1] + cp.v[0][1] * q[2] >= -r && cp.v[1][0] * q[1] + cp.v[1][1] * q[2] >= -r;
}

// grid-stride over the bricks of the envelope; block = 64 threads = the (lx,ly) columns of the brick in hand
__global__ void __launch_bounds__(64)
k_classify(const __grid_constant__ BatchParams bp, const __grid_constant__ FsBatch cb, const FsParams fs, uint2* __restrict__ cnt,
           const uint16_t* __restrict__ depth, const float* __restrict__ lut, unsigned long long* __restrict__ pairs) {
  __shared__ float4 s_a[kMaxBatch][3];       // row i of Rt*vs: (A_i0, A_i1, A_i2)
  __shared__ float4 s_k[kMaxBatch];          // (fx, fy, cx, cy)
  __shared__ float4 s_base[kMaxBatch];       // base of the brick in hand, per frame
  __shared__ unsigned s_mask;
  const int t = threadIdx.x;
  for (int k = t; k < bp.n; k += 64) {
    const FrameParams& fp = bp.f[k];
#pragma unroll
    for (int i = 0; i < 3; ++i) s_a[k][i] = make_float4(fp.Avs[3 * i], fp.Avs[3 * i + 1], fp.Avs[3 * i + 2], 0.f);
    s_k[k] = make_float4(fp.fx, fp.fy, fp.cx, fp.cy);
  }
  const int lx = t & 7, ly = t >> 3;
  const float lxf = (float)lx, lyf = (float)ly;
  const size_t frame_px = (size_t)fs.W * fs.H;
  unsigned long long n_pairs = 0;
  for (unsigned long long brick = blockIdx.x; brick < fs.n_bricks; brick += gridDim.x) {
    const int bx = fs.blo[0] + (int)(brick % fs.nb[0]);
    const int by = fs.blo[1] + (int)((brick / fs.nb[0]) % fs.nb[1]);
    const int bz = fs.blo[2] + (int)(brick / ((unsigned long long)fs.nb[0] * fs.nb[1]));
    if (t < 32) {
      const bool vis = t < bp.n && brick_visible(bp.f[t], cb.c[t], fs, bx, by, bz);
      const unsigned m = __ballot_sync(0xffffffffu, vis);
      if (t == 0) s_mask = m;
      if (vis) {                             // spec step C: o = float(8b)*vs, base = Rt*o + tinv in the stated fma order
        const FrameParams& fp = bp.f[t];
        const float o[3] = {__fmul_rn((float)(8 * bx), fs.vs), __fmul_rn((float)(8 * by), fs.vs), __fmul_rn((float)(8 * bz), fs.vs)};
        float b[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) b[i] = __fmaf_rn(fp.Rt[3 * i + 2], o[2], __fmaf_rn(fp.Rt[3 * i + 1], o[1], __fmaf_rn(fp.Rt[3 * i + 0], o[0], fp.tinv[i])));
        s_base[t] = make_float4(b[0], b[1], b[2], 0.f);
      }
    }
    __syncthreads();
    unsigned m = s_mask;
    if (t == 0) n_pairs += __popc(m);
    // this thread's column inside the envelope: (ex, ey) and the voxels lz whose ez is inside too
    const int ex = 8 * bx + lx - fs.lo[0], ey = 8 * by + ly - fs.lo[1], ez0 = 8 * bz - fs.lo[2];
    if (m && (unsigned)ex < fs.dims[0] && (unsigned)ey < fs.dims[1]) {
      unsigned zin = 0;
#pragma unroll
      for (int z = 0; z < 8; ++z) zin |= ((unsigned)(ez0 + z) < fs.dims[2] ? 1u : 0u) << z;
      const size_t plane = (size_t)fs.dims[0] * fs.dims[1];
      uint2* col = cnt + (size_t)ey * fs.dims[0] + ex;
      unsigned nf[8], no[8];
#pragma unroll
      for (int z = 0; z < 8; ++z) {
        const uint2 c = (zin >> z) & 1u ? col[(size_t)(ez0 + z) * plane] : make_uint2(0u, 0u);
        nf[z] = c.x; no[z] = c.y;
      }
      while (m) {
        const int k = __ffs(m) - 1;
        m &= m - 1;
        const float4 b = s_base[k];
        const float4 a0 = s_a[k][0], a1 = s_a[k][1], a2 = s_a[k][2];
        const float qx = __fmaf_rn(lyf, a0.y, __fmaf_rn(lxf, a0.x, b.x));
        const float qy = __fmaf_rn(lyf, a1.y, __fmaf_rn(lxf, a1.x, b.y));
        const float qz = __fmaf_rn(lyf, a2.y, __fmaf_rn(lxf, a2.x, b.z));
        const float4 kk = s_k[k];
        const uint16_t* dep = depth + (size_t)bp.f[k].src * frame_px;
#pragma unroll
        for (int z = 0; z < 8; ++z) {
          const float zf = (float)z;
          observe(__fmaf_rn(zf, a0.z, qx), __fmaf_rn(zf, a1.z, qy), __fmaf_rn(zf, a2.z, qz), kk, fs, dep, lut, nf[z], no[z]);
        }
      }
#pragma unroll
      for (int z = 0; z < 8; ++z)
        if ((zin >> z) & 1u) col[(size_t)(ez0 + z) * plane] = make_uint2(nf[z], no[z]);
    }
    __syncthreads();                         // s_mask / s_base are rewritten for the next brick
  }
  if (t == 0 && n_pairs) atomicAdd(pairs, n_pairs);
}

// spec step D
__device__ __forceinline__ unsigned label_of(uint2 c) { return (c.x | c.y) == 0u ? 0u : (c.y > 0u && c.y >= c.x ? 2u : 1u); }

// box[0..2] = min index, box[3..5] = max index of the labelled voxels, box[6] / box[7] = free / occupied voxels.
// The loop bound is warp-uniform (the stride is a multiple of 32), so every lane takes part in the reductions.
__global__ void k_box(const uint2* __restrict__ cnt, unsigned d0, unsigned d1, unsigned long long nvox, unsigned* __restrict__ box) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  unsigned mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u}, n_free = 0, n_occ = 0;
  bool any = false;
  for (unsigned long long i0 = (unsigned long long)blockIdx.x * blockDim.x; i0 < nvox; i0 += stride) {
    const unsigned long long i = i0 + threadIdx.x;
    if (i >= nvox) break;
    const unsigned l = label_of(cnt[i]);
    if (!l) continue;
    const unsigned x = (unsigned)(i % d0), y = (unsigned)((i / d0) % d1), z = (unsigned)(i / ((unsigned long long)d0 * d1));
    mn[0] = min(mn[0], x); mn[1] = min(mn[1], y); mn[2] = min(mn[2], z);
    mx[0] = max(mx[0], x); mx[1] = max(mx[1], y); mx[2] = max(mx[2], z);
    any = true;
    if (l == 1u) ++n_free; else ++n_occ;
  }
  const unsigned full = 0xffffffffu;
  if (!__any_sync(full, any)) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) { mn[a] = __reduce_min_sync(full, mn[a]); mx[a] = __reduce_max_sync(full, mx[a]); }
  n_free = __reduce_add_sync(full, n_free); n_occ = __reduce_add_sync(full, n_occ);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { atomicMin(&box[a], mn[a]); atomicMax(&box[3 + a], mx[a]); }
    atomicAdd(&box[6], n_free); atomicAdd(&box[7], n_occ);
  }
}

// labels (and counts) of the crop box o0 .. o0+od-1 (envelope indices), x fastest
__global__ void k_gather(const uint2* __restrict__ cnt, unsigned d0, unsigned d1, uint3 o0, uint3 od, unsigned long long n,
                         uint8_t* __restrict__ labels, unsigned* __restrict__ n_free, unsigned* __restrict__ n_occ) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned x = (unsigned)(i % od.x), y = (unsigned)((i / od.x) % od.y), z = (unsigned)(i / ((unsigned long long)od.x * od.y));
    const uint2 c = cnt[((size_t)(z + o0.z) * d1 + (y + o0.y)) * d0 + (x + o0.x)];
    labels[i] = (uint8_t)label_of(c);
    if (n_free) { n_free[i] = c.x; n_occ[i] = c.y; }
  }
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int check_params(const scn_freespace_params* p) {
  if (!p) return scn::fail(SCN_ERR_ARG, "null argument");
  if (!(p->voxel_size > 0.f) || !std::isfinite(p->voxel_size)) return scn::fail(SCN_ERR_ARG, "voxel_size %g: must be > 0", p->voxel_size);
  if (!(p->band_base >= 0.f) || !(p->band_scale >= 0.f)) return scn::fail(SCN_ERR_ARG, "band terms %g + %g*d: must be >= 0", p->band_base, p->band_scale);
  if (!(p->depth_max > p->depth_min)) return scn::fail(SCN_ERR_ARG, "depth range [%g, %g] is empty", p->depth_min, p->depth_max);
  if (!(p->max_distance > 0.f)) return scn::fail(SCN_ERR_ARG, "max_distance %g: must be > 0", p->max_distance);
  return SCN_OK;
}

// a lattice box inside +-2^23 voxels per axis (float(8b) exact, indices far inside int)
int check_box(const int32_t lo[3], const uint64_t dims[3]) {
  for (int a = 0; a < 3; ++a)
    if (lo[a] < -kMaxCoord || dims[a] > (uint64_t)(2 * kMaxCoord) || (int64_t)lo[a] + (int64_t)dims[a] > kMaxCoord)
      return scn::fail(SCN_ERR_ARG, "lattice box %d+%llu on axis %d leaves +-2^23 voxels", lo[a], (unsigned long long)dims[a], a);
  return SCN_OK;
}

int64_t floor_div8(int64_t x) { return x >= 0 ? x / 8 : -((-x + 7) / 8); }

}  // namespace

struct scn_freespace {
  scn_freespace_params p{};
  int device = 0;
  int grid = 0;                              // CTAs of k_classify
  FsParams fs{};
  float depth_shift = 0.f;
  int32_t lo[3] = {0, 0, 0};
  uint64_t dims[3] = {0, 0, 0};
  uint64_t nvox = 0;
  scn::DBuf cnt, lut, box, pairs, staging;   // staging: host frames of one batch (scn_freespace_integrate)
  scn::PinnedPtr<uint16_t> h_staging;        // the same batch packed in pinned memory: one copy on `stream`
  scn::StreamPtr stream;
  scn::EventPtr ev0, ev1;
  scn_freespace_report_t rep{};              // frames, pairs, classify time; the last download's box, labels and time
};

namespace {

// one batch of <= 32 frames whose depth sits at d_depth + src * W*H
int run_batch(scn_freespace* h, const BatchParams& bp, const FsBatch& cb, const uint16_t* d_depth) {
  if (bp.n == 0) return SCN_OK;
  h->rep.frames_used += bp.n;
  h->rep.pairs_culled += (uint64_t)bp.n * h->fs.n_bricks;        // classified pairs are subtracted when the counter is read
  if (!h->nvox) return SCN_OK;
  k_classify<<<h->grid, 64, 0, h->stream.get()>>>(bp, cb, h->fs, h->cnt.as<uint2>(), d_depth, h->lut.as<float>(),
                                                  h->pairs.as<unsigned long long>());
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

void make_cull_planes(const FsParams& fs, const FrameParams& fp, CullPlanes& c) {
  // u >= -1.5  <=>  fx x + (cx + 1.5) z >= 0;  u <= W + 0.5  <=>  -fx x + (W + 0.5 - cx) z >= 0 (z > 0, fx > 0); v likewise
  const double fx = fp.fx, fy = fp.fy, cx = fp.cx, cy = fp.cy, W = fs.W, H = fs.H;
  const double nu[2][2] = {{fx, cx + 1.5}, {-fx, W + 0.5 - cx}}, nv[2][2] = {{fy, cy + 1.5}, {-fy, H + 0.5 - cy}};
  for (int i = 0; i < 2; ++i) {
    const double lu = std::sqrt(nu[i][0] * nu[i][0] + nu[i][1] * nu[i][1]), lv = std::sqrt(nv[i][0] * nv[i][0] + nv[i][1] * nv[i][1]);
    c.u[i][0] = nu[i][0] / lu; c.u[i][1] = nu[i][1] / lu; c.v[i][0] = nv[i][0] / lv; c.v[i][1] = nv[i][1] / lv;
  }
}

int check_intrinsics(const float* K) {
  if (!(K[0] > 0.f) || !(K[5] > 0.f) || !std::isfinite(K[0]) || !std::isfinite(K[5]) || !std::isfinite(K[2]) || !std::isfinite(K[6]))
    return scn::fail(SCN_ERR_ARG, "intrinsics need finite fx, fy > 0 and finite cx, cy");
  return SCN_OK;
}

// Frames [0, n) with a pose, in batches of <= 32; `upload(first, count, bp)` makes the batch's depth available and returns
// its device base (src indices of bp relative to it)
template <class Upload>
int integrate_frames(scn_freespace* h, uint32_t n, const float* cam2world, const float K[16], Upload upload) {
  if (int rc = check_intrinsics(K)) return rc;
  SCN_CUDA_TRY(cudaSetDevice(h->device));
  SCN_CUDA_TRY(cudaEventRecord(h->ev0.get(), h->stream.get()));
  BatchParams bp; bp.n = 0;
  FsBatch cb;
  std::vector<uint32_t> idx;
  auto flush = [&]() -> int {
    const uint16_t* base = nullptr;
    if (int rc = upload(idx, bp, &base)) return rc;
    int rc = run_batch(h, bp, cb, base);
    bp.n = 0; idx.clear();
    return rc;
  };
  for (uint32_t i = 0; i < n; ++i) {
    const float* T = cam2world + 16 * (size_t)i;
    if (T[0] == -INFINITY) { h->rep.frames_skipped_pose++; continue; }   // sensorData.h:382
    scn_tsdf_detail::make_frame_params(h->fs.vs, T, K, (int)i, false, bp.f[bp.n]);
    make_cull_planes(h->fs, bp.f[bp.n], cb.c[bp.n]);
    idx.push_back(i);
    if (++bp.n == kMaxBatch) { if (int rc = flush()) return rc; }
  }
  if (bp.n) { if (int rc = flush()) return rc; }
  SCN_CUDA_TRY(cudaEventRecord(h->ev1.get(), h->stream.get()));
  SCN_CUDA_TRY(cudaEventSynchronize(h->ev1.get()));
  float ms = 0.f;
  SCN_CUDA_TRY(cudaEventElapsedTime(&ms, h->ev0.get(), h->ev1.get()));
  h->rep.classify_ms += ms;
  return SCN_OK;
}

int read_pairs(const scn_freespace* h, uint64_t* classified) {
  unsigned long long v = 0;
  if (h->pairs.p) SCN_CUDA_TRY(cudaMemcpy(&v, h->pairs.p, 8, cudaMemcpyDeviceToHost));
  *classified = v;
  return SCN_OK;
}

}  // namespace

extern "C" {

void scn_freespace_default_params(scn_freespace_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->voxel_size = 0.05f;
  p->band_base = 0.05f;
  p->band_scale = 0.01f;
  p->depth_min = 0.1f;                  // zParametersScanNet.txt:35
  p->depth_max = 6.0f;                  // :34
  p->max_distance = 4.0f;               // :51 (s_SDFMaxIntegrationDistance)
  p->max_voxels = 1ull << 28;           // 2 GiB of counters
}

size_t scn_freespace_report_sizeof(void) { return sizeof(scn_freespace_report_t); }

int scn_freespace_envelope(const float* cam2world, uint32_t n, const float K[16], uint32_t width, uint32_t height,
                           const scn_freespace_params* p, int32_t lo[3], uint64_t dims[3]) {
  if (!K || !lo || !dims || (n && !cam2world)) return scn::fail(SCN_ERR_ARG, "null argument");
  if (int rc = check_params(p)) return rc;
  if (int rc = check_intrinsics(K)) return rc;
  if (!width || !height) return scn::fail(SCN_ERR_ARG, "empty frame size");
  const double fx = K[0], cx = K[2], fy = K[5], cy = K[6], vs = p->voxel_size, md = p->max_distance;
  const double ax = std::max(std::fabs(-1.5 - cx), std::fabs(width + 0.5 - cx)) / fx;
  const double ay = std::max(std::fabs(-1.5 - cy), std::fabs(height + 0.5 - cy)) / fy;
  const double reach = (md + (double)p->band_scale * md + (double)p->band_base) * std::sqrt(1.0 + ax * ax + ay * ay) + vs;
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  bool any = false;
  for (uint32_t i = 0; i < n; ++i) {
    const float* T = cam2world + 16 * (size_t)i;
    if (T[0] == -INFINITY) continue;
    const double c[3] = {T[3], T[7], T[11]};
    if (!std::isfinite(c[0]) || !std::isfinite(c[1]) || !std::isfinite(c[2])) continue;   // a NaN pose observes nothing
    for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], c[a]); mx[a] = std::max(mx[a], c[a]); }
    any = true;
  }
  if (!any) { for (int a = 0; a < 3; ++a) { lo[a] = 0; dims[a] = 0; } return SCN_OK; }
  int32_t l[3]; uint64_t d[3];
  for (int a = 0; a < 3; ++a) {
    const double g0 = std::floor((mn[a] - reach) / vs), g1 = std::ceil((mx[a] + reach) / vs);
    if (!(g0 >= -(double)kMaxCoord) || !(g1 < (double)kMaxCoord))
      return scn::fail(SCN_ERR_ARG, "envelope [%g, %g] m on axis %d leaves +-2^23 voxels of %g m", mn[a] - reach, mx[a] + reach, a, vs);
    l[a] = (int32_t)g0; d[a] = (uint64_t)(g1 - g0) + 1;
  }
  for (int a = 0; a < 3; ++a) { lo[a] = l[a]; dims[a] = d[a]; }
  return SCN_OK;
}

int scn_freespace_create(const scn_freespace_params* p, uint32_t width, uint32_t height, float depth_shift, const int32_t lo[3],
                         const uint64_t dims[3], int device, scn_freespace** out) {
  if (!p || !lo || !dims || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (int rc = check_params(p)) return rc;
  if (!width || !height || (uint64_t)width * height > kMaxFramePx) return scn::fail(SCN_ERR_ARG, "frame size %ux%u not supported", width, height);
  if (!(depth_shift > 0.f)) return scn::fail(SCN_ERR_ARG, "depth_shift %g: must be > 0", depth_shift);
  if (int rc = check_box(lo, dims)) return rc;
  const uint64_t nvox = dims[0] * dims[1] * dims[2];                // each factor <= 2^24: no overflow
  if (nvox > p->max_voxels)
    return scn::fail(SCN_ERR_CAPACITY, "lattice box %llux%llux%llu = %llu voxels (%.2f GiB of counters) exceeds max_voxels = %llu",
                     (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)nvox,
                     nvox * 8.0 / (1ull << 30), (unsigned long long)p->max_voxels);
  int ndev = 0;
  SCN_CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return scn::fail(SCN_ERR_CUDA, "no CUDA device %d (have %d)", device, ndev);
  SCN_CUDA_TRY(cudaSetDevice(device));
  std::unique_ptr<scn_freespace> h(new scn_freespace());
  h->p = *p; h->device = device; h->depth_shift = depth_shift; h->nvox = nvox;
  FsParams& fs = h->fs;
  fs.vs = p->voxel_size; fs.band_base = p->band_base; fs.band_scale = p->band_scale; fs.maxd = p->max_distance;
  fs.W = width; fs.H = height; fs.Wf = (float)width; fs.Hf = (float)height;
  uint64_t n_bricks = 1;
  for (int a = 0; a < 3; ++a) {
    h->lo[a] = lo[a]; h->dims[a] = dims[a];
    fs.lo[a] = lo[a]; fs.dims[a] = (unsigned)dims[a];
    const int64_t b0 = floor_div8(lo[a]), b1 = dims[a] ? floor_div8((int64_t)lo[a] + (int64_t)dims[a] - 1) : b0 - 1;
    fs.blo[a] = (int)b0; fs.nb[a] = (unsigned)(b1 - b0 + 1);
    n_bricks *= fs.nb[a];
  }
  fs.n_bricks = nvox ? n_bricks : 0;
  fs.cull_r = (3.5 * std::sqrt(3.0) + 0.5) * (double)p->voxel_size + 1e-3;
  fs.zfar = (double)p->max_distance + ((double)p->band_scale * p->max_distance + p->band_base);
  cudaDeviceProp prop{};
  SCN_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  h->grid = (int)std::max<uint64_t>(1, std::min<uint64_t>(fs.n_bricks, (uint64_t)prop.multiProcessorCount * 16));
  SCN_ALLOC(h->cnt, nvox * 8);
  SCN_ALLOC(h->box, 8 * 4);
  SCN_ALLOC(h->pairs, 8);
  SCN_ALLOC(h->lut, 65536 * 4);
  SCN_CUDA_TRY(scn::create(h->stream, nullptr, 0));
  SCN_CUDA_TRY(scn::create(h->ev0));
  SCN_CUDA_TRY(scn::create(h->ev1));
  // every initialisation on the handle's (non-blocking) stream, which also runs the kernels; complete before the handle is returned
  std::vector<float> lut;
  scn_tsdf_detail::make_depth_lut(depth_shift, p->depth_min, p->depth_max, lut);
  lut[0] = NAN;                                                     // raw 0 is no measurement, whatever the range
  SCN_CUDA_TRY(cudaMemcpyAsync(h->lut.p, lut.data(), 65536 * 4, cudaMemcpyHostToDevice, h->stream.get()));
  SCN_CUDA_TRY(cudaMemsetAsync(h->cnt.p, 0, nvox * 8, h->stream.get()));
  SCN_CUDA_TRY(cudaMemsetAsync(h->pairs.p, 0, 8, h->stream.get()));
  SCN_CUDA_TRY(cudaStreamSynchronize(h->stream.get()));
  for (int a = 0; a < 3; ++a) { h->rep.envelope_lo[a] = lo[a]; h->rep.envelope_dims[a] = dims[a]; }
  *out = h.release();
  return SCN_OK;
}

void scn_freespace_destroy(scn_freespace* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream.get());
  delete h;
}

int scn_freespace_integrate_device(scn_freespace* h, uint32_t n, const uint16_t* d_depth, const float* cam2world, const float K[16]) {
  if (!h || (n && (!d_depth || !cam2world)) || !K) return scn::fail(SCN_ERR_ARG, "null argument");
  return integrate_frames(h, n, cam2world, K, [&](const std::vector<uint32_t>&, const BatchParams&, const uint16_t** base) {
    *base = d_depth;
    return SCN_OK;
  });
}

int scn_freespace_integrate(scn_freespace* h, uint32_t n, const uint16_t* depth, const float* cam2world, const float K[16]) {
  if (!h || (n && (!depth || !cam2world)) || !K) return scn::fail(SCN_ERR_ARG, "null argument");
  SCN_CUDA_TRY(cudaSetDevice(h->device));
  const size_t px = (size_t)h->fs.W * h->fs.H;
  if (!h->staging.p) SCN_ALLOC(h->staging, (size_t)kMaxBatch * px * 2);
  if (!h->h_staging) SCN_CUDA_TRY(scn::create(h->h_staging, (size_t)kMaxBatch * px * 2));
  return integrate_frames(h, n, cam2world, K, [&](const std::vector<uint32_t>& idx, BatchParams& bp, const uint16_t** base) {
    // The batch's frames, packed into pinned memory and sent in ONE copy on the handle's stream, which orders it before the
    // classify kernel of this batch and after the previous batch's.  The pinned buffer itself is free again once the previous
    // copy has completed.
    SCN_CUDA_TRY(cudaStreamSynchronize(h->stream.get()));
    for (size_t j = 0; j < idx.size(); ++j) {
      memcpy(h->h_staging.get() + j * px, depth + (size_t)idx[j] * px, px * 2);
      bp.f[j].src = (int)j;
    }
    SCN_CUDA_TRY(cudaMemcpyAsync(h->staging.p, h->h_staging.get(), idx.size() * px * 2, cudaMemcpyHostToDevice, h->stream.get()));
    *base = h->staging.as<uint16_t>();
    return SCN_OK;
  });
}

int scn_freespace_download(scn_freespace* h, int32_t lo_out[3], uint64_t dims_out[3], uint8_t** labels, uint32_t** n_free, uint32_t** n_occ) {
  if (!h || !lo_out || !dims_out || !labels) return scn::fail(SCN_ERR_ARG, "null argument");
  const double t0 = now_s();
  SCN_CUDA_TRY(cudaSetDevice(h->device));
  const cudaStream_t st = h->stream.get();
  unsigned box[8] = {~0u, ~0u, ~0u, 0u, 0u, 0u, 0u, 0u};
  if (h->nvox) {
    SCN_CUDA_TRY(cudaMemcpyAsync(h->box.p, box, sizeof(box), cudaMemcpyHostToDevice, st));
    k_box<<<(unsigned)std::min<uint64_t>((h->nvox + 255) / 256, 4096), 256, 0, st>>>(h->cnt.as<uint2>(), (unsigned)h->dims[0], (unsigned)h->dims[1],
                                                                                     h->nvox, h->box.as<unsigned>());
    SCN_CUDA_TRY(cudaGetLastError());
    SCN_CUDA_TRY(cudaMemcpyAsync(box, h->box.p, sizeof(box), cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
  }
  int32_t olo[3] = {0, 0, 0};
  uint64_t od[3] = {0, 0, 0};
  const bool empty = box[0] == ~0u;
  if (!empty)
    for (int a = 0; a < 3; ++a) { olo[a] = h->lo[a] + (int32_t)box[a]; od[a] = (uint64_t)(box[3 + a] - box[a]) + 1; }
  const uint64_t n = od[0] * od[1] * od[2];
  scn::MallocPtr<uint8_t> hl;
  scn::MallocPtr<uint32_t> hf, ho;
  if (n) {
    const bool counts = n_free || n_occ;
    scn::DBuf dl, df, dn;
    SCN_ALLOC(dl, n);
    if (counts) { SCN_ALLOC(df, n * 4); SCN_ALLOC(dn, n * 4); }
    k_gather<<<(unsigned)std::min<uint64_t>((n + 255) / 256, 4096), 256, 0, st>>>(
        h->cnt.as<uint2>(), (unsigned)h->dims[0], (unsigned)h->dims[1], make_uint3(box[0], box[1], box[2]),
        make_uint3((unsigned)od[0], (unsigned)od[1], (unsigned)od[2]), n, dl.as<uint8_t>(), counts ? df.as<unsigned>() : nullptr,
        counts ? dn.as<unsigned>() : nullptr);
    SCN_CUDA_TRY(cudaGetLastError());
    hl.reset((uint8_t*)malloc(n));
    if (!hl) return scn::fail(SCN_ERR_ARG, "out of host memory (%llu bytes)", (unsigned long long)n);   // the library's code for a failed malloc (mc.cu, meshclean.cu, segs.cu)
    SCN_CUDA_TRY(cudaMemcpyAsync(hl.get(), dl.p, n, cudaMemcpyDeviceToHost, st));
    if (n_free) { hf.reset((uint32_t*)malloc(n * 4)); if (!hf) return scn::fail(SCN_ERR_ARG, "out of host memory");
                  SCN_CUDA_TRY(cudaMemcpyAsync(hf.get(), df.p, n * 4, cudaMemcpyDeviceToHost, st)); }
    if (n_occ) { ho.reset((uint32_t*)malloc(n * 4)); if (!ho) return scn::fail(SCN_ERR_ARG, "out of host memory");
                 SCN_CUDA_TRY(cudaMemcpyAsync(ho.get(), dn.p, n * 4, cudaMemcpyDeviceToHost, st)); }
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
  }
  for (int a = 0; a < 3; ++a) {
    lo_out[a] = olo[a]; dims_out[a] = od[a];
    h->rep.output_lo[a] = olo[a]; h->rep.output_dims[a] = od[a];
  }
  h->rep.voxels_free = box[6]; h->rep.voxels_occupied = box[7];
  h->rep.voxels_unknown = n - box[6] - box[7];
  *labels = hl.release();
  if (n_free) *n_free = hf.release();
  if (n_occ) *n_occ = ho.release();
  h->rep.crop_ms = (now_s() - t0) * 1e3;
  return SCN_OK;
}

int scn_freespace_handle_report(const scn_freespace* h, scn_freespace_report_t* r) {
  if (!h || !r) return scn::fail(SCN_ERR_ARG, "null argument");
  SCN_CUDA_TRY(cudaSetDevice(h->device));
  SCN_CUDA_TRY(cudaStreamSynchronize(h->stream.get()));
  *r = h->rep;
  uint64_t classified = 0;
  if (int rc = read_pairs(h, &classified)) return rc;
  r->pairs_classified = classified;
  r->pairs_culled = h->rep.pairs_culled - classified;
  return SCN_OK;
}

}  // extern "C"
