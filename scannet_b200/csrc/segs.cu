// segs.json consumers on the GPU (SURVEY.md §8f-4): what the annotation tools do with Segmentator's ids.
//
//   scn_segs_aggregate           Segmentation::m_segIdsToVertIds (AnnotationTools/common/Segmentation.h:70-75) and
//                                computeSurfaceAreaPerSegment (Segmentation.h:113-147)
//   scn_segs_objects_per_vertex  Visualizer::computeObjectIdsAndColorsPerVertex, the id assignment loop
//                                (AnnotationTools/ProjectAnnotations/Visualizer.cpp:284-297)
//   scn_mesh_vertex_normals      mLib MeshData::computeVertexNormals (external/mLib/include/core-mesh/meshData.h:758-782)
//   scn_propagate_labels         Visualizer::propagateAnnotations (Visualizer.cpp:308-377), exact 3-NN on a uniform grid
//
// The reference builds hash maps of vectors on one thread; here everything is a stable LSD radix sort (hand-written
// below: per-tile digit histograms, one device-wide scan, rank-preserving scatter) followed by flat segmented passes.
// Integer outputs (ids, vertex lists, labels) are exact; float normals are bit-identical to the sequential loop; areas
// carry a tolerance because the reference itself adds them in hash-map order.
#include <algorithm>
#include <cmath>
#include <vector>

#include "radix_sort.cuh"
#include "scan.cuh"
#include "scn_common.h"

namespace {

// stable LSD radix sort: radix_sort.cuh
using namespace scn;

// ------------------------------------------------------------------------------------------ aggregate
__global__ void k_heads(const unsigned* __restrict__ sk, size_t n, unsigned* __restrict__ head) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || sk[i] != sk[i - 1]) ? 1u : 0u;
}
// idx[i] = exclusive scan of head = (dense segment index of element i) - (head ? 0 : 1) + ...; with an exclusive scan the
// dense index of element i is idx[i] + head[i] - 1.
__global__ void k_emit_segments(const unsigned* __restrict__ sk, const unsigned* __restrict__ sv, const unsigned* __restrict__ head,
                                const unsigned* __restrict__ idx, size_t n, unsigned* __restrict__ seg_ids,
                                unsigned long long* __restrict__ offsets, unsigned* __restrict__ dense_of_vertex) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned d = idx[i] + head[i] - 1u;
  if (head[i]) { seg_ids[d] = sk[i]; offsets[d] = i; }
  dense_of_vertex[sv[i]] = d;
  if (i == n - 1) offsets[d + 1] = n;
}

// Trianglef::getArea (mLib core-graphics/triangle.h:23-35), literal: 0.5*|ab||ac|*sin(acos(cos)), 0 when |cos| is within 1e-5 of 1
__device__ __forceinline__ float tri_area_mlib(const float* a, const float* b, const float* c) {
  const float abx = __fsub_rn(b[0], a[0]), aby = __fsub_rn(b[1], a[1]), abz = __fsub_rn(b[2], a[2]);
  const float acx = __fsub_rn(c[0], a[0]), acy = __fsub_rn(c[1], a[1]), acz = __fsub_rn(c[2], a[2]);
  const float lab = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(abx, abx), __fmul_rn(aby, aby)), __fmul_rn(abz, abz)));
  const float lac = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(acx, acx), __fmul_rn(acy, acy)), __fmul_rn(acz, acz)));
  const float len = __fmul_rn(lab, lac);
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(abx, acx), __fmul_rn(aby, acy)), __fmul_rn(abz, acz));
  const float ct = __fdiv_rn(dot, len);
  if (fabsf(__fadd_rn(ct, 1.0f)) < 0.00001f || fabsf(__fsub_rn(ct, 1.0f)) < 0.00001f) return 0.f;
  const float th = acosf(ct);
  return __fmul_rn(__fmul_rn(0.5f, len), sinf(th));
}

__global__ void k_face_keys(const float* __restrict__ xyz, const unsigned* __restrict__ tri, size_t nF, size_t nV,
                            const unsigned* __restrict__ dense, unsigned nS, unsigned* __restrict__ key, unsigned* __restrict__ fid,
                            float* __restrict__ area) {
  const size_t f = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (f >= nF) return;
  const unsigned i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
  unsigned k = nS; float a = 0.f;
  if (i0 < nV && i1 < nV && i2 < nV) {
    const unsigned d0 = dense[i0];
    if (d0 == dense[i1] && d0 == dense[i2]) { k = d0; a = tri_area_mlib(xyz + 3 * (size_t)i0, xyz + 3 * (size_t)i1, xyz + 3 * (size_t)i2); }
  }
  key[f] = k; fid[f] = (unsigned)f; area[f] = a;
}

__device__ __forceinline__ size_t lower_bound_u32(const unsigned* a, size_t n, unsigned x) {
  size_t lo = 0, hi = n;
  while (lo < hi) { const size_t m = (lo + hi) >> 1; if (a[m] < x) lo = m + 1; else hi = m; }
  return lo;
}

// one warp per segment: lane l adds faces l, l+32, ... of the segment's run (ascending face id), then a fixed shuffle tree:
// the summation order depends only on the data, never on scheduling.
__global__ void k_segment_area(const unsigned* __restrict__ skey, const unsigned* __restrict__ sfid, size_t nF,
                               const float* __restrict__ area, unsigned nS, float* __restrict__ out) {
  const size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= nS) return;
  const size_t b = lower_bound_u32(skey, nF, (unsigned)w), e = lower_bound_u32(skey, nF, (unsigned)w + 1u);
  double s = 0.0;
  for (size_t i = b + lane; i < e; i += 32) s += (double)area[sfid[i]];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (lane == 0) out[w] = (float)s;
}

// ------------------------------------------------------------------------------------------ objects per vertex
__global__ void k_objects(const unsigned* __restrict__ seg, size_t nV, const unsigned* __restrict__ tab_seg,
                          const unsigned* __restrict__ tab_obj, size_t nT, unsigned* __restrict__ obj) {
  const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (v >= nV) return;
  const unsigned s = seg[v];
  const size_t p = lower_bound_u32(tab_seg, nT, s);
  obj[v] = (p < nT && tab_seg[p] == s) ? tab_obj[p] : 0u;
}

// ------------------------------------------------------------------------------------------ mLib vertex normals
__global__ void k_face_normals_mlib(const float* __restrict__ xyz, const unsigned* __restrict__ tri, size_t nF,
                                    float4* __restrict__ fn, unsigned* __restrict__ deg) {
  const size_t f = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (f >= nF) return;
  const unsigned i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
  const float* p0 = xyz + 3 * (size_t)i0; const float* p1 = xyz + 3 * (size_t)i1; const float* p2 = xyz + 3 * (size_t)i2;
  const float ux = __fsub_rn(p1[0], p0[0]), uy = __fsub_rn(p1[1], p0[1]), uz = __fsub_rn(p1[2], p0[2]);
  const float vx = __fsub_rn(p2[0], p0[0]), vy = __fsub_rn(p2[1], p0[1]), vz = __fsub_rn(p2[2], p0[2]);
  // n = 0 + (u ^ v)  (vec3.h:154-156); the += onto a zero vector is exact except that -0 becomes +0
  float cx = __fadd_rn(0.f, __fsub_rn(__fmul_rn(uy, vz), __fmul_rn(uz, vy)));
  float cy = __fadd_rn(0.f, __fsub_rn(__fmul_rn(uz, vx), __fmul_rn(ux, vz)));
  float cz = __fadd_rn(0.f, __fsub_rn(__fmul_rn(ux, vy), __fmul_rn(uy, vx)));
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
  const float inv = __fdiv_rn(1.0f, len);                                   // vec3.h:238-243
  fn[f] = make_float4(__fmul_rn(cx, inv), __fmul_rn(cy, inv), __fmul_rn(cz, inv), 0.f);
  atomicAdd(&deg[i0], 1u); atomicAdd(&deg[i1], 1u); atomicAdd(&deg[i2], 1u);
}

__global__ void k_fill_corners(const unsigned* __restrict__ tri, size_t nC, const unsigned* __restrict__ off,
                               unsigned* __restrict__ cursor, unsigned* __restrict__ csr) {
  const size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (c >= nC) return;
  const unsigned v = tri[c];
  csr[off[v] + atomicAdd(&cursor[v], 1u)] = (unsigned)c;
}

__device__ void sift_u32(unsigned* a, unsigned hole, unsigned len, unsigned val) {
  for (;;) {
    unsigned child = 2 * hole + 1;
    if (child >= len) break;
    if (child + 1 < len && a[child + 1] > a[child]) ++child;
    if (a[child] <= val) break;
    a[hole] = a[child]; hole = child;
  }
  a[hole] = val;
}

// one thread per vertex: order its corners ascending (= face order, corner order inside a face), add, normalise
__global__ void k_vertex_normals_mlib(const unsigned* __restrict__ off, unsigned* __restrict__ csr, const float4* __restrict__ fn,
                                      size_t nV, float* __restrict__ nrm) {
  const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (v >= nV) return;
  const unsigned b = off[v], n = off[v + 1] - b;
  unsigned* lst = csr + b;
  if (n <= 24) { for (unsigned i = 1; i < n; ++i) { const unsigned c = lst[i]; unsigned j = i; while (j > 0 && lst[j - 1] > c) { lst[j] = lst[j - 1]; --j; } lst[j] = c; } }
  else {
    for (unsigned p = n / 2; p-- > 0;) sift_u32(lst, p, n, lst[p]);
    for (unsigned last = n; last > 1;) { --last; const unsigned t = lst[last]; lst[last] = lst[0]; sift_u32(lst, 0, last, t); }
  }
  float x = 0.f, y = 0.f, z = 0.f;
  for (unsigned i = 0; i < n; ++i) { const float4 q = fn[lst[i] / 3u]; x = __fadd_rn(x, q.x); y = __fadd_rn(y, q.y); z = __fadd_rn(z, q.z); }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  const float inv = __fdiv_rn(1.0f, len);
  nrm[3 * v] = __fmul_rn(x, inv); nrm[3 * v + 1] = __fmul_rn(y, inv); nrm[3 * v + 2] = __fmul_rn(z, inv);
}

// ------------------------------------------------------------------------------------------ label propagation
struct Grid { float minx, miny, minz, inv; int nx, ny, nz; };

__device__ __forceinline__ int cell_coord(float p, float mn, float inv, int n) {
  const float t = floorf(__fmul_rn(__fsub_rn(p, mn), inv));
  return t < 0.f ? 0 : (t >= (float)n ? n - 1 : (int)t);
}

__global__ void k_cell_keys(const float* __restrict__ xyz, const unsigned* __restrict__ obj, size_t n, Grid g,
                            unsigned* __restrict__ key, unsigned* __restrict__ val, unsigned* __restrict__ count) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned ncell = (unsigned)(g.nx * g.ny * g.nz);
  unsigned k = ncell;                                                      // unlabelled vertices sort behind every cell
  const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  if (obj[i] > 0u && x == x && y == y && z == z) {
    k = (unsigned)((cell_coord(z, g.minz, g.inv, g.nz) * g.ny + cell_coord(y, g.miny, g.inv, g.ny)) * g.nx + cell_coord(x, g.minx, g.inv, g.nx));
    atomicAdd(&count[k], 1u);
  }
  key[i] = k; val[i] = (unsigned)i;
}

__global__ void k_propagate(const float* __restrict__ sxyz, const float* __restrict__ snrm, const unsigned* __restrict__ sobj,
                            const unsigned* __restrict__ order, const unsigned* __restrict__ cell_start, Grid g,
                            const float* __restrict__ dxyz, const float* __restrict__ dnrm, size_t nD, float max_thresh,
                            float normal_thresh, unsigned* __restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= nD) return;
  const float px = dxyz[3 * i], py = dxyz[3 * i + 1], pz = dxyz[3 * i + 2];
  float bd[3] = {INFINITY, INFINITY, INFINITY}; unsigned bi[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  if (px == px && py == py && pz == pz) {
    // cells whose points can lie within max_thresh: cell edge is a hair above max_thresh, so +-1 around the query's cell
    const float fx = floorf(__fmul_rn(__fsub_rn(px, g.minx), g.inv)), fy = floorf(__fmul_rn(__fsub_rn(py, g.miny), g.inv)),
                fz = floorf(__fmul_rn(__fsub_rn(pz, g.minz), g.inv));
    if (fx >= -1.f && fy >= -1.f && fz >= -1.f && fx <= (float)g.nx && fy <= (float)g.ny && fz <= (float)g.nz) {
      const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
      for (int z = max(cz - 1, 0); z <= min(cz + 1, g.nz - 1); ++z)
        for (int y = max(cy - 1, 0); y <= min(cy + 1, g.ny - 1); ++y) {
          const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
          if (x0 > x1) continue;
          const unsigned c0 = (unsigned)((z * g.ny + y) * g.nx + x0), c1 = (unsigned)((z * g.ny + y) * g.nx + x1);
          for (unsigned q = cell_start[c0]; q < cell_start[c1 + 1]; ++q) {       // the x-run of cells is contiguous in the sorted order
            const unsigned s = order[q];
            const float dx = __fsub_rn(sxyz[3 * (size_t)s], px), dy = __fsub_rn(sxyz[3 * (size_t)s + 1], py), dz = __fsub_rn(sxyz[3 * (size_t)s + 2], pz);
            const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            if (!(d < max_thresh)) continue;
            // insert by (distance, source index)
            if (d < bd[2] || (d == bd[2] && s < bi[2])) {
              bd[2] = d; bi[2] = s;
              if (bd[2] < bd[1] || (bd[2] == bd[1] && bi[2] < bi[1])) { float t = bd[1]; bd[1] = bd[2]; bd[2] = t; unsigned u = bi[1]; bi[1] = bi[2]; bi[2] = u; }
              if (bd[1] < bd[0] || (bd[1] == bd[0] && bi[1] < bi[0])) { float t = bd[0]; bd[0] = bd[1]; bd[1] = t; unsigned u = bi[0]; bi[0] = bi[1]; bi[1] = u; }
            }
          }
        }
    }
  }
  // decision rule, Visualizer.cpp:346-371 (neighbours that are not closer than maxThresh only clear `allSame`)
  unsigned res = 0u;
  if (bi[0] != 0xFFFFFFFFu) {
    const unsigned val = sobj[bi[0]];
    bool all_same = true; int best = -1;
    const float nx = dnrm[3 * i], ny = dnrm[3 * i + 1], nz = dnrm[3 * i + 2];
    for (int k = 0; k < 3; ++k) {
      if (bi[k] != 0xFFFFFFFFu) {
        const float* sn = snrm + 3 * (size_t)bi[k];
        float dot = __fadd_rn(__fadd_rn(__fmul_rn(sn[0], nx), __fmul_rn(sn[1], ny)), __fmul_rn(sn[2], nz));
        dot = dot < -1.0f ? -1.0f : (dot > 1.0f ? 1.0f : dot);                 // math::clamp
        if (acosf(dot) < normal_thresh) { best = k; break; }
        if (sobj[bi[k]] != val) all_same = false;
      } else all_same = false;
    }
    if (best >= 0) res = sobj[bi[best]]; else if (all_same) res = val;
  }
  out[i] = res;
}

}  // namespace

extern "C" {

int scn_segs_aggregate(const uint32_t* seg, uint64_t nV, const float* xyz, const uint32_t* tri, uint64_t nF,
                       uint32_t** seg_ids_out, uint64_t* n_segs, uint64_t** vert_offsets, uint32_t** vert_ids, float** area_out) {
  if (!seg || !seg_ids_out || !n_segs || !vert_offsets || !vert_ids) return scn::fail(SCN_ERR_ARG, "scn_segs_aggregate: null argument");
  if (nV > 0x7FFFFFFFull || nF > 0x7FFFFFFFull) return scn::fail(SCN_ERR_ARG, "scn_segs_aggregate: mesh too large");
  const bool want_area = area_out && xyz && tri;
  *seg_ids_out = nullptr; *vert_offsets = nullptr; *vert_ids = nullptr; *n_segs = 0; if (area_out) *area_out = nullptr;
  if (nV == 0) { *vert_offsets = (uint64_t*)calloc(1, 8); return SCN_OK; }
  unsigned maxv = 0; for (uint64_t i = 0; i < nV; ++i) maxv = std::max(maxv, seg[i]);
  cudaStream_t st = 0;
  const size_t nmax = std::max<size_t>(nV, want_area ? nF : 0);
  Scratch s; DBuf head, idx, dense, dsegids, doff;
  if (int rc = s.ensure(nmax, nmax + 1)) return rc;
  SCN_ALLOC(head, nV * 4); SCN_ALLOC(idx, (nV + 1) * 4); SCN_ALLOC(dense, nV * 4); SCN_ALLOC(dsegids, nV * 4); SCN_ALLOC(doff, (nV + 1) * 8);
  unsigned *k0 = s.k0.as<unsigned>(), *v0 = s.v0.as<unsigned>(), *k1 = s.k1.as<unsigned>(), *v1 = s.v1.as<unsigned>();
  SCN_CUDA_TRY(cudaMemcpyAsync(k0, seg, nV * 4, cudaMemcpyHostToDevice, st));
  k_iota<<<grid_for(nV), 256, 0, st>>>(v0, nV);
  const int w = radix_sort_pairs(k0, v0, k1, v1, nV, bits_for(maxv), s.hist.as<unsigned>(), s.scr.as<unsigned>(), st);
  unsigned* sk = w ? k1 : k0; unsigned* sv = w ? v1 : v0;
  k_heads<<<grid_for(nV), 256, 0, st>>>(sk, nV, head.as<unsigned>());
  scn::exclusive_scan_u32(head.as<unsigned>(), idx.as<unsigned>(), nV, s.scr.as<unsigned>(), st);
  k_emit_segments<<<grid_for(nV), 256, 0, st>>>(sk, sv, head.as<unsigned>(), idx.as<unsigned>(), nV, dsegids.as<unsigned>(),
                                                doff.as<unsigned long long>(), dense.as<unsigned>());
  unsigned nS = 0;
  SCN_CUDA_TRY(cudaMemcpyAsync(&nS, idx.as<unsigned>() + nV, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  MallocPtr<uint32_t> h_ids((uint32_t*)malloc((size_t)nS * 4)); MallocPtr<uint64_t> h_off((uint64_t*)malloc(((size_t)nS + 1) * 8));
  MallocPtr<uint32_t> h_vid((uint32_t*)malloc(nV * 4)); MallocPtr<float> h_area(want_area ? (float*)malloc((size_t)nS * 4) : nullptr);
  if (!h_ids || !h_off || !h_vid || (want_area && !h_area)) return scn::fail(SCN_ERR_ARG, "scn_segs_aggregate: out of host memory");
  if (cudaMemcpyAsync(h_ids.get(), dsegids.p, (size_t)nS * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaMemcpyAsync(h_off.get(), doff.p, ((size_t)nS + 1) * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaMemcpyAsync(h_vid.get(), sv, nV * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
    return scn::fail(SCN_ERR_CUDA, "scn_segs_aggregate: download failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (want_area) {
    DBuf dxyz, dtri, darea, dout;
    if (!dxyz.alloc(nV * 12) || !dtri.alloc(std::max<size_t>(nF, 1) * 12) || !darea.alloc(std::max<size_t>(nF, 1) * 4) || !dout.alloc((size_t)nS * 4))
      return scn::fail(SCN_ERR_CUDA, "scn_segs_aggregate: cudaMalloc failed");
    cudaMemcpyAsync(dxyz.p, xyz, nV * 12, cudaMemcpyHostToDevice, st);
    if (nF) cudaMemcpyAsync(dtri.p, tri, nF * 12, cudaMemcpyHostToDevice, st);
    unsigned* fk = sk == k0 ? k1 : k0;     // the buffers not holding the sorted vertex lists
    unsigned* fv = sk == k0 ? v1 : v0;
    // sort faces by dense segment index; needs a second pair of buffers
    DBuf fk2, fv2;
    if (!fk2.alloc(std::max<size_t>(nF, 1) * 4) || !fv2.alloc(std::max<size_t>(nF, 1) * 4)) return scn::fail(SCN_ERR_CUDA, "scn_segs_aggregate: cudaMalloc failed");
    const unsigned* skey = fk; const unsigned* sfid = fv;
    if (nF) {
      k_face_keys<<<grid_for(nF), 256, 0, st>>>(dxyz.as<float>(), dtri.as<unsigned>(), nF, nV, dense.as<unsigned>(), nS, fk, fv, darea.as<float>());
      const int w2 = radix_sort_pairs(fk, fv, fk2.as<unsigned>(), fv2.as<unsigned>(), nF, bits_for(nS), s.hist.as<unsigned>(), s.scr.as<unsigned>(), st);
      if (w2) { skey = fk2.as<unsigned>(); sfid = fv2.as<unsigned>(); }
    }
    k_segment_area<<<(unsigned)(((size_t)nS * 32 + 255) / 256), 256, 0, st>>>(skey, sfid, nF, darea.as<float>(), nS, dout.as<float>());
    if (cudaMemcpyAsync(h_area.get(), dout.p, (size_t)nS * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
      return scn::fail(SCN_ERR_CUDA, "scn_segs_aggregate: area pass failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess)
    return scn::fail(SCN_ERR_CUDA, "scn_segs_aggregate: kernel failed");
  *seg_ids_out = h_ids.release(); *n_segs = nS; *vert_offsets = h_off.release(); *vert_ids = h_vid.release(); if (area_out) *area_out = h_area.release();
  return SCN_OK;
}

int scn_segs_objects_per_vertex(const uint32_t* seg, uint64_t nV, const uint32_t* group_segs, const uint64_t* group_offsets,
                                uint64_t n_groups, uint32_t* obj_out) {
  if (!seg || !obj_out || (n_groups && (!group_offsets || !group_segs))) return scn::fail(SCN_ERR_ARG, "scn_segs_objects_per_vertex: null argument");
  if (nV == 0) return SCN_OK;
  // (segment id -> object id) table, later groups win (the reference overwrites colours group after group)
  std::vector<std::pair<uint32_t, uint32_t>> tab;
  for (uint64_t g = 0; g < n_groups; ++g) {
    if (group_offsets[g + 1] < group_offsets[g]) return scn::fail(SCN_ERR_ARG, "scn_segs_objects_per_vertex: group offsets not monotone");
    for (uint64_t j = group_offsets[g]; j < group_offsets[g + 1]; ++j) tab.emplace_back(group_segs[j], (uint32_t)(g + 1));
  }
  std::stable_sort(tab.begin(), tab.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  std::vector<uint32_t> ts, to;
  for (size_t i = 0; i < tab.size(); ++i) if (i + 1 == tab.size() || tab[i + 1].first != tab[i].first) { ts.push_back(tab[i].first); to.push_back(tab[i].second); }
  cudaStream_t st = 0;
  DBuf dseg, dts, dto, dobj;
  SCN_ALLOC(dseg, nV * 4); SCN_ALLOC(dts, ts.size() * 4); SCN_ALLOC(dto, ts.size() * 4); SCN_ALLOC(dobj, nV * 4);
  SCN_CUDA_TRY(cudaMemcpyAsync(dseg.p, seg, nV * 4, cudaMemcpyHostToDevice, st));
  if (!ts.empty()) { SCN_CUDA_TRY(cudaMemcpyAsync(dts.p, ts.data(), ts.size() * 4, cudaMemcpyHostToDevice, st)); SCN_CUDA_TRY(cudaMemcpyAsync(dto.p, to.data(), ts.size() * 4, cudaMemcpyHostToDevice, st)); }
  k_objects<<<grid_for(nV), 256, 0, st>>>(dseg.as<unsigned>(), nV, dts.as<unsigned>(), dto.as<unsigned>(), ts.size(), dobj.as<unsigned>());
  SCN_CUDA_TRY(cudaMemcpyAsync(obj_out, dobj.p, nV * 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

int scn_mesh_vertex_normals(const float* xyz, uint64_t nV, const uint32_t* tri, uint64_t nF, float* normals_out) {
  if (!xyz || !normals_out || (nF && !tri)) return scn::fail(SCN_ERR_ARG, "scn_mesh_vertex_normals: null argument");
  if (nV > 0x7FFFFFFFull || nF > 0x55555555ull) return scn::fail(SCN_ERR_ARG, "scn_mesh_vertex_normals: mesh too large");
  if (nV == 0) return SCN_OK;
  for (uint64_t c = 0; c < 3 * nF; ++c) if (tri[c] >= nV) return scn::fail(SCN_ERR_ARG, "scn_mesh_vertex_normals: face %llu references vertex %u of %llu", (unsigned long long)(c / 3), tri[c], (unsigned long long)nV);
  cudaStream_t st = 0;
  DBuf dxyz, dtri, dfn, ddeg, doff, dcur, dcsr, dscr, dn;
  SCN_ALLOC(dxyz, nV * 12); SCN_ALLOC(dtri, nF * 12); SCN_ALLOC(dfn, nF * 16); SCN_ALLOC(ddeg, nV * 4); SCN_ALLOC(doff, (nV + 1) * 4);
  SCN_ALLOC(dcur, nV * 4); SCN_ALLOC(dcsr, nF * 12); SCN_ALLOC(dscr, scn::scan_scratch_elems(nV) * 4); SCN_ALLOC(dn, nV * 12);
  SCN_CUDA_TRY(cudaMemcpyAsync(dxyz.p, xyz, nV * 12, cudaMemcpyHostToDevice, st));
  if (nF) SCN_CUDA_TRY(cudaMemcpyAsync(dtri.p, tri, nF * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemsetAsync(ddeg.p, 0, nV * 4, st)); SCN_CUDA_TRY(cudaMemsetAsync(dcur.p, 0, nV * 4, st));
  if (nF) k_face_normals_mlib<<<grid_for(nF), 256, 0, st>>>(dxyz.as<float>(), dtri.as<unsigned>(), nF, dfn.as<float4>(), ddeg.as<unsigned>());
  scn::exclusive_scan_u32(ddeg.as<unsigned>(), doff.as<unsigned>(), nV, dscr.as<unsigned>(), st);
  if (nF) k_fill_corners<<<grid_for(3 * nF), 256, 0, st>>>(dtri.as<unsigned>(), 3 * nF, doff.as<unsigned>(), dcur.as<unsigned>(), dcsr.as<unsigned>());
  k_vertex_normals_mlib<<<grid_for(nV), 256, 0, st>>>(doff.as<unsigned>(), dcsr.as<unsigned>(), dfn.as<float4>(), nV, dn.as<float>());
  SCN_CUDA_TRY(cudaMemcpyAsync(normals_out, dn.p, nV * 12, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

int scn_propagate_labels(const float* src_xyz, const float* src_normals, const uint32_t* src_obj, uint64_t nS, const float* dst_xyz,
                         const float* dst_normals, uint64_t nD, float normal_thresh, uint32_t* dst_obj_out) {
  if ((nS && (!src_xyz || !src_normals || !src_obj)) || (nD && (!dst_xyz || !dst_normals || !dst_obj_out)))
    return scn::fail(SCN_ERR_ARG, "scn_propagate_labels: null argument");
  if (nS > 0x7FFFFFFFull || nD > 0x7FFFFFFFull) return scn::fail(SCN_ERR_ARG, "scn_propagate_labels: mesh too large");
  if (nD == 0) return SCN_OK;
  if (nS == 0) { memset(dst_obj_out, 0, nD * 4); return SCN_OK; }
  // bbox over ALL source vertices (meshSrc.computeBoundingBox, Visualizer.cpp:313); maxThresh, Visualizer.cpp:335
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint64_t i = 0; i < nS; ++i) for (int k = 0; k < 3; ++k) { const float v = src_xyz[3 * i + k]; if (v < mn[k]) mn[k] = v; if (v > mx[k]) mx[k] = v; }
  float ext = 0.f; for (int k = 0; k < 3; ++k) { const float e = mx[k] - mn[k]; if (e > ext) ext = e; }
  if (!(ext >= 0.f) || std::isinf(ext)) return scn::fail(SCN_ERR_ARG, "scn_propagate_labels: source bounding box is not finite");
  const float max_thresh = std::max(ext * 0.01f, 0.05f);
  Grid g; g.minx = mn[0]; g.miny = mn[1]; g.minz = mn[2];
  const float cell = max_thresh * 1.0001f; g.inv = 1.0f / cell;
  g.nx = (int)std::floor((mx[0] - mn[0]) * g.inv) + 1; g.ny = (int)std::floor((mx[1] - mn[1]) * g.inv) + 1; g.nz = (int)std::floor((mx[2] - mn[2]) * g.inv) + 1;
  const size_t ncell = (size_t)g.nx * g.ny * g.nz;                       // <= 101^3: cell edge >= 1 % of the largest extent
  cudaStream_t st = 0;
  DBuf sx, sn, so, dx, dn, dout, cnt, cstart;
  Scratch s;
  SCN_ALLOC(sx, nS * 12); SCN_ALLOC(sn, nS * 12); SCN_ALLOC(so, nS * 4); SCN_ALLOC(dx, nD * 12); SCN_ALLOC(dn, nD * 12); SCN_ALLOC(dout, nD * 4);
  if (int rc = s.ensure(nS, ncell + 2)) return rc;
  SCN_ALLOC(cnt, (ncell + 1) * 4); SCN_ALLOC(cstart, (ncell + 2) * 4);
  SCN_CUDA_TRY(cudaMemcpyAsync(sx.p, src_xyz, nS * 12, cudaMemcpyHostToDevice, st)); SCN_CUDA_TRY(cudaMemcpyAsync(sn.p, src_normals, nS * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(so.p, src_obj, nS * 4, cudaMemcpyHostToDevice, st)); SCN_CUDA_TRY(cudaMemcpyAsync(dx.p, dst_xyz, nD * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(dn.p, dst_normals, nD * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemsetAsync(cnt.p, 0, (ncell + 1) * 4, st));
  unsigned* order = s.v0.as<unsigned>();
  k_cell_keys<<<grid_for(nS), 256, 0, st>>>(sx.as<float>(), so.as<unsigned>(), nS, g, s.k0.as<unsigned>(), order, cnt.as<unsigned>());
  sort_pass(s, order, nS, bits_for((unsigned)ncell), st);
  scn::exclusive_scan_u32(cnt.as<unsigned>(), cstart.as<unsigned>(), ncell + 1, s.scr.as<unsigned>(), st);
  k_propagate<<<grid_for(nD), 256, 0, st>>>(sx.as<float>(), sn.as<float>(), so.as<unsigned>(), order, cstart.as<unsigned>(), g,
                                            dx.as<float>(), dn.as<float>(), nD, max_thresh, normal_thresh, dout.as<unsigned>());
  SCN_CUDA_TRY(cudaMemcpyAsync(dst_obj_out, dout.p, nD * 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

}  // extern "C"
