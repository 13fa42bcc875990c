// Mesh cleaning on the GPU (DESIGN.md §6f): MeshLab's clean.mlx stage (`_vh.ply` -> `_vh_clean.ply`, Server/scan_processor.py:143)
// stated as mLib's MeshData operators (external/mLib/include/core-mesh/meshData.cpp), in clean.mlx's order:
//
//   merge   mergeCloseVertices(t, approx=false) :217-289 + removeDegeneratedFaces :293-318
//           Cells are sorted (three stable radix sorts: x, y, z), every distinct cell gets its 27 neighbour cells in mLib's scan
//           order, and a device union-find joins vertices closer than t in neighbouring cells.  The sequential rule ("a vertex
//           maps to the first earlier representative in scan order within t, else it becomes one") only ever looks at such
//           neighbours, so replaying it inside each component - one thread per component, members in index order - gives
//           exactly the sequential result.
//   dedup   removeDuplicateFaces :40-104: faces sorted stably by their sorted index triple; the first of every run survives.
//   pieces  removeIsolatedPieces :407-454 + removeIsolatedVertices :324-360: union-find over face corners, per-piece vertex and
//           face counts, then first-appearance renumbering (atomicMin of the corner index per vertex + a scan in corner order).
//
// The mesh is uploaded once and stays in device memory until the result is downloaded.  Nothing depends on scheduling: the
// union-find roots are component minima, the sorts are stable and every compaction is a scan.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "meshclean_steps.h"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "scn_common.h"

namespace scn::mc {

enum : unsigned { ERR_INDEX = 1u, ERR_CELL = 2u };
__device__ __forceinline__ size_t tid() { return blockIdx.x * (size_t)blockDim.x + threadIdx.x; }

__global__ void k_check_faces(const unsigned* __restrict__ tri, size_t nC, unsigned nV, unsigned* err) {
  const size_t c = tid();
  if (c < nC && tri[c] >= nV) atomicOr(err, ERR_INDEX);
}

// ------------------------------------------------------------------------------------------ union-find (roots = minima)
__device__ __forceinline__ unsigned uf_find(unsigned* p, unsigned x) {
  volatile unsigned* vp = p;
  for (;;) {
    const unsigned q = vp[x];
    if (q == x) return x;
    const unsigned g = vp[q];
    if (g != q) vp[x] = g;           // path halving: g is an ancestor of x, and parents only ever move towards the root
    x = q;
  }
}
__device__ __forceinline__ void uf_union(unsigned* p, unsigned a, unsigned b) {
  for (;;) {
    a = uf_find(p, a); b = uf_find(p, b);
    if (a == b) return;
    if (a < b) { const unsigned t = a; a = b; b = t; }
    const unsigned old = atomicCAS(&p[a], a, b);        // hook the larger root under the smaller one
    if (old == a) return;
  }
}
// root[v] into a separate array: a write of the root into p[v] could be overwritten by another thread's (still valid, but
// less compressed) path-halving store, and then p[v] would not name the root
__global__ void k_uf_roots(unsigned* p, unsigned n, unsigned* __restrict__ root) { const size_t v = tid(); if (v < n) root[v] = uf_find(p, (unsigned)v); }

// ------------------------------------------------------------------------------------------ step 1: merge close vertices
__device__ __forceinline__ float dist_sq(const float* a, const float* b) {               // vec3::distSq, vec3.h:199-201
  const float dx = __fsub_rn(a[0], b[0]), dy = __fsub_rn(a[1], b[1]), dz = __fsub_rn(a[2], b[2]);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__device__ __forceinline__ unsigned biased(int c) { return (unsigned)c ^ 0x80000000u; }

// toVirtualVoxelPos (meshData.h:946-948): (int)(v * (1/t) + 0.5f * sign(v)), sign(+-0) = 0, truncating conversion
__global__ void k_cells(const float* __restrict__ xyz, unsigned n, float inv, int* __restrict__ cell, unsigned* __restrict__ key,
                        unsigned* __restrict__ val, unsigned* err) {
  const size_t v = tid();
  if (v >= n) return;
  int c[3];
  for (int i = 0; i < 3; ++i) {
    const float x = xyz[3 * v + i];
    const float s = __fmul_rn(x, inv);
    if (!(fabsf(s) < 2147483648.0f)) { atomicOr(err, ERR_CELL); c[i] = 0; continue; }
    const float sg = (0.f < x) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
    c[i] = (int)__fadd_rn(s, __fmul_rn(0.5f, sg));
  }
  cell[3 * v] = c[0]; cell[3 * v + 1] = c[1]; cell[3 * v + 2] = c[2];
  key[v] = biased(c[0]); val[v] = (unsigned)v;
}
__global__ void k_gather_axis(const int* __restrict__ cell, int axis, const unsigned* __restrict__ order, unsigned n, unsigned* __restrict__ key) {
  const size_t i = tid();
  if (i < n) key[i] = biased(cell[3 * (size_t)order[i] + axis]);
}
__device__ __forceinline__ bool same_cell(const int* a, const int* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; }
__global__ void k_cell_heads(const int* __restrict__ cell, const unsigned* __restrict__ order, unsigned n, unsigned* __restrict__ head) {
  const size_t i = tid();
  if (i < n) head[i] = (i == 0 || !same_cell(cell + 3 * (size_t)order[i], cell + 3 * (size_t)order[i - 1])) ? 1u : 0u;
}
// distinct cell u = hidx[i] + head[i] - 1 holds sorted positions ustart[u] .. ustart[u+1]
__global__ void k_cell_table(const int* __restrict__ cell, const unsigned* __restrict__ order, const unsigned* __restrict__ head,
                             const unsigned* __restrict__ hidx, unsigned n, int* __restrict__ ucell, unsigned* __restrict__ ustart,
                             unsigned* __restrict__ cellidx) {
  const size_t i = tid();
  if (i >= n) return;
  const unsigned u = hidx[i] + head[i] - 1u, v = order[i];
  if (head[i]) { ucell[3 * u] = cell[3 * v]; ucell[3 * u + 1] = cell[3 * v + 1]; ucell[3 * u + 2] = cell[3 * v + 2]; ustart[u] = (unsigned)i; }
  cellidx[v] = u;
  if (i == n - 1) ustart[u + 1] = n;
}
// lexicographic (z, y, x): the order the three stable sorts produced
__device__ __forceinline__ bool cell_less(const int* a, long long x, long long y, long long z) {
  if (a[2] != z) return a[2] < z;
  if (a[1] != y) return a[1] < y;
  return a[0] < x;
}
// nb[27u + o] = distinct-cell index of neighbour o (o = (dx+1)*9 + (dy+1)*3 + (dz+1): hasNearestNeighbor's scan order,
// meshData.cpp:180-183) or -1
__global__ void k_cell_neighbours(const int* __restrict__ ucell, const unsigned* __restrict__ nU_dev, int* __restrict__ nb) {
  const unsigned nU = *nU_dev;
  const size_t u = tid();
  if (u >= nU) return;
  const int* c = ucell + 3 * u;
  for (int o = 0; o < 27; ++o) {
    const long long x = (long long)c[0] + o / 9 - 1, y = (long long)c[1] + (o / 3) % 3 - 1, z = (long long)c[2] + o % 3 - 1;
    int r = -1;
    if (x >= INT_MIN && x <= INT_MAX && y >= INT_MIN && y <= INT_MAX && z >= INT_MIN && z <= INT_MAX) {
      unsigned lo = 0, hi = nU;
      while (lo < hi) { const unsigned m = (lo + hi) >> 1; if (cell_less(ucell + 3 * (size_t)m, x, y, z)) lo = m + 1; else hi = m; }
      if (lo < nU && ucell[3 * (size_t)lo] == x && ucell[3 * (size_t)lo + 1] == y && ucell[3 * (size_t)lo + 2] == z) r = (int)lo;
    }
    nb[27 * u + o] = r;
  }
}
// union every vertex with the EARLIER vertices within t in its 27 cells (members of a cell are in ascending index order)
__global__ void k_merge_union(const float* __restrict__ xyz, const unsigned* __restrict__ cellidx, const int* __restrict__ nb,
                              const unsigned* __restrict__ ustart, const unsigned* __restrict__ order, unsigned n, float tsq, unsigned* par) {
  const size_t v = tid();
  if (v >= n) return;
  const unsigned k = cellidx[v];
  const float* pv = xyz + 3 * v;
  for (int o = 0; o < 27; ++o) {
    const int c = nb[27 * (size_t)k + o];
    if (c < 0) continue;
    for (unsigned q = ustart[c], e = ustart[c + 1]; q < e; ++q) {
      const unsigned u = order[q];
      if (u >= v) break;
      if (dist_sq(pv, xyz + 3 * (size_t)u) < tsq) uf_union(par, u, (unsigned)v);
    }
  }
}
__global__ void k_count_roots(const unsigned* __restrict__ root, unsigned n, unsigned* __restrict__ size) {
  const size_t v = tid();
  if (v < n) atomicAdd(&size[root[v]], 1u);
}
// stats[0] = largest component, stats[1] = components of >= 2 vertices
__global__ void k_component_stats(const unsigned* __restrict__ root, const unsigned* __restrict__ size, unsigned n, unsigned* stats) {
  const size_t v = tid();
  if (v >= n || root[v] != v) return;
  atomicMax(&stats[0], size[v]);
  if (size[v] >= 2) atomicAdd(&stats[1], 1u);
}
// One thread per component (sorted by root, members ascending): the sequential rule.  rep[] and target[] of earlier members
// were written by this same thread; every vertex within t of v is in v's component.
__global__ void k_merge_replay(const unsigned* __restrict__ sroot, const unsigned* __restrict__ smember, unsigned n,
                               const float* __restrict__ xyz, const unsigned* __restrict__ cellidx, const int* __restrict__ nb,
                               const unsigned* __restrict__ ustart, const unsigned* __restrict__ order, float tsq,
                               unsigned* rep, unsigned* __restrict__ target) {
  const size_t i = tid();
  if (i >= n || (i > 0 && sroot[i] == sroot[i - 1])) return;
  const unsigned r = sroot[i];
  if (i + 1 == n || sroot[i + 1] != r) { const unsigned v = smember[i]; rep[v] = 1u; target[v] = v; return; }   // alone
  for (size_t j = i; j < n && sroot[j] == r; ++j) {
    const unsigned v = smember[j], k = cellidx[v];
    const float* pv = xyz + 3 * (size_t)v;
    unsigned t = v;
    for (int o = 0; o < 27 && t == v; ++o) {
      const int c = nb[27 * (size_t)k + o];
      if (c < 0) continue;
      for (unsigned q = ustart[c], e = ustart[c + 1]; q < e; ++q) {
        const unsigned u = order[q];
        if (u >= v) break;
        if (dist_sq(pv, xyz + 3 * (size_t)u) < tsq && rep[u]) { t = u; break; }
      }
    }
    rep[v] = t == v ? 1u : 0u;
    target[v] = t;
  }
}
__global__ void k_merge_vertices(const float* __restrict__ xyz, const unsigned char* __restrict__ rgb, const unsigned* __restrict__ rep,
                                 const unsigned* __restrict__ newid, unsigned n, float* __restrict__ oxyz, unsigned char* __restrict__ orgb) {
  const size_t v = tid();
  if (v >= n || !rep[v]) return;
  const unsigned d = newid[v];
  oxyz[3 * (size_t)d] = xyz[3 * v]; oxyz[3 * (size_t)d + 1] = xyz[3 * v + 1]; oxyz[3 * (size_t)d + 2] = xyz[3 * v + 2];
  if (rgb) { orgb[3 * (size_t)d] = rgb[3 * v]; orgb[3 * (size_t)d + 1] = rgb[3 * v + 1]; orgb[3 * (size_t)d + 2] = rgb[3 * v + 2]; }
}
__global__ void k_merge_faces(const unsigned* __restrict__ tri, unsigned nF, const unsigned* __restrict__ target,
                              const unsigned* __restrict__ newid, unsigned* __restrict__ otri, unsigned* __restrict__ keep) {
  const size_t f = tid();
  if (f >= nF) return;
  const unsigned a = newid[target[tri[3 * f]]], b = newid[target[tri[3 * f + 1]]], c = newid[target[tri[3 * f + 2]]];
  otri[3 * f] = a; otri[3 * f + 1] = b; otri[3 * f + 2] = c;
  keep[f] = (a != b && a != c && b != c) ? 1u : 0u;                                // removeDegeneratedFaces
}
__global__ void k_compact_faces(const unsigned* __restrict__ tri, const unsigned* __restrict__ keep, const unsigned* __restrict__ pos,
                                unsigned nF, unsigned* __restrict__ otri) {
  const size_t f = tid();
  if (f >= nF || !keep[f]) return;
  const unsigned d = pos[f];
  otri[3 * (size_t)d] = tri[3 * f]; otri[3 * (size_t)d + 1] = tri[3 * f + 1]; otri[3 * (size_t)d + 2] = tri[3 * f + 2];
}

// ------------------------------------------------------------------------------------------ step 2: duplicate faces
__device__ __forceinline__ void sorted3(const unsigned* t, unsigned& a, unsigned& b, unsigned& c) {
  a = t[0]; b = t[1]; c = t[2];
  unsigned x;
  if (a > b) { x = a; a = b; b = x; }
  if (b > c) { x = b; b = c; c = x; }
  if (a > b) { x = a; a = b; b = x; }
}
__global__ void k_face_key(const unsigned* __restrict__ tri, const unsigned* __restrict__ order, unsigned nF, int which, unsigned* __restrict__ key) {
  const size_t i = tid();
  if (i >= nF) return;
  unsigned s[3];
  sorted3(tri + 3 * (size_t)order[i], s[0], s[1], s[2]);
  key[i] = s[which];
}
__global__ void k_dup_keep(const unsigned* __restrict__ tri, const unsigned* __restrict__ order, unsigned nF, unsigned* __restrict__ keep) {
  const size_t i = tid();
  if (i >= nF) return;
  const unsigned f = order[i];
  bool first = true;
  if (i > 0) {
    unsigned a, b, c, p, q, r;
    sorted3(tri + 3 * (size_t)f, a, b, c); sorted3(tri + 3 * (size_t)order[i - 1], p, q, r);
    first = !(a == p && b == q && c == r);
  }
  keep[f] = first ? 1u : 0u;                 // the sort is stable: the first of a run is the lowest face index
}

// ------------------------------------------------------------------------------------------ step 3: isolated pieces
__global__ void k_piece_union(const unsigned* __restrict__ tri, unsigned nF, unsigned* par) {
  const size_t f = tid();
  if (f >= nF) return;
  uf_union(par, tri[3 * f], tri[3 * f + 1]);
  uf_union(par, tri[3 * f], tri[3 * f + 2]);
}
__global__ void k_piece_faces(const unsigned* __restrict__ tri, unsigned nF, const unsigned* __restrict__ root, unsigned* __restrict__ fcount) {
  const size_t f = tid();
  if (f < nF) atomicAdd(&fcount[root[tri[3 * f]]], 1u);
}
__device__ __forceinline__ bool piece_kept(unsigned vc, unsigned fc, unsigned min_v, unsigned min_f) { return vc >= min_v && fc >= min_f; }
// stats[0] = pieces with a face, stats[1] = removed pieces, stats[2] = faces in removed pieces
__global__ void k_piece_stats(const unsigned* __restrict__ root, const unsigned* __restrict__ vcount, const unsigned* __restrict__ fcount,
                              unsigned n, unsigned min_v, unsigned min_f, unsigned* stats) {
  const size_t v = tid();
  if (v >= n || root[v] != v || fcount[v] == 0) return;
  atomicAdd(&stats[0], 1u);
  if (!piece_kept(vcount[v], fcount[v], min_v, min_f)) { atomicAdd(&stats[1], 1u); atomicAdd(&stats[2], fcount[v]); }
}
__global__ void k_piece_keep(const unsigned* __restrict__ tri, unsigned nF, const unsigned* __restrict__ root, const unsigned* __restrict__ vcount,
                             const unsigned* __restrict__ fcount, unsigned min_v, unsigned min_f, unsigned* __restrict__ keep) {
  const size_t f = tid();
  if (f >= nF) return;
  const unsigned r = root[tri[3 * f]];
  keep[f] = piece_kept(vcount[r], fcount[r], min_v, min_f) ? 1u : 0u;
}
__global__ void k_mark_used(const unsigned* __restrict__ tri, unsigned nC, unsigned* __restrict__ used) {
  const size_t c = tid();
  if (c < nC) used[tri[c]] = 1u;
}
__global__ void k_first_corner(const unsigned* __restrict__ tri, unsigned nC, unsigned* __restrict__ first) {
  const size_t c = tid();
  if (c < nC) atomicMin(&first[tri[c]], (unsigned)c);
}
__global__ void k_first_flags(const unsigned* __restrict__ tri, unsigned nC, const unsigned* __restrict__ first, unsigned* __restrict__ flag) {
  const size_t c = tid();
  if (c < nC) flag[c] = first[tri[c]] == (unsigned)c ? 1u : 0u;
}
__global__ void k_renumber(const unsigned* __restrict__ tri, unsigned nC, const unsigned* __restrict__ first, const unsigned* __restrict__ flag,
                           const unsigned* __restrict__ pos, const float* __restrict__ xyz, const unsigned char* __restrict__ rgb,
                           unsigned* __restrict__ otri, float* __restrict__ oxyz, unsigned char* __restrict__ orgb) {
  const size_t c = tid();
  if (c >= nC) return;
  const unsigned v = tri[c];
  otri[c] = pos[first[v]];
  if (flag[c]) {
    const unsigned d = pos[c];
    oxyz[3 * (size_t)d] = xyz[3 * (size_t)v]; oxyz[3 * (size_t)d + 1] = xyz[3 * (size_t)v + 1]; oxyz[3 * (size_t)d + 2] = xyz[3 * (size_t)v + 2];
    if (rgb) { orgb[3 * (size_t)d] = rgb[3 * (size_t)v]; orgb[3 * (size_t)d + 1] = rgb[3 * (size_t)v + 1]; orgb[3 * (size_t)d + 2] = rgb[3 * (size_t)v + 2]; }
  }
}

// ------------------------------------------------------------------------------------------ host driver
int read_u32(const unsigned* d, unsigned* h, size_t n, cudaStream_t st) {
  SCN_CUDA_TRY(cudaMemcpyAsync(h, d, n * 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

int upload_mesh(Mesh& m, const float* xyz, const uint8_t* rgb, uint64_t nV, const uint32_t* tri, uint64_t nF, PinnedPtr<unsigned>& h_small,
                DBuf& err, cudaEvent_t start, cudaStream_t st) {
  SCN_CUDA_TRY(create(h_small, 16));
  m.nV = (unsigned)nV; m.nF = (unsigned)nF; m.has_rgb = rgb != nullptr;
  SCN_ALLOC(m.xyz, nV * 12); SCN_ALLOC(m.tri, nF * 12); SCN_ALLOC(err, 4);
  if (m.has_rgb) SCN_ALLOC(m.rgb, nV * 3);
  SCN_CUDA_TRY(cudaEventRecord(start, st));
  if (nV) SCN_CUDA_TRY(cudaMemcpyAsync(m.xyz.p, xyz, nV * 12, cudaMemcpyHostToDevice, st));
  if (nV && rgb) SCN_CUDA_TRY(cudaMemcpyAsync(m.rgb.p, rgb, nV * 3, cudaMemcpyHostToDevice, st));
  if (nF) SCN_CUDA_TRY(cudaMemcpyAsync(m.tri.p, tri, nF * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemsetAsync(err.p, 0, 4, st));
  return SCN_OK;
}

int download_mesh(const Mesh& m, float** xyz, uint8_t** rgb, uint32_t** tri, cudaEvent_t done, cudaStream_t st, const char* who) {
  const bool want_rgb = m.has_rgb && rgb;
  MallocPtr<float> hx((float*)malloc(std::max<size_t>((size_t)m.nV * 12, 1)));
  MallocPtr<uint32_t> ht((uint32_t*)malloc(std::max<size_t>((size_t)m.nF * 12, 1)));
  MallocPtr<uint8_t> hc(want_rgb ? (uint8_t*)malloc(std::max<size_t>((size_t)m.nV * 3, 1)) : nullptr);
  if (!hx || !ht || (want_rgb && !hc)) return scn::fail(SCN_ERR_ARG, "%s: out of host memory", who);
  if ((m.nV && cudaMemcpyAsync(hx.get(), m.xyz.p, (size_t)m.nV * 12, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
      (m.nF && cudaMemcpyAsync(ht.get(), m.tri.p, (size_t)m.nF * 12, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
      (hc && m.nV && cudaMemcpyAsync(hc.get(), m.rgb.p, (size_t)m.nV * 3, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
      cudaEventRecord(done, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess)
    return scn::fail(SCN_ERR_CUDA, "%s: download failed: %s", who, cudaGetErrorString(cudaGetLastError()));
  *xyz = hx.release(); *tri = ht.release(); if (rgb) *rgb = hc.release();
  return SCN_OK;
}

int step_merge(Mesh& m, float t, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st, unsigned* d_err, unsigned* h_small) {
  const unsigned n = m.nV;
  if (n == 0) return SCN_OK;
  const float inv = 1.0f / t, tsq = t * t;
  DBuf cell, order, head, hidx, ucell, ustart, cellidx, nb, par, size, stats, target, rep_flag, newid, oxyz, orgb, otri, keep, fpos;
  if (int rc = s.ensure(n, std::max<size_t>(n, m.nF) + 1)) return rc;
  SCN_ALLOC(cell, (size_t)n * 12); SCN_ALLOC(order, (size_t)n * 4);
  unsigned* k0 = s.k0.as<unsigned>();
  unsigned* vals = s.v0.as<unsigned>();
  k_cells<<<grid_for(n), 256, 0, st>>>(m.xyz.as<float>(), n, inv, cell.as<int>(), k0, vals, d_err);
  SCN_CUDA_TRY(cudaMemcpyAsync(h_small, d_err, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  if (h_small[0] & ERR_CELL)
    return scn::fail(SCN_ERR_ARG, "scn_mesh_clean: a vertex coordinate is not finite or |v/t| >= 2^31 (merge_threshold %g)", (double)t);
  // cells in (z, y, x) order, equal cells in ascending vertex index: x, then y, then z, each sort stable
  sort_pass(s, vals, n, 32, st);
  k_gather_axis<<<grid_for(n), 256, 0, st>>>(cell.as<int>(), 1, vals, n, k0);
  sort_pass(s, vals, n, 32, st);
  k_gather_axis<<<grid_for(n), 256, 0, st>>>(cell.as<int>(), 2, vals, n, k0);
  sort_pass(s, vals, n, 32, st);
  SCN_CUDA_TRY(cudaMemcpyAsync(order.p, vals, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
  SCN_ALLOC(head, (size_t)n * 4); SCN_ALLOC(hidx, ((size_t)n + 1) * 4); SCN_ALLOC(ucell, (size_t)n * 12); SCN_ALLOC(ustart, ((size_t)n + 1) * 4);
  SCN_ALLOC(cellidx, (size_t)n * 4); SCN_ALLOC(nb, (size_t)n * 27 * 4);
  k_cell_heads<<<grid_for(n), 256, 0, st>>>(cell.as<int>(), order.as<unsigned>(), n, head.as<unsigned>());
  scn::exclusive_scan_u32(head.as<unsigned>(), hidx.as<unsigned>(), n, s.scr.as<unsigned>(), st);
  k_cell_table<<<grid_for(n), 256, 0, st>>>(cell.as<int>(), order.as<unsigned>(), head.as<unsigned>(), hidx.as<unsigned>(), n,
                                            ucell.as<int>(), ustart.as<unsigned>(), cellidx.as<unsigned>());
  k_cell_neighbours<<<grid_for(n), 256, 0, st>>>(ucell.as<int>(), hidx.as<unsigned>() + n, nb.as<int>());
  // proximity components
  SCN_ALLOC(par, (size_t)n * 4); SCN_ALLOC(size, (size_t)n * 4); SCN_ALLOC(stats, 8);
  k_iota<<<grid_for(n), 256, 0, st>>>(par.as<unsigned>(), n);
  k_merge_union<<<grid_for(n), 256, 0, st>>>(m.xyz.as<float>(), cellidx.as<unsigned>(), nb.as<int>(), ustart.as<unsigned>(), order.as<unsigned>(),
                                             n, tsq, par.as<unsigned>());
  k_uf_roots<<<grid_for(n), 256, 0, st>>>(par.as<unsigned>(), n, k0);
  SCN_CUDA_TRY(cudaMemsetAsync(size.p, 0, (size_t)n * 4, st)); SCN_CUDA_TRY(cudaMemsetAsync(stats.p, 0, 8, st));
  k_count_roots<<<grid_for(n), 256, 0, st>>>(k0, n, size.as<unsigned>());
  k_component_stats<<<grid_for(n), 256, 0, st>>>(k0, size.as<unsigned>(), n, stats.as<unsigned>());
  // members of every component in index order: stable sort of (root, vertex)
  k_iota<<<grid_for(n), 256, 0, st>>>(s.v0.as<unsigned>(), n);
  vals = s.v0.as<unsigned>();
  unsigned* skeys = sort_pass(s, vals, n, bits_for(n - 1), st) == s.v0.as<unsigned>() ? s.k0.as<unsigned>() : s.k1.as<unsigned>();
  SCN_ALLOC(target, (size_t)n * 4); SCN_ALLOC(rep_flag, (size_t)n * 4); SCN_ALLOC(newid, ((size_t)n + 1) * 4);
  k_merge_replay<<<grid_for(n), 256, 0, st>>>(skeys, vals, n, m.xyz.as<float>(), cellidx.as<unsigned>(), nb.as<int>(), ustart.as<unsigned>(),
                                              order.as<unsigned>(), tsq, rep_flag.as<unsigned>(), target.as<unsigned>());
  scn::exclusive_scan_u32(rep_flag.as<unsigned>(), newid.as<unsigned>(), n, s.scr.as<unsigned>(), st);
  if (int rc = read_u32(newid.as<unsigned>() + n, h_small, 1, st)) return rc;
  const unsigned nV2 = h_small[0];
  if (int rc = read_u32(stats.as<unsigned>(), h_small, 2, st)) return rc;
  rep.largest_merge_component = h_small[0]; rep.merge_components = h_small[1];
  rep.vertices_merged = n - nV2;
  SCN_ALLOC(oxyz, (size_t)nV2 * 12);
  if (m.has_rgb) SCN_ALLOC(orgb, (size_t)nV2 * 3);
  k_merge_vertices<<<grid_for(n), 256, 0, st>>>(m.xyz.as<float>(), m.rgb.as<unsigned char>(), rep_flag.as<unsigned>(), newid.as<unsigned>(), n,
                                                oxyz.as<float>(), orgb.as<unsigned char>());
  unsigned nF2 = 0;
  if (m.nF) {
    SCN_ALLOC(otri, (size_t)m.nF * 12); SCN_ALLOC(keep, (size_t)m.nF * 4); SCN_ALLOC(fpos, ((size_t)m.nF + 1) * 4);
    k_merge_faces<<<grid_for(m.nF), 256, 0, st>>>(m.tri.as<unsigned>(), m.nF, target.as<unsigned>(), newid.as<unsigned>(), otri.as<unsigned>(), keep.as<unsigned>());
    scn::exclusive_scan_u32(keep.as<unsigned>(), fpos.as<unsigned>(), m.nF, s.scr.as<unsigned>(), st);
    if (int rc = read_u32(fpos.as<unsigned>() + m.nF, &nF2, 1, st)) return rc;
    k_compact_faces<<<grid_for(m.nF), 256, 0, st>>>(otri.as<unsigned>(), keep.as<unsigned>(), fpos.as<unsigned>(), m.nF, m.tri.as<unsigned>());
  }
  rep.degenerate_faces = m.nF - nF2;
  m.xyz.swap(oxyz); if (m.has_rgb) m.rgb.swap(orgb);
  m.nV = nV2; m.nF = nF2;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));           // the scope's buffers are freed on return
  return SCN_OK;
}

int step_dedup(Mesh& m, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st) {
  const unsigned nF = m.nF;
  if (nF == 0) return SCN_OK;
  if (int rc = s.ensure(nF, (size_t)nF + 1)) return rc;
  DBuf keep, fpos, otri;
  SCN_ALLOC(keep, (size_t)nF * 4); SCN_ALLOC(fpos, ((size_t)nF + 1) * 4); SCN_ALLOC(otri, (size_t)nF * 12);
  const int bits = bits_for(m.nV ? m.nV - 1 : 0);
  unsigned* k0 = s.k0.as<unsigned>();
  unsigned* vals = s.v0.as<unsigned>();
  k_iota<<<grid_for(nF), 256, 0, st>>>(vals, nF);
  for (int which = 2; which >= 0; --which) {                  // LSD: largest index first, smallest last
    k_face_key<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), vals, nF, which, k0);
    sort_pass(s, vals, nF, bits, st);
  }
  k_dup_keep<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), vals, nF, keep.as<unsigned>());
  scn::exclusive_scan_u32(keep.as<unsigned>(), fpos.as<unsigned>(), nF, s.scr.as<unsigned>(), st);
  unsigned nF2 = 0;
  if (int rc = read_u32(fpos.as<unsigned>() + nF, &nF2, 1, st)) return rc;
  k_compact_faces<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), keep.as<unsigned>(), fpos.as<unsigned>(), nF, otri.as<unsigned>());
  m.tri.swap(otri);
  rep.duplicate_faces = nF - nF2;
  m.nF = nF2;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

int step_pieces(Mesh& m, unsigned min_v, unsigned min_f, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st, unsigned* h_small) {
  const unsigned n = m.nV, nF = m.nF;
  if (int rc = s.ensure(std::max(n, nF), 3 * (size_t)nF + 1)) return rc;
  DBuf par, root, vcount, fcount, stats, keep, fpos, ktri, first, flag, cpos, otri, oxyz, orgb;
  SCN_ALLOC(par, (size_t)n * 4); SCN_ALLOC(root, (size_t)n * 4); SCN_ALLOC(vcount, (size_t)n * 4); SCN_ALLOC(fcount, (size_t)n * 4); SCN_ALLOC(stats, 12);
  SCN_CUDA_TRY(cudaMemsetAsync(stats.p, 0, 12, st));
  unsigned nF2 = 0, nV2 = 0;
  if (n) {
    k_iota<<<grid_for(n), 256, 0, st>>>(par.as<unsigned>(), n);
    if (nF) k_piece_union<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), nF, par.as<unsigned>());
    k_uf_roots<<<grid_for(n), 256, 0, st>>>(par.as<unsigned>(), n, root.as<unsigned>());
    SCN_CUDA_TRY(cudaMemsetAsync(vcount.p, 0, (size_t)n * 4, st)); SCN_CUDA_TRY(cudaMemsetAsync(fcount.p, 0, (size_t)n * 4, st));
    k_count_roots<<<grid_for(n), 256, 0, st>>>(root.as<unsigned>(), n, vcount.as<unsigned>());
    if (nF) k_piece_faces<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), nF, root.as<unsigned>(), fcount.as<unsigned>());
    k_piece_stats<<<grid_for(n), 256, 0, st>>>(root.as<unsigned>(), vcount.as<unsigned>(), fcount.as<unsigned>(), n, min_v, min_f, stats.as<unsigned>());
  }
  if (nF) {
    SCN_ALLOC(keep, (size_t)nF * 4); SCN_ALLOC(fpos, ((size_t)nF + 1) * 4); SCN_ALLOC(ktri, (size_t)nF * 12);
    k_piece_keep<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), nF, root.as<unsigned>(), vcount.as<unsigned>(), fcount.as<unsigned>(), min_v, min_f,
                                               keep.as<unsigned>());
    scn::exclusive_scan_u32(keep.as<unsigned>(), fpos.as<unsigned>(), nF, s.scr.as<unsigned>(), st);
    if (int rc = read_u32(fpos.as<unsigned>() + nF, &nF2, 1, st)) return rc;
    k_compact_faces<<<grid_for(nF), 256, 0, st>>>(m.tri.as<unsigned>(), keep.as<unsigned>(), fpos.as<unsigned>(), nF, ktri.as<unsigned>());
  }
  if (int rc = read_u32(stats.as<unsigned>(), h_small, 3, st)) return rc;
  rep.pieces_total = h_small[0]; rep.pieces_removed = h_small[1]; rep.faces_in_removed_pieces = h_small[2];
  // removeIsolatedVertices: vertices numbered by their first corner in the surviving faces
  const unsigned nC = 3 * nF2;
  SCN_ALLOC(otri, (size_t)nC * 4);
  if (nC) {
    SCN_ALLOC(first, (size_t)n * 4); SCN_ALLOC(flag, (size_t)nC * 4); SCN_ALLOC(cpos, ((size_t)nC + 1) * 4);
    SCN_CUDA_TRY(cudaMemsetAsync(first.p, 0xFF, (size_t)n * 4, st));
    k_first_corner<<<grid_for(nC), 256, 0, st>>>(ktri.as<unsigned>(), nC, first.as<unsigned>());
    k_first_flags<<<grid_for(nC), 256, 0, st>>>(ktri.as<unsigned>(), nC, first.as<unsigned>(), flag.as<unsigned>());
    scn::exclusive_scan_u32(flag.as<unsigned>(), cpos.as<unsigned>(), nC, s.scr.as<unsigned>(), st);
    if (int rc = read_u32(cpos.as<unsigned>() + nC, &nV2, 1, st)) return rc;
  }
  SCN_ALLOC(oxyz, (size_t)nV2 * 12);
  if (m.has_rgb) SCN_ALLOC(orgb, (size_t)nV2 * 3);
  if (nC)
    k_renumber<<<grid_for(nC), 256, 0, st>>>(ktri.as<unsigned>(), nC, first.as<unsigned>(), flag.as<unsigned>(), cpos.as<unsigned>(), m.xyz.as<float>(),
                                            m.rgb.as<unsigned char>(), otri.as<unsigned>(), oxyz.as<float>(), orgb.as<unsigned char>());
  m.xyz.swap(oxyz); if (m.has_rgb) m.rgb.swap(orgb); m.tri.swap(otri);
  m.nV = nV2; m.nF = nF2;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

int drop_unreferenced(Mesh& m, Scratch& s, cudaStream_t st, unsigned* h_small) {
  const unsigned n = m.nV, nC = 3 * m.nF;
  if (int rc = s.ensure(1, (size_t)n + 1)) return rc;
  DBuf used, newid, ident, keep, otri, oxyz, orgb;
  SCN_ALLOC(used, (size_t)n * 4); SCN_ALLOC(newid, ((size_t)n + 1) * 4); SCN_ALLOC(ident, (size_t)n * 4); SCN_ALLOC(keep, (size_t)m.nF * 4);
  SCN_ALLOC(otri, (size_t)nC * 4);
  unsigned nV2 = 0;
  if (n) {
    SCN_CUDA_TRY(cudaMemsetAsync(used.p, 0, (size_t)n * 4, st));
    if (nC) k_mark_used<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), nC, used.as<unsigned>());
    k_iota<<<grid_for(n), 256, 0, st>>>(ident.as<unsigned>(), n);
    scn::exclusive_scan_u32(used.as<unsigned>(), newid.as<unsigned>(), n, s.scr.as<unsigned>(), st);
    if (int rc = read_u32(newid.as<unsigned>() + n, h_small, 1, st)) return rc;
    nV2 = h_small[0];
  }
  SCN_ALLOC(oxyz, (size_t)nV2 * 12);
  if (m.has_rgb) SCN_ALLOC(orgb, (size_t)nV2 * 3);
  if (n) k_merge_vertices<<<grid_for(n), 256, 0, st>>>(m.xyz.as<float>(), m.rgb.as<unsigned char>(), used.as<unsigned>(), newid.as<unsigned>(), n,
                                                       oxyz.as<float>(), orgb.as<unsigned char>());
  if (m.nF) k_merge_faces<<<grid_for(m.nF), 256, 0, st>>>(m.tri.as<unsigned>(), m.nF, ident.as<unsigned>(), newid.as<unsigned>(), otri.as<unsigned>(),
                                                          keep.as<unsigned>());
  m.xyz.swap(oxyz); if (m.has_rgb) m.rgb.swap(orgb); m.tri.swap(otri);
  m.nV = nV2;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  return SCN_OK;
}

int run_clean_steps(Mesh& m, const scn_mesh_clean_params& params, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st,
                    unsigned* d_err, unsigned* h_small, const EventPtr* ev) {
  int rc = SCN_OK;
  if (!(params.flags & SCN_CLEAN_SKIP_MERGE)) rc = step_merge(m, params.merge_threshold, s, rep, st, d_err, h_small);
  if (rc) return rc;
  SCN_CUDA_TRY(cudaEventRecord(ev[1].get(), st));
  if (!(params.flags & SCN_CLEAN_SKIP_DEDUP)) rc = step_dedup(m, s, rep, st);
  if (rc) return rc;
  SCN_CUDA_TRY(cudaEventRecord(ev[2].get(), st));
  if (!(params.flags & SCN_CLEAN_SKIP_PIECES)) rc = step_pieces(m, params.min_piece_vertices, params.min_piece_faces, s, rep, st, h_small);
  if (rc) return rc;
  SCN_CUDA_TRY(cudaEventRecord(ev[3].get(), st));
  SCN_CUDA_TRY(cudaEventSynchronize(ev[3].get()));
  rep.merge_ms = ms_between(ev[0], ev[1]); rep.dedup_ms = ms_between(ev[1], ev[2]); rep.pieces_ms = ms_between(ev[2], ev[3]);
  return SCN_OK;
}

}  // namespace scn::mc

using namespace scn;
using namespace scn::mc;

extern "C" {

void scn_mesh_clean_default_params(scn_mesh_clean_params* p) {
  if (!p) return;
  p->merge_threshold = 0.0010689f;                 // Server/tools/meshclean/clean.mlx
  p->min_piece_vertices = 0;
  p->min_piece_faces = 7500;
  p->flags = 0;
}

size_t scn_mesh_clean_report_sizeof(void) { return sizeof(scn_mesh_clean_report_t); }

int scn_mesh_clean(const float* xyz, const uint8_t* rgb, uint64_t nV, const uint32_t* tri, uint64_t nF, const scn_mesh_clean_params* params,
                   float** xyz_out, uint8_t** rgb_out, uint32_t** tri_out, uint64_t* nV_out, uint64_t* nF_out, scn_mesh_clean_report_t* report) {
  if (!params || !xyz_out || !tri_out || !nV_out || !nF_out || (nV && !xyz) || (nF && !tri))
    return scn::fail(SCN_ERR_ARG, "scn_mesh_clean: null argument");
  *xyz_out = nullptr; *tri_out = nullptr; if (rgb_out) *rgb_out = nullptr; *nV_out = 0; *nF_out = 0;
  if (nV > 0x7FFFFFFFull || nF > 0x55555555ull) return scn::fail(SCN_ERR_ARG, "scn_mesh_clean: mesh too large (%llu vertices, %llu faces)",
                                                                (unsigned long long)nV, (unsigned long long)nF);
  const bool merge = !(params->flags & SCN_CLEAN_SKIP_MERGE);
  const float t = params->merge_threshold;
  if (merge && !(t > 0.f)) return scn::fail(SCN_ERR_ARG, "scn_mesh_clean: invalid merge threshold %g", (double)t);   // meshData.cpp:219
  scn_mesh_clean_report_t rep;
  memset(&rep, 0, sizeof(rep));
  rep.vertices_in = nV; rep.faces_in = nF;
  const auto t0 = std::chrono::steady_clock::now();
  StreamPtr S; EventPtr ev[6];
  SCN_CUDA_TRY(create(S, ev, 6));
  const cudaStream_t st = S.get();
  Mesh m; Scratch s; DBuf err; PinnedPtr<unsigned> h_small;
  if (int rc = upload_mesh(m, xyz, rgb, nV, tri, nF, h_small, err, ev[0].get(), st)) return rc;
  if (nF) k_check_faces<<<grid_for(3 * nF), 256, 0, st>>>(m.tri.as<unsigned>(), 3 * nF, (unsigned)nV, err.as<unsigned>());
  SCN_CUDA_TRY(cudaEventRecord(ev[1].get(), st));
  if (int rc = read_u32(err.as<unsigned>(), h_small.get(), 1, st)) return rc;
  if (h_small[0] & ERR_INDEX) return scn::fail(SCN_ERR_ARG, "scn_mesh_clean: a face references a vertex >= %llu", (unsigned long long)nV);
  if (int rc = run_clean_steps(m, *params, s, rep, st, err.as<unsigned>(), h_small.get(), ev + 1)) return rc;
  if (int rc = download_mesh(m, xyz_out, rgb_out, tri_out, ev[5].get(), st, "scn_mesh_clean")) return rc;
  rep.vertices_out = m.nV; rep.faces_out = m.nF;
  rep.upload_ms = ms_between(ev[0], ev[1]); rep.download_ms = ms_between(ev[4], ev[5]);
  rep.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *nV_out = m.nV; *nF_out = m.nF;
  if (report) *report = rep;
  return SCN_OK;
}

}  // extern "C"
