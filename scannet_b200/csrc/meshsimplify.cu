// Quadric edge-collapse decimation on the GPU (DESIGN.md §6g): MeshLab's simplify.mlx step of the ScanNet `decimate` stage
// (`_vh_clean.ply` -> `_vh_clean_1.ply` -> `_vh_clean_2.ply`, Server/scan_processor.py:144-145), stated as this repository's
// own spec.  MeshLab/VCG is not in the reference tree, and its sequential priority-queue decimation could not be reproduced in
// parallel anyway: the output is NOT MeshLab's mesh.  The spec collapses edges in deterministic rounds of independent
// collapses with Garland-Heckbert quadrics in binary64:
//
//   quadrics   Q_v = sum of the area-weighted face quadrics K_f over v's corners, faces ascending (one thread per vertex over
//              its corner ring; the ring is a stable radix sort of the corners by vertex)
//   round      edges = distinct corner pairs of the alive faces (two stable radix sorts of the corner pairs); per edge the
//              placement, the quadric error at the rounded placement and the quality penalty; edges ranked by (cost, a, b)
//              (two stable radix sorts of the cost bits: cost > 0, so the bits are monotone); m(x) = smallest rank at x and
//              M(x) = min of m over x and its neighbours by atomicMin; e = (a, b) is selected iff M(a) = M(b) = rank(e).
//              Selected edges are two apart in the edge graph, so their collapses commute; they are applied in rank order
//              while the face count is above the target (an exclusive scan of the faces each one removes).
//   AutoClean  duplicate faces and unreferenced vertices, with meshclean.cu's own steps; then the script's clean filters.
//
// The mesh is uploaded once; every round runs in HBM and reads back two counts.  Nothing depends on scheduling: the sorts are
// stable, the minima are atomicMin of integers and every compaction is a scan.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>

#include "meshclean_steps.h"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "scn_common.h"

namespace {

using namespace scn;
using namespace scn::mc;

__device__ __forceinline__ size_t tid() { return blockIdx.x * (size_t)blockDim.x + threadIdx.x; }

// ------------------------------------------------------------------------------------------ §6g arithmetic (binary64, no FMA)
constexpr double kQualityScale = 2.0 * 1.7320508075688772;     // 2*sqrt(3): q = 4*sqrt(3)*area / sum l^2 = 2*sqrt(3)*|n| / sum l^2

__device__ void face_quadric(const float* p0, const float* p1, const float* p2, double* K) {
  const double x0 = p0[0], y0 = p0[1], z0 = p0[2];
  const double ux = (double)p1[0] - x0, uy = (double)p1[1] - y0, uz = (double)p1[2] - z0;
  const double vx = (double)p2[0] - x0, vy = (double)p2[1] - y0, vz = (double)p2[2] - z0;
  const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
  const double len = sqrt((nx * nx + ny * ny) + nz * nz);
  if (len == 0.0) { for (int i = 0; i < 10; ++i) K[i] = 0.0; return; }
  const double d = -((nx * x0 + ny * y0) + nz * z0);
  const double v[4] = {nx, ny, nz, d};
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j) K[k++] = (v[i] * v[j]) / len;
}

__device__ double quality(const float* p0, const float* p1, const float* p2) {
  const double ux = (double)p1[0] - p0[0], uy = (double)p1[1] - p0[1], uz = (double)p1[2] - p0[2];
  const double vx = (double)p2[0] - p0[0], vy = (double)p2[1] - p0[1], vz = (double)p2[2] - p0[2];
  const double wx = (double)p2[0] - p1[0], wy = (double)p2[1] - p1[1], wz = (double)p2[2] - p1[2];
  const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
  const double len = sqrt((nx * nx + ny * ny) + nz * nz);
  const double s = (((ux * ux + uy * uy) + uz * uz) + ((wx * wx + wy * wy) + wz * wz)) + ((vx * vx + vy * vy) + vz * vz);
  return s > 0.0 ? (kQualityScale * len) / s : 0.0;
}

__device__ double qerr(const double* q, const float* p) {
  const double x = p[0], y = p[1], z = p[2];
  return ((((((((q[0] * x * x + 2.0 * q[1] * x * y) + 2.0 * q[2] * x * z) + 2.0 * q[3] * x) + q[4] * y * y) + 2.0 * q[5] * y * z) +
            2.0 * q[6] * y) + q[7] * z * z) + 2.0 * q[8] * z) + q[9];
}

// placement of an edge whose summed quadric is q; returns the error at the (rounded) placement
__device__ double place(const double* q, const float* pa, const float* pb, float* out) {
  const double c00 = q[4] * q[7] - q[5] * q[5], c01 = q[2] * q[5] - q[1] * q[7], c02 = q[1] * q[5] - q[2] * q[4];
  const double c11 = q[0] * q[7] - q[2] * q[2], c12 = q[1] * q[2] - q[0] * q[5], c22 = q[0] * q[4] - q[1] * q[1];
  const double det = (q[0] * c00 + q[1] * c01) + q[2] * c02;
  if (det > 1e-9 * q[0] * q[4] * q[7]) {                       // Hadamard: det <= q00*q11*q22, so a scale-free conditioning test
    const double b0 = -q[3], b1 = -q[6], b2 = -q[8];
    const float x[3] = {(float)(((c00 * b0 + c01 * b1) + c02 * b2) / det), (float)(((c01 * b0 + c11 * b1) + c12 * b2) / det),
                        (float)(((c02 * b0 + c12 * b1) + c22 * b2) / det)};
    if (isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2])) { out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; return qerr(q, out); }
  }
  const float mid[3] = {(float)(0.5 * ((double)pa[0] + (double)pb[0])), (float)(0.5 * ((double)pa[1] + (double)pb[1])),
                        (float)(0.5 * ((double)pa[2] + (double)pb[2]))};
  const float* cand[3] = {pa, pb, mid};
  double best = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double e = qerr(q, cand[i]);
    if (i == 0 || e < best) { best = e; out[0] = cand[i][0]; out[1] = cand[i][1]; out[2] = cand[i][2]; }
  }
  return best;
}

__device__ __forceinline__ bool has(const unsigned* t, unsigned v) { return t[0] == v || t[1] == v || t[2] == v; }

// ------------------------------------------------------------------------------------------ kernels
enum : unsigned { ERR_INDEX = 1u, ERR_COORD = 2u };

__global__ void k_check(const float* __restrict__ xyz, size_t n3, const unsigned* __restrict__ tri, size_t nC, unsigned nV, unsigned* err) {
  const size_t i = tid();
  if (i < nC && tri[i] >= nV) atomicOr(err, ERR_INDEX);
  if (i < n3 && !isfinite(xyz[i])) atomicOr(err, ERR_COORD);
}

// corner ring: k0 = vertex of corner c, v0 = c (then a stable sort by vertex)
__global__ void k_corner_keys(const unsigned* __restrict__ tri, size_t nC, unsigned* __restrict__ key, unsigned* __restrict__ val) {
  const size_t c = tid();
  if (c < nC) { key[c] = tri[c]; val[c] = (unsigned)c; }
}
// rs/re (zeroed): the sorted positions of each vertex's corners
__global__ void k_ring_bounds(const unsigned* __restrict__ skey, size_t nC, unsigned* __restrict__ rs, unsigned* __restrict__ re) {
  const size_t i = tid();
  if (i >= nC) return;
  const unsigned v = skey[i];
  if (i == 0 || skey[i - 1] != v) rs[v] = (unsigned)i;
  if (i + 1 == nC || skey[i + 1] != v) re[v] = (unsigned)i + 1u;
}
__global__ void k_ring_max(const unsigned* __restrict__ rs, const unsigned* __restrict__ re, unsigned n, unsigned* big) {
  const size_t v = tid();
  if (v < n && re[v] > rs[v]) atomicMax(big, re[v] - rs[v]);
}

// Q_v: K_f of every corner at v, corners ascending (faces ascending)
__global__ void k_vertex_quadrics(const unsigned* __restrict__ rs, const unsigned* __restrict__ re, const unsigned* __restrict__ ring,
                                  const unsigned* __restrict__ tri, const float* __restrict__ xyz, unsigned n, double* __restrict__ Q) {
  const size_t v = tid();
  if (v >= n) return;
  double q[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (unsigned i = rs[v]; i < re[v]; ++i) {
    const unsigned* t = tri + 3 * (size_t)(ring[i] / 3);
    double K[10];
    face_quadric(xyz + 3 * (size_t)t[0], xyz + 3 * (size_t)t[1], xyz + 3 * (size_t)t[2], K);
#pragma unroll
    for (int j = 0; j < 10; ++j) q[j] = q[j] + K[j];
  }
#pragma unroll
  for (int j = 0; j < 10; ++j) Q[10 * v + j] = q[j];
}

// edge of corner c: (tri[c], next corner of its face), normalised to a < b; a == b gives the sentinel (sorts last)
__device__ __forceinline__ void corner_edge(const unsigned* tri, unsigned c, unsigned sentinel, unsigned& a, unsigned& b) {
  const unsigned f = c / 3, k = c - 3 * f;
  const unsigned u = tri[c], v = tri[3 * f + (k == 2 ? 0 : k + 1)];
  if (u == v) { a = b = sentinel; return; }
  a = min(u, v); b = max(u, v);
}
__global__ void k_edge_key_b(const unsigned* __restrict__ tri, size_t nC, unsigned sentinel, unsigned* __restrict__ key, unsigned* __restrict__ val) {
  const size_t c = tid();
  if (c >= nC) return;
  unsigned a, b;
  corner_edge(tri, (unsigned)c, sentinel, a, b);
  key[c] = b; val[c] = (unsigned)c;
}
__global__ void k_edge_key_a(const unsigned* __restrict__ tri, const unsigned* __restrict__ order, size_t nC, unsigned sentinel, unsigned* __restrict__ key) {
  const size_t i = tid();
  if (i >= nC) return;
  unsigned a, b;
  corner_edge(tri, order[i], sentinel, a, b);
  key[i] = a;
}
__global__ void k_edge_heads(const unsigned* __restrict__ tri, const unsigned* __restrict__ order, size_t nC, unsigned sentinel, unsigned* __restrict__ head) {
  const size_t i = tid();
  if (i >= nC) return;
  unsigned a, b, pa, pb;
  corner_edge(tri, order[i], sentinel, a, b);
  bool h = a != sentinel;
  if (h && i > 0) { corner_edge(tri, order[i - 1], sentinel, pa, pb); h = !(pa == a && pb == b); }
  head[i] = h ? 1u : 0u;
}
__global__ void k_edge_write(const unsigned* __restrict__ tri, const unsigned* __restrict__ order, const unsigned* __restrict__ head,
                             const unsigned* __restrict__ hidx, size_t nC, unsigned* __restrict__ ea, unsigned* __restrict__ eb) {
  const size_t i = tid();
  if (i >= nC || !head[i]) return;
  unsigned a, b;
  corner_edge(tri, order[i], 0xFFFFFFFFu, a, b);
  ea[hidx[i]] = a; eb[hidx[i]] = b;
}

// per edge: placement, f(e) and cost = max(err, 1e-15) * penalty
__global__ void k_edge_cost(const unsigned* __restrict__ ea, const unsigned* __restrict__ eb, unsigned nE, const float* __restrict__ xyz,
                            const double* __restrict__ Q, const unsigned* __restrict__ tri, const unsigned* __restrict__ ring,
                            const unsigned* __restrict__ rs, const unsigned* __restrict__ re, double thr, float* __restrict__ pstar,
                            unsigned* __restrict__ fcount, double* __restrict__ cost) {
  const size_t e = tid();
  if (e >= nE) return;
  const unsigned a = ea[e], b = eb[e];
  double q[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) q[j] = Q[10 * (size_t)a + j] + Q[10 * (size_t)b + j];
  float p[3];
  const double err = place(q, xyz + 3 * (size_t)a, xyz + 3 * (size_t)b, p);
  double qmin = 1.0;
  unsigned f = 0;
  for (int k = 0; k < 2; ++k) {
    const unsigned v = k ? b : a;
    for (unsigned i = rs[v]; i < re[v]; ++i) {
      const unsigned face = ring[i] / 3;
      const unsigned* t = tri + 3 * (size_t)face;
      if (has(t, a) && has(t, b)) {
        if (k == 0 && (i == rs[v] || ring[i - 1] / 3 != face)) ++f;
        continue;
      }
      const float* c[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) c[j] = (t[j] == a || t[j] == b) ? p : xyz + 3 * (size_t)t[j];
      const double qq = quality(c[0], c[1], c[2]);
      if (qq < qmin) qmin = qq;
    }
  }
  const double pen = qmin < thr ? thr / (qmin > 1e-6 ? qmin : 1e-6) : 1.0;
  cost[e] = (err > 1e-15 ? err : 1e-15) * pen;
  pstar[3 * e] = p[0]; pstar[3 * e + 1] = p[1]; pstar[3 * e + 2] = p[2];
  fcount[e] = f;
}

// key[i] = low (hi = 0) or high (hi = 1) 32 bits of cost[order[i]]: cost > 0, so its bits order like the value
__global__ void k_cost_key(const double* __restrict__ cost, const unsigned* __restrict__ order, unsigned n, int hi, unsigned* __restrict__ key) {
  const size_t i = tid();
  if (i >= n) return;
  const unsigned long long b = (unsigned long long)__double_as_longlong(cost[order[i]]);
  key[i] = hi ? (unsigned)(b >> 32) : (unsigned)b;
}
__global__ void k_rank(const unsigned* __restrict__ order, unsigned n, unsigned* __restrict__ rank) {
  const size_t i = tid();
  if (i < n) rank[order[i]] = (unsigned)i;
}
__global__ void k_min_rank(const unsigned* __restrict__ ea, const unsigned* __restrict__ eb, const unsigned* __restrict__ rank, unsigned n, unsigned* m) {
  const size_t e = tid();
  if (e < n) { atomicMin(&m[ea[e]], rank[e]); atomicMin(&m[eb[e]], rank[e]); }
}
__global__ void k_min_neighbour(const unsigned* __restrict__ ea, const unsigned* __restrict__ eb, const unsigned* __restrict__ m, unsigned n, unsigned* M) {
  const size_t e = tid();
  if (e < n) { const unsigned a = ea[e], b = eb[e]; atomicMin(&M[a], m[b]); atomicMin(&M[b], m[a]); }
}
// in rank order: the faces the i-th edge removes if it is selected, else 0
__global__ void k_select(const unsigned* __restrict__ order, const unsigned* __restrict__ ea, const unsigned* __restrict__ eb,
                         const unsigned* __restrict__ fcount, const unsigned* __restrict__ M, unsigned n, unsigned* __restrict__ sf) {
  const size_t i = tid();
  if (i >= n) return;
  const unsigned e = order[i];
  sf[i] = (M[ea[e]] == (unsigned)i && M[eb[e]] == (unsigned)i) ? fcount[e] : 0u;
}
// the selected prefix that is still needed: alive - (faces removed by earlier selected edges) > target
__global__ void k_apply(const unsigned* __restrict__ order, const unsigned* __restrict__ ea, const unsigned* __restrict__ eb,
                        const unsigned* __restrict__ sf, const unsigned* __restrict__ pre, unsigned n, unsigned alive, unsigned long long target,
                        const float* __restrict__ pstar, float* __restrict__ xyz, double* __restrict__ Q, unsigned* __restrict__ remap,
                        unsigned long long* counters) {
  const size_t i = tid();
  if (i >= n || sf[i] == 0 || (unsigned long long)(alive - pre[i]) <= target) return;
  const unsigned e = order[i], a = ea[e], b = eb[e];
  xyz[3 * (size_t)a] = pstar[3 * (size_t)e]; xyz[3 * (size_t)a + 1] = pstar[3 * (size_t)e + 1]; xyz[3 * (size_t)a + 2] = pstar[3 * (size_t)e + 2];
#pragma unroll
  for (int j = 0; j < 10; ++j) Q[10 * (size_t)a + j] = Q[10 * (size_t)a + j] + Q[10 * (size_t)b + j];
  remap[b] = a;
  atomicAdd(&counters[0], 1ull);
  atomicAdd(&counters[1], (unsigned long long)sf[i]);
}
// faces with both ends of a collapsed edge die; in the others b becomes a (a face meets at most one collapsed edge)
__global__ void k_collapse_faces(unsigned* __restrict__ tri, unsigned nF, const unsigned* __restrict__ remap, unsigned* __restrict__ keep) {
  const size_t f = tid();
  if (f >= nF) return;
  unsigned* t = tri + 3 * f;
  unsigned k = 1u;
  for (int j = 0; j < 3; ++j) {
    const unsigned a = remap[t[j]], b = t[j];
    if (a == 0xFFFFFFFFu) continue;
    if (has(t, a)) k = 0u;
    else for (int i = 0; i < 3; ++i) if (t[i] == b) t[i] = a;      // every corner at b (a degenerate face may hold it twice)
    break;
  }
  keep[f] = k;
}

// ------------------------------------------------------------------------------------------ host driver
struct Work {                       // per-round buffers, sized once for the input
  DBuf Q, rs, re, ring, head, hidx, ea, eb, cost, pstar, fcount, rank, m, M, sf, pre, remap, keep, fpos, otri, big, counters;
};

// corner ring of the current faces (and, if `big`, the largest ring into it)
int build_ring(Mesh& m, Scratch& s, Work& w, cudaStream_t st, bool big) {
  const size_t nC = 3 * (size_t)m.nF;
  SCN_CUDA_TRY(cudaMemsetAsync(w.rs.p, 0, (size_t)m.nV * 4, st)); SCN_CUDA_TRY(cudaMemsetAsync(w.re.p, 0, (size_t)m.nV * 4, st));
  if (nC == 0) return SCN_OK;
  unsigned* vals = s.v0.as<unsigned>();
  k_corner_keys<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), nC, s.k0.as<unsigned>(), vals);
  sort_pass(s, vals, nC, bits_for(m.nV - 1), st);
  const unsigned* skeys = vals == s.v0.as<unsigned>() ? s.k0.as<unsigned>() : s.k1.as<unsigned>();
  k_ring_bounds<<<grid_for(nC), 256, 0, st>>>(skeys, nC, w.rs.as<unsigned>(), w.re.as<unsigned>());
  SCN_CUDA_TRY(cudaMemcpyAsync(w.ring.p, vals, nC * 4, cudaMemcpyDeviceToDevice, st));
  if (big) k_ring_max<<<grid_for(m.nV), 256, 0, st>>>(w.rs.as<unsigned>(), w.re.as<unsigned>(), m.nV, w.big.as<unsigned>());
  return SCN_OK;
}

// one round; *applied = false when the mesh has no edge left
int run_round(Mesh& m, Scratch& s, Work& w, double thr, unsigned long long target, cudaStream_t st, unsigned* h_small, bool* applied) {
  *applied = false;
  const size_t nC = 3 * (size_t)m.nF;
  if (int rc = build_ring(m, s, w, st, true)) return rc;
  const unsigned sentinel = m.nV;                       // bits_for(nV) bits hold it
  unsigned* vals = s.v0.as<unsigned>();
  k_edge_key_b<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), nC, sentinel, s.k0.as<unsigned>(), vals);
  sort_pass(s, vals, nC, bits_for(sentinel), st);
  k_edge_key_a<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), vals, nC, sentinel, s.k0.as<unsigned>());
  sort_pass(s, vals, nC, bits_for(sentinel), st);
  k_edge_heads<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), vals, nC, sentinel, w.head.as<unsigned>());
  scn::exclusive_scan_u32(w.head.as<unsigned>(), w.hidx.as<unsigned>(), nC, s.scr.as<unsigned>(), st);
  if (int rc = read_u32(w.hidx.as<unsigned>() + nC, h_small, 1, st)) return rc;
  const unsigned nE = h_small[0];
  if (nE == 0) return SCN_OK;
  k_edge_write<<<grid_for(nC), 256, 0, st>>>(m.tri.as<unsigned>(), vals, w.head.as<unsigned>(), w.hidx.as<unsigned>(), nC, w.ea.as<unsigned>(), w.eb.as<unsigned>());
  k_edge_cost<<<grid_for(nE), 256, 0, st>>>(w.ea.as<unsigned>(), w.eb.as<unsigned>(), nE, m.xyz.as<float>(), w.Q.as<double>(), m.tri.as<unsigned>(),
                                            w.ring.as<unsigned>(), w.rs.as<unsigned>(), w.re.as<unsigned>(), thr, w.pstar.as<float>(),
                                            w.fcount.as<unsigned>(), w.cost.as<double>());
  // rank order (cost, a, b): the edges are already in (a, b) order, and both sorts are stable
  vals = s.v0.as<unsigned>();
  k_iota<<<grid_for(nE), 256, 0, st>>>(vals, nE);
  k_cost_key<<<grid_for(nE), 256, 0, st>>>(w.cost.as<double>(), vals, nE, 0, s.k0.as<unsigned>());
  sort_pass(s, vals, nE, 32, st);
  k_cost_key<<<grid_for(nE), 256, 0, st>>>(w.cost.as<double>(), vals, nE, 1, s.k0.as<unsigned>());
  sort_pass(s, vals, nE, 32, st);
  const unsigned* order = vals;
  k_rank<<<grid_for(nE), 256, 0, st>>>(order, nE, w.rank.as<unsigned>());
  SCN_CUDA_TRY(cudaMemsetAsync(w.m.p, 0xFF, (size_t)m.nV * 4, st));
  k_min_rank<<<grid_for(nE), 256, 0, st>>>(w.ea.as<unsigned>(), w.eb.as<unsigned>(), w.rank.as<unsigned>(), nE, w.m.as<unsigned>());
  SCN_CUDA_TRY(cudaMemcpyAsync(w.M.p, w.m.p, (size_t)m.nV * 4, cudaMemcpyDeviceToDevice, st));
  k_min_neighbour<<<grid_for(nE), 256, 0, st>>>(w.ea.as<unsigned>(), w.eb.as<unsigned>(), w.m.as<unsigned>(), nE, w.M.as<unsigned>());
  k_select<<<grid_for(nE), 256, 0, st>>>(order, w.ea.as<unsigned>(), w.eb.as<unsigned>(), w.fcount.as<unsigned>(), w.M.as<unsigned>(), nE,
                                         w.sf.as<unsigned>());
  scn::exclusive_scan_u32(w.sf.as<unsigned>(), w.pre.as<unsigned>(), nE, s.scr.as<unsigned>(), st);
  SCN_CUDA_TRY(cudaMemsetAsync(w.remap.p, 0xFF, (size_t)m.nV * 4, st));
  k_apply<<<grid_for(nE), 256, 0, st>>>(order, w.ea.as<unsigned>(), w.eb.as<unsigned>(), w.sf.as<unsigned>(), w.pre.as<unsigned>(), nE, m.nF, target,
                                        w.pstar.as<float>(), m.xyz.as<float>(), w.Q.as<double>(), w.remap.as<unsigned>(),
                                        w.counters.as<unsigned long long>());
  k_collapse_faces<<<grid_for(m.nF), 256, 0, st>>>(m.tri.as<unsigned>(), m.nF, w.remap.as<unsigned>(), w.keep.as<unsigned>());
  scn::exclusive_scan_u32(w.keep.as<unsigned>(), w.fpos.as<unsigned>(), m.nF, s.scr.as<unsigned>(), st);
  k_compact_faces<<<grid_for(m.nF), 256, 0, st>>>(m.tri.as<unsigned>(), w.keep.as<unsigned>(), w.fpos.as<unsigned>(), m.nF, w.otri.as<unsigned>());
  if (int rc = read_u32(w.fpos.as<unsigned>() + m.nF, h_small, 1, st)) return rc;
  m.tri.swap(w.otri);
  m.nF = h_small[0];
  *applied = true;
  return SCN_OK;
}

}  // namespace

extern "C" {

void scn_mesh_simplify_default_params(scn_mesh_simplify_params* p, scn_mesh_clean_params* after) {
  if (p) {                                         // Server/tools/meshclean/simplify.mlx
    p->target_faces = 0;
    p->target_perc = 0.2;
    p->quality_thr = 0.3;
  }
  if (after) {
    scn_mesh_clean_default_params(after);
    after->min_piece_faces = 1000;
  }
}

size_t scn_mesh_simplify_report_sizeof(void) { return sizeof(scn_mesh_simplify_report_t); }

int scn_mesh_simplify(const float* xyz, const uint8_t* rgb, uint64_t nV, const uint32_t* tri, uint64_t nF, const scn_mesh_simplify_params* params,
                      const scn_mesh_clean_params* after, float** xyz_out, uint8_t** rgb_out, uint32_t** tri_out, uint64_t* nV_out,
                      uint64_t* nF_out, scn_mesh_simplify_report_t* report) {
  if (!params || !xyz_out || !tri_out || !nV_out || !nF_out || (nV && !xyz) || (nF && !tri))
    return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: null argument");
  *xyz_out = nullptr; *tri_out = nullptr; if (rgb_out) *rgb_out = nullptr; *nV_out = 0; *nF_out = 0;
  if (nV > 0x7FFFFFFFull || nF > 0x55555555ull) return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: mesh too large (%llu vertices, %llu faces)",
                                                                (unsigned long long)nV, (unsigned long long)nF);
  if (!(params->target_perc >= 0.0 && params->target_perc <= 1.0))
    return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: target_perc %g is not in [0, 1]", params->target_perc);
  if (!(params->quality_thr >= 0.0)) return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: quality_thr %g is NaN or negative", params->quality_thr);
  if (after && !(after->flags & SCN_CLEAN_SKIP_MERGE) && !(after->merge_threshold > 0.f))
    return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: invalid merge threshold %g", (double)after->merge_threshold);
  const unsigned long long target =
      params->target_perc != 0.0 ? (unsigned long long)std::floor((double)nF * params->target_perc) : (unsigned long long)params->target_faces;
  scn_mesh_simplify_report_t rep;
  memset(&rep, 0, sizeof(rep));
  rep.vertices_in = nV; rep.faces_in = nF; rep.target_faces = target;
  const auto t0 = std::chrono::steady_clock::now();
  StreamPtr S; EventPtr ev[11];                 // ev[7..10]: the clean filters' steps
  SCN_CUDA_TRY(create(S, ev, 11));
  const cudaStream_t st = S.get();
  Mesh m; Scratch s; Work w; DBuf err; PinnedPtr<unsigned> hp;
  const size_t nC = 3 * (size_t)nF;
  if (int rc = upload_mesh(m, xyz, rgb, nV, tri, nF, hp, err, ev[0].get(), st)) return rc;
  unsigned* h_small = hp.get();
  if (nV || nF) k_check<<<grid_for(std::max<size_t>(3 * nV, nC)), 256, 0, st>>>(m.xyz.as<float>(), 3 * nV, m.tri.as<unsigned>(), nC, (unsigned)nV,
                                                                                err.as<unsigned>());
  SCN_CUDA_TRY(cudaEventRecord(ev[1].get(), st));
  if (int rc = read_u32(err.as<unsigned>(), h_small, 1, st)) return rc;
  if (h_small[0] & ERR_INDEX) return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: a face references a vertex >= %llu", (unsigned long long)nV);
  if (h_small[0] & ERR_COORD) return scn::fail(SCN_ERR_ARG, "scn_mesh_simplify: a vertex coordinate is not finite");
  // per-round buffers, sized for the input (every round has at most nC corners and edges)
  if (int rc = s.ensure(std::max<size_t>(nC, 1), nC + 1)) return rc;
  SCN_ALLOC(w.Q, nV * 80); SCN_ALLOC(w.rs, nV * 4); SCN_ALLOC(w.re, nV * 4); SCN_ALLOC(w.ring, nC * 4); SCN_ALLOC(w.head, nC * 4);
  SCN_ALLOC(w.hidx, (nC + 1) * 4); SCN_ALLOC(w.ea, nC * 4); SCN_ALLOC(w.eb, nC * 4); SCN_ALLOC(w.cost, nC * 8); SCN_ALLOC(w.pstar, nC * 12);
  SCN_ALLOC(w.fcount, nC * 4); SCN_ALLOC(w.rank, nC * 4); SCN_ALLOC(w.m, nV * 4); SCN_ALLOC(w.M, nV * 4); SCN_ALLOC(w.sf, nC * 4);
  SCN_ALLOC(w.pre, (nC + 1) * 4); SCN_ALLOC(w.remap, nV * 4); SCN_ALLOC(w.keep, nF * 4); SCN_ALLOC(w.fpos, (nF + 1) * 4); SCN_ALLOC(w.otri, nF * 12);
  SCN_ALLOC(w.big, 4); SCN_ALLOC(w.counters, 16);
  SCN_CUDA_TRY(cudaMemsetAsync(w.big.p, 0, 4, st)); SCN_CUDA_TRY(cudaMemsetAsync(w.counters.p, 0, 16, st));
  if (int rc = build_ring(m, s, w, st, false)) return rc;
  if (nV) k_vertex_quadrics<<<grid_for(nV), 256, 0, st>>>(w.rs.as<unsigned>(), w.re.as<unsigned>(), w.ring.as<unsigned>(), m.tri.as<unsigned>(),
                                                          m.xyz.as<float>(), (unsigned)nV, w.Q.as<double>());
  SCN_CUDA_TRY(cudaEventRecord(ev[2].get(), st));
  while (m.nF > target) {
    bool applied = false;
    if (int rc = run_round(m, s, w, params->quality_thr, target, st, h_small, &applied)) return rc;
    if (!applied) break;
    ++rep.rounds;
  }
  SCN_CUDA_TRY(cudaEventRecord(ev[3].get(), st));
  {
    unsigned long long c[2];
    SCN_CUDA_TRY(cudaMemcpyAsync(c, w.counters.p, 16, cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(h_small, w.big.p, 4, cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    rep.collapses = c[0]; rep.faces_collapsed = c[1]; rep.max_vertex_faces = h_small[0];
    if (rep.faces_collapsed != nF - m.nF)
      return scn::fail(SCN_ERR_CUDA, "scn_mesh_simplify: internal error: %llu faces collapsed, %llu removed", rep.faces_collapsed,
                       (unsigned long long)(nF - m.nF));
  }
  // AutoClean: duplicate faces (mLib's rule) and unreferenced vertices, survivors in ascending order
  {
    scn_mesh_clean_report_t dup;
    memset(&dup, 0, sizeof(dup));
    if (int rc = step_dedup(m, s, dup, st)) return rc;
    rep.autoclean_duplicate_faces = dup.duplicate_faces;
    if (int rc = drop_unreferenced(m, s, st, h_small)) return rc;
  }
  SCN_CUDA_TRY(cudaEventRecord(ev[4].get(), st));
  SCN_CUDA_TRY(cudaEventRecord(ev[7].get(), st));
  if (after) {
    rep.clean.vertices_in = m.nV; rep.clean.faces_in = m.nF;
    if (int rc = run_clean_steps(m, *after, s, rep.clean, st, err.as<unsigned>(), h_small, ev + 7)) return rc;
    rep.clean.vertices_out = m.nV; rep.clean.faces_out = m.nF;
  }
  SCN_CUDA_TRY(cudaEventRecord(ev[5].get(), st));
  if (int rc = download_mesh(m, xyz_out, rgb_out, tri_out, ev[6].get(), st, "scn_mesh_simplify")) return rc;
  rep.vertices_out = m.nV; rep.faces_out = m.nF;
  rep.upload_ms = ms_between(ev[0], ev[1]); rep.quadrics_ms = ms_between(ev[1], ev[2]); rep.rounds_ms = ms_between(ev[2], ev[3]);
  rep.autoclean_ms = ms_between(ev[3], ev[4]); rep.clean_ms = ms_between(ev[4], ev[5]); rep.download_ms = ms_between(ev[5], ev[6]);
  rep.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  *nV_out = m.nV; *nF_out = m.nF;
  if (report) *report = rep;
  return SCN_OK;
}

}  // extern "C"
