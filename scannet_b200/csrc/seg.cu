// Segmentator on H100 (sm_90a): Felzenszwalb–Huttenlocher graph segmentation of a triangle mesh
// on vertex normals, bit-identical to /root/reference/Segmentator/segmentator.cpp compiled with
// libstdc++ (GCC 13).
//
//   K1  k_face_normals / k_fill_csr / k_vertex_normals   segmentator.cpp:185-208
//       The reference's vertex normal is a SEQUENTIAL running average in face-file order; each
//       vertex replays its incident (face, corner) list in ascending order, so the float result is
//       the same bit pattern.
//   K2  k_edge_weights                                    segmentator.cpp:211-229
//   K3  introsort emulation                               segmentator.cpp:67-72 (std::sort, comparator on w only)
//       std::sort's tie order is observable in segIndices (SURVEY.md §0 fact 4).  libstdc++'s
//       introsort (bits/stl_algo.h:1848-1952) is reproduced exactly, in parallel:
//         tier 1  level-synchronous over the recursion tree: every segment longer than kSmall is
//                 partitioned by ALL CTAs with a parallel formulation of __unguarded_partition
//                 (the k-th element >= pivot from the left swaps with the k-th element <= pivot from
//                 the right while their positions have not crossed; two device-wide scans per level);
//         tier 2  one warp per remaining segment (<= kSmall records): the warp stages the segment in shared memory,
//                 lane 0 runs the literal sequential introsort loop + insertion sort there.
//       The final __final_insertion_sort pass never moves a record across a partition boundary, so
//       running it per segment is identical to running it over the whole array.
//   S5-S7 Kruskal-with-threshold, small-segment merge and labelling (segmentator.cpp:71-91,236-250)
//       are a strictly sequential, latency-bound replay (edge i's decision depends on the forest left
//       by edges 0..i-1); they run on the host over the device-sorted records.
// Float arithmetic: explicit round-to-nearest intrinsics, no contraction (-fmad=false), IEEE sqrt/div.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <new>
#include <thread>
#include <vector>

#include <sys/mman.h>

#include "scan.cuh"
#include "scn_common.h"

namespace {

using scn::block_excl_scan;

constexpr int kSmall = 256;          // tier-2 threshold (records)
constexpr int kTile = 2048;          // tier-1 tile (records per CTA)
constexpr int kTileThreads = 256;
constexpr int kTileItems = kTile / kTileThreads;   // 8

struct Rec { float w; unsigned i; };
static_assert(sizeof(Rec) == 8, "Rec must be 8 bytes");
struct Edge12 { float w; int a, b; };
static_assert(sizeof(Edge12) == 12, "edge record must be 12 bytes");

// ------------------------------------------------------------------------------ K1: normals
__global__ void k_face_normals(const float* __restrict__ xyz, const unsigned* __restrict__ tri, size_t nF,
                               size_t nV, float4* __restrict__ fn, unsigned* __restrict__ deg) {
  const size_t f = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (f >= nF) return;
  const unsigned i1 = tri[3 * f], i2 = tri[3 * f + 1], i3 = tri[3 * f + 2];
  const float* p1 = xyz + 3 * (size_t)i1; const float* p2 = xyz + 3 * (size_t)i2; const float* p3 = xyz + 3 * (size_t)i3;
  const float ux = __fsub_rn(p2[0], p1[0]), uy = __fsub_rn(p2[1], p1[1]), uz = __fsub_rn(p2[2], p1[2]);
  const float vx = __fsub_rn(p3[0], p1[0]), vy = __fsub_rn(p3[1], p1[1]), vz = __fsub_rn(p3[2], p1[2]);
  float cx = __fsub_rn(__fmul_rn(uy, vz), __fmul_rn(uz, vy));
  float cy = __fsub_rn(__fmul_rn(uz, vx), __fmul_rn(ux, vz));
  float cz = __fsub_rn(__fmul_rn(ux, vy), __fmul_rn(uy, vx));
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
  cx = __fdiv_rn(cx, len); cy = __fdiv_rn(cy, len); cz = __fdiv_rn(cz, len);
  fn[f] = make_float4(cx, cy, cz, 0.f);
  atomicAdd(&deg[i1], 1u); atomicAdd(&deg[i2], 1u); atomicAdd(&deg[i3], 1u);
}

__global__ void k_fill_csr(const unsigned* __restrict__ tri, size_t nF, const unsigned* __restrict__ off,
                           unsigned* __restrict__ cursor, unsigned* __restrict__ csr) {
  const size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x;       // corner id = 3f+k
  if (c >= 3 * nF) return;
  const unsigned v = tri[c];
  const unsigned pos = atomicAdd(&cursor[v], 1u);
  csr[off[v] + pos] = (unsigned)c;
}

__device__ void heap_sift_u32(unsigned* a, unsigned hole, unsigned len, unsigned val) {
  for (;;) {
    unsigned child = 2 * hole + 1;
    if (child >= len) break;
    if (child + 1 < len && a[child + 1] > a[child]) ++child;
    if (a[child] <= val) break;
    a[hole] = a[child]; hole = child;
  }
  a[hole] = val;
}

// one thread per vertex: sort its corner list ascending, replay the running average (segmentator.cpp:203-207)
__global__ void k_vertex_normals(const unsigned* __restrict__ off, unsigned* __restrict__ csr,
                                 const float4* __restrict__ fn, size_t nV, float* __restrict__ nrm) {
  const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (v >= nV) return;
  const unsigned b = off[v], n = off[v + 1] - b;
  unsigned loc[32];
  unsigned* lst = csr + b;
  const bool small = n <= 32;
  if (small) {
    for (unsigned i = 0; i < n; ++i) {                        // insertion sort into registers/local
      const unsigned c = lst[i];
      unsigned j = i;
      while (j > 0 && loc[j - 1] > c) { loc[j] = loc[j - 1]; --j; }
      loc[j] = c;
    }
  } else {                                                     // in-place heap sort in global memory
    for (unsigned p = n / 2; p-- > 0;) heap_sift_u32(lst, p, n, lst[p]);
    for (unsigned last = n; last > 1;) { --last; const unsigned t = lst[last]; lst[last] = lst[0]; heap_sift_u32(lst, 0, last, t); }
  }
  float nx = 0.f, ny = 0.f, nz = 0.f;
  unsigned cnt = 0, pending = 0, prev_f = 0xFFFFFFFFu;
  for (unsigned i = 0; i < n; ++i) {
    const unsigned c = small ? loc[i] : lst[i];
    const unsigned f = c / 3u;
    if (f != prev_f) { cnt += pending; pending = 0; prev_f = f; }   // counts[] bumped only after the face's 3 lerps
    const float4 q = fn[f];
    const float t = __fdiv_rn(1.0f, __fadd_rn((float)cnt, 1.0f));
    const float u = __fsub_rn(1.0f, t);
    nx = __fadd_rn(__fmul_rn(t, q.x), __fmul_rn(u, nx));
    ny = __fadd_rn(__fmul_rn(t, q.y), __fmul_rn(u, ny));
    nz = __fadd_rn(__fmul_rn(t, q.z), __fmul_rn(u, nz));
    ++pending;
  }
  nrm[3 * v] = nx; nrm[3 * v + 1] = ny; nrm[3 * v + 2] = nz;
}

// ------------------------------------------------------------------------------ K2: edge weights
__device__ __forceinline__ void edge_ends(const unsigned* __restrict__ tri, size_t e, unsigned& a, unsigned& b) {
  const size_t f = e / 3; const unsigned k = (unsigned)(e - 3 * f);
  const unsigned i1 = tri[3 * f], i2 = tri[3 * f + 1], i3 = tri[3 * f + 2];
  if (k == 0) { a = i1; b = i2; } else if (k == 1) { a = i1; b = i3; } else { a = i3; b = i2; }   // segmentator.cpp:198-200
}

__global__ void k_edge_weights(const float* __restrict__ xyz, const unsigned* __restrict__ tri,
                               const float* __restrict__ nrm, size_t nE, Rec* __restrict__ rec) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= nE) return;
  unsigned a, b;
  edge_ends(tri, e, a, b);
  const float* n1 = nrm + 3 * (size_t)a; const float* n2 = nrm + 3 * (size_t)b;
  const float* p1 = xyz + 3 * (size_t)a; const float* p2 = xyz + 3 * (size_t)b;
  float dx = __fsub_rn(p2[0], p1[0]), dy = __fsub_rn(p2[1], p1[1]), dz = __fsub_rn(p2[2], p1[2]);
  const float dd = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  dx = __fdiv_rn(dx, dd); dy = __fdiv_rn(dy, dd); dz = __fdiv_rn(dz, dd);
  const float n2x = n2[0], n2y = n2[1], n2z = n2[2];
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(n1[0], n2x), __fmul_rn(n1[1], n2y)), __fmul_rn(n1[2], n2z));
  const float dot2 = __fadd_rn(__fadd_rn(__fmul_rn(n2x, dx), __fmul_rn(n2y, dy)), __fmul_rn(n2z, dz));
  float ww = __fsub_rn(1.0f, dot);
  if (dot2 > 0) ww = __fmul_rn(ww, ww);
  rec[e].w = ww; rec[e].i = (unsigned)e;
}

__global__ void k_gather_edges(const Rec* __restrict__ rec, const unsigned* __restrict__ tri, size_t nE, Edge12* __restrict__ out) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE) return;
  const Rec r = rec[j];
  unsigned a, b;
  edge_ends(tri, r.i, a, b);
  out[j].w = r.w; out[j].a = (int)a; out[j].b = (int)b;
}
__global__ void k_gather_edges12(const Rec* __restrict__ rec, const Edge12* __restrict__ src, size_t nE, Edge12* __restrict__ out) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE) return;
  out[j] = src[rec[j].i];
}
__global__ void k_rec_from_edges12(const Edge12* __restrict__ src, size_t nE, Rec* __restrict__ rec) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE) return;
  rec[j].w = src[j].w; rec[j].i = (unsigned)j;
}

// ------------------------------------------------------------------------------ K3: libstdc++ introsort
struct SortCtl {           // device-resident counters
  unsigned n_next;         // large segments emitted for the next level
  unsigned n_small;        // tier-2 segments
  unsigned n_heap;         // depth-limit fallback segments
  unsigned pad;
};

// sequential pieces (bits/stl_heap.h, bits/stl_algo.h), used by tier 2 and the heap fallback
__device__ __forceinline__ bool rec_lt(const Rec& x, const Rec& y) { return x.w < y.w; }

__device__ void d_adjust_heap(Rec* a, long hole, long len, Rec val) {
  const long top = hole;
  long child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (rec_lt(a[child], a[child - 1])) child--;
    a[hole] = a[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    a[hole] = a[child - 1];
    hole = child - 1;
  }
  long parent = (hole - 1) / 2;
  while (hole > top && rec_lt(a[parent], val)) { a[hole] = a[parent]; hole = parent; parent = (hole - 1) / 2; }
  a[hole] = val;
}
__device__ void d_heap_sort(Rec* a, long len) {            // __partial_sort(first, last, last)
  if (len >= 2) for (long parent = (len - 2) / 2;; --parent) { d_adjust_heap(a, parent, len, a[parent]); if (parent == 0) break; }
  for (long last = len; last > 1;) { --last; const Rec v = a[last]; a[last] = a[0]; d_adjust_heap(a, 0, last, v); }
}
__device__ __forceinline__ void d_swap(Rec* x, Rec* y) { const Rec t = *x; *x = *y; *y = t; }
__device__ __forceinline__ void d_median_to_first(Rec* r, Rec* x, Rec* y, Rec* z) {   // __move_median_to_first
  if (rec_lt(*x, *y)) {
    if (rec_lt(*y, *z)) d_swap(r, y); else if (rec_lt(*x, *z)) d_swap(r, z); else d_swap(r, x);
  } else if (rec_lt(*x, *z)) d_swap(r, x);
  else if (rec_lt(*y, *z)) d_swap(r, z);
  else d_swap(r, y);
}
__device__ long d_partition_pivot(Rec* a, long first, long last) {
  const long mid = first + (last - first) / 2;
  d_median_to_first(a + first, a + first + 1, a + mid, a + last - 1);
  long lo = first + 1, hi = last;
  const Rec piv = a[first];
  for (;;) {
    while (rec_lt(a[lo], piv)) ++lo;
    --hi;
    while (rec_lt(piv, a[hi])) --hi;
    if (!(lo < hi)) return lo;
    d_swap(a + lo, a + hi);
    ++lo;
  }
}
__device__ void d_insertion_sort(Rec* a, long n) {        // __insertion_sort on a whole (<= kSmall) segment
  for (long i = 1; i < n; ++i) {
    const Rec v = a[i];
    if (rec_lt(v, a[0])) { for (long j = i; j > 0; --j) a[j] = a[j - 1]; a[0] = v; }
    else { long j = i; while (rec_lt(v, a[j - 1])) { a[j] = a[j - 1]; --j; } a[j] = v; }
  }
}

// tier 2: one WARP per segment.  The segment (<= kSmall records = 2 KB) is copied into shared memory by the warp, lane 0 runs
// the literal sequential introsort + insertion sort there, the warp copies it back.  (One thread per segment working in
// global memory was most of the sort's time: ~2,300 threads, every access a dependent L2 round trip.)
constexpr int kSmallWarps = 4;
__global__ void __launch_bounds__(32 * kSmallWarps)
k_sort_small(Rec* A, const unsigned* __restrict__ s_start, const unsigned* __restrict__ s_lend, unsigned n_small) {
  __shared__ Rec s_buf[kSmallWarps][kSmall];
  const unsigned g = blockIdx.x * kSmallWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (g >= n_small) return;
  Rec* const src = A + s_start[g];
  const long len = (long)(s_lend[g] >> 8);
  const int depth0 = (int)(s_lend[g] & 0xFFu);
  Rec* const a = s_buf[threadIdx.x >> 5];
  for (long i = lane; i < len; i += 32) a[i] = src[i];
  __syncwarp();
  if (lane == 0) {
    // explicit stack for `__introsort_loop(cut, last, depth)` (recursion on the right part, loop on the left)
    long st_first[64], st_last[64]; int st_depth[64]; int sp = 0;
    long first = 0, last = len; int depth = depth0;
    for (;;) {
      while (last - first > 16) {
        if (depth == 0) { d_heap_sort(a + first, last - first); break; }
        --depth;
        const long cut = d_partition_pivot(a, first, last);
        // recurse right first in the reference; order between disjoint parts does not matter, push the right part
        st_first[sp] = cut; st_last[sp] = last; st_depth[sp] = depth; ++sp;
        last = cut;
      }
      if (sp == 0) break;
      --sp; first = st_first[sp]; last = st_last[sp]; depth = st_depth[sp];
    }
    d_insertion_sort(a, len);
  }
  __syncwarp();
  for (long i = lane; i < len; i += 32) src[i] = a[i];
}

__global__ void k_sort_heap_fallback(Rec* __restrict__ A, const unsigned* __restrict__ h_start, const unsigned* __restrict__ h_end,
                                     unsigned n_heap) {
  const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_heap) return;
  d_heap_sort(A + h_start[g], (long)h_end[g] - (long)h_start[g]);
}

// tier 1 -----------------------------------------------------------------------------------------
// per segment: median-of-3 to front (bits/stl_algo.h:1890-1900) and the number of tiles covering [s+1, e)
__device__ __forceinline__ void d_pivot(unsigned g, Rec* A, const unsigned* segS, const unsigned* segE,
                                        unsigned* tileCnt) {
  const long first = segS[g], last = segE[g];
  const long mid = first + (last - first) / 2;
  d_median_to_first(A + first, A + first + 1, A + mid, A + last - 1);
  tileCnt[g] = (unsigned)((last - first - 1 + kTile - 1) / kTile);
}
__global__ void k_pivot(Rec* __restrict__ A, const unsigned* __restrict__ segS, const unsigned* __restrict__ segE,
                        unsigned nseg, unsigned* __restrict__ tileCnt) {
  const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < nseg) d_pivot(g, A, segS, segE, tileCnt);
}

__device__ __forceinline__ unsigned find_seg(const unsigned* tileOff, unsigned nseg, unsigned tile) {
  unsigned lo = 0, hi = nseg;                 // largest g with tileOff[g] <= tile
  while (hi - lo > 1) { const unsigned m = (lo + hi) >> 1; if (tileOff[m] <= tile) lo = m; else hi = m; }
  return lo;
}

struct TileCtx { unsigned g, s, e, t0; long base, end; float piv; };
__device__ __forceinline__ TileCtx tile_ctx(const Rec* A, const unsigned* segS, const unsigned* segE,
                                            const unsigned* tileOff, unsigned nseg, unsigned tile) {
  __shared__ TileCtx sc;
  __syncthreads();                                    // (the persistent kernel calls this in a loop: the previous tile's readers are done)
  if (threadIdx.x == 0) {
    TileCtx c;
    c.g = find_seg(tileOff, nseg, tile);
    c.s = segS[c.g]; c.e = segE[c.g]; c.t0 = tileOff[c.g];
    c.base = (long)c.s + 1 + (long)(tile - c.t0) * kTile;
    c.end = min((long)c.e, c.base + kTile);
    c.piv = A[c.s].w;
    sc = c;
  }
  __syncthreads();
  return sc;
}

__device__ __forceinline__ void d_count(unsigned tile, const Rec* A, const unsigned* segS, const unsigned* segE,
        const unsigned* tileOff, unsigned nseg, unsigned* tL, unsigned* tR) {
  const TileCtx c = tile_ctx(A, segS, segE, tileOff, nseg, tile);
  unsigned nl = 0, nr = 0;
  const long p0 = c.base + (long)threadIdx.x * kTileItems;
#pragma unroll
  for (int i = 0; i < kTileItems; ++i) {
    const long p = p0 + i;
    if (p < c.end) { const float w = A[p].w; nl += !(w < c.piv); nr += !(c.piv < w); }
  }
  unsigned totl, totr;
  block_excl_scan(nl, &totl);
  block_excl_scan(nr, &totr);
  if (threadIdx.x == 0) { tL[tile] = totl; tR[tile] = totr; }
}
__global__ void __launch_bounds__(kTileThreads)
k_count(const Rec* __restrict__ A, const unsigned* __restrict__ segS, const unsigned* __restrict__ segE,
        const unsigned* __restrict__ tileOff, unsigned nseg, unsigned* __restrict__ tL, unsigned* __restrict__ tR) {
  d_count(blockIdx.x, A, segS, segE, tileOff, nseg, tL, tR);
}

__device__ __forceinline__ void d_scatter(unsigned tile, const Rec* A, const unsigned* segS, const unsigned* segE,
          const unsigned* tileOff, unsigned nseg, const unsigned* gL, const unsigned* gR,
          const unsigned* tR, unsigned* Lpos, unsigned* Rpos) {
  const TileCtx c = tile_ctx(A, segS, segE, tileOff, nseg, tile);
  const unsigned t1 = tileOff[c.g + 1];
  const unsigned baseL = gL[tile] - gL[c.t0];
  const unsigned totR = gR[t1] - gR[c.t0];
  const unsigned baseR = totR - (gR[tile] - gR[c.t0]) - tR[tile];     // right stoppers in later tiles
  bool fl[kTileItems], fr[kTileItems];
  unsigned nl = 0, nr = 0;
  const long p0 = c.base + (long)threadIdx.x * kTileItems;
#pragma unroll
  for (int i = 0; i < kTileItems; ++i) {
    const long p = p0 + i;
    fl[i] = fr[i] = false;
    if (p < c.end) { const float w = A[p].w; fl[i] = !(w < c.piv); fr[i] = !(c.piv < w); }
    nl += fl[i]; nr += fr[i];
  }
  unsigned totr_tile;
  unsigned exl = block_excl_scan(nl, nullptr);
  unsigned exr = block_excl_scan(nr, &totr_tile);
  // left stoppers: ascending rank from the left; right stoppers: rank counted from the right end
  unsigned rl = baseL + exl;
  unsigned after = totr_tile - exr - nr;                // right stoppers in later threads of this tile
  unsigned rr_end = baseR + after + nr;                 // rank (from right) just past this thread's first item
#pragma unroll
  for (int i = 0; i < kTileItems; ++i) {
    const long p = p0 + i;
    if (fl[i]) { Lpos[c.s + rl] = (unsigned)p; ++rl; }
    if (fr[i]) { --rr_end; Rpos[c.s + rr_end] = (unsigned)p; }
  }
}
__global__ void __launch_bounds__(kTileThreads)
k_scatter(const Rec* __restrict__ A, const unsigned* __restrict__ segS, const unsigned* __restrict__ segE,
          const unsigned* __restrict__ tileOff, unsigned nseg, const unsigned* __restrict__ gL, const unsigned* __restrict__ gR,
          const unsigned* __restrict__ tR, unsigned* __restrict__ Lpos, unsigned* __restrict__ Rpos) {
  d_scatter(blockIdx.x, A, segS, segE, tileOff, nseg, gL, gR, tR, Lpos, Rpos);
}

// swaps + cut.  k-th pair (Lpos[s+k], Rpos[s+k]) swaps iff Lpos < Rpos; cut = min(L[m], R[m-1]).
__device__ __forceinline__ void d_swap_tile(unsigned tile, Rec* A, const unsigned* segS, const unsigned* segE,
       const unsigned* tileOff, unsigned nseg, const unsigned* gL, const unsigned* gR,
       const unsigned* Lpos, const unsigned* Rpos, unsigned* segCut) {
  const TileCtx c = tile_ctx(A, segS, segE, tileOff, nseg, tile);
  const unsigned t1 = tileOff[c.g + 1];
  const unsigned nL = gL[t1] - gL[c.t0], nR = gR[t1] - gR[c.t0];
  const unsigned mn = min(nL, nR);
  const unsigned k0 = (tile - c.t0) * kTile + threadIdx.x * kTileItems;
#pragma unroll
  for (int i = 0; i < kTileItems; ++i) {
    const unsigned k = k0 + i;
    if (k >= mn) break;
    const unsigned L = Lpos[c.s + k], R = Rpos[c.s + k];
    const bool sw = L < R;
    if (sw) { const Rec t = A[L]; A[L] = A[R]; A[R] = t; }
    if (k == 0 && !sw) segCut[c.g] = L;                                        // m = 0
    if (sw) {
      const bool last = (k + 1 >= mn) || !(Lpos[c.s + k + 1] < Rpos[c.s + k + 1]);
      if (last) {                                                              // m = k+1
        const unsigned m = k + 1;
        const unsigned lm = m < nL ? Lpos[c.s + m] : 0xFFFFFFFFu;
        segCut[c.g] = min(lm, R);
      }
    }
  }
}
__global__ void __launch_bounds__(kTileThreads)
k_swap(Rec* __restrict__ A, const unsigned* __restrict__ segS, const unsigned* __restrict__ segE,
       const unsigned* __restrict__ tileOff, unsigned nseg, const unsigned* __restrict__ gL, const unsigned* __restrict__ gR,
       const unsigned* __restrict__ Lpos, const unsigned* __restrict__ Rpos, unsigned* __restrict__ segCut) {
  d_swap_tile(blockIdx.x, A, segS, segE, tileOff, nseg, gL, gR, Lpos, Rpos, segCut);
}

__device__ __forceinline__ void d_children(unsigned g, const unsigned* segS, const unsigned* segE, const unsigned* segD,
                           const unsigned* segCut,
                           unsigned* nS, unsigned* nE, unsigned* nD,
                           unsigned* smStart, unsigned* smLenD,
                           unsigned* hpStart, unsigned* hpEnd, SortCtl* ctl) {
  const unsigned s = segS[g], e = segE[g], cut = segCut[g], d = segD[g] - 1;
  const unsigned cs[2] = { s, cut }, ce[2] = { cut, e };
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const unsigned len = ce[c] - cs[c];
    if (len <= 1) continue;
    if (len <= (unsigned)kSmall) { const unsigned p = atomicAdd(&ctl->n_small, 1u); smStart[p] = cs[c]; smLenD[p] = (len << 8) | d; }
    else if (d == 0) { const unsigned p = atomicAdd(&ctl->n_heap, 1u); hpStart[p] = cs[c]; hpEnd[p] = ce[c]; }
    else { const unsigned p = atomicAdd(&ctl->n_next, 1u); nS[p] = cs[c]; nE[p] = ce[c]; nD[p] = d; }
  }
}
__global__ void k_children(const unsigned* __restrict__ segS, const unsigned* __restrict__ segE, const unsigned* __restrict__ segD,
                           const unsigned* __restrict__ segCut, unsigned nseg,
                           unsigned* __restrict__ nS, unsigned* __restrict__ nE, unsigned* __restrict__ nD,
                           unsigned* __restrict__ smStart, unsigned* __restrict__ smLenD,
                           unsigned* __restrict__ hpStart, unsigned* __restrict__ hpEnd, SortCtl* __restrict__ ctl) {
  const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < nseg) d_children(g, segS, segE, segD, segCut, nS, nE, nD, smStart, smLenD, hpStart, hpEnd, ctl);
}

// ---- the whole tier-1 loop as ONE persistent kernel ------------------------------------------------------------------
// The level-synchronous partitioning used to be ~8 kernel launches and two host round trips (tile count, child count) per
// level of the recursion tree - 254 launches for a 50 k-vertex mesh, launch- and sync-bound.  Here every resident CTA loops
// over the levels itself: the phases of a level are separated by a grid-wide barrier (cooperative launch: all CTAs are
// co-resident), tiles and segments are taken grid-stride, the three small scans of a level run inside one CTA, and the
// loop ends on the device when no large segment is left.
struct SortLevelsArgs {
  Rec* A;
  unsigned* seg[2];              // S | E | D, each maxLarge long
  unsigned maxLarge;
  unsigned* cut; unsigned* tileCnt; unsigned* tileOff; unsigned* tL; unsigned* tR; unsigned* gL; unsigned* gR;
  unsigned* Lpos; unsigned* Rpos; unsigned* smStart; unsigned* smLenD; unsigned* hpStart; unsigned* hpEnd;
  SortCtl* ctl; unsigned* bar;   // bar[0] arrivals, bar[1] generation, bar[2] levels done
  unsigned nseg0;
};
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned gen = *(volatile unsigned*)&bar[1];
    if (atomicAdd(&bar[0], 1u) == nblocks - 1) { bar[0] = 0; __threadfence(); atomicAdd(&bar[1], 1u); }
    else { while (*(volatile unsigned*)&bar[1] == gen) __nanosleep(40); }      // back off: hundreds of CTAs polling one line starve the arrivals
    __threadfence();
  }
  __syncthreads();
}
// (none of the device functions above takes __restrict__ pointers: inside the persistent kernel these arrays are written by
//  other CTAs between grid barriers, so their loads must stay coherent - no ld.global.nc)
// exclusive scan of in[0..n) into out[0..n], out[n] = total, by ONE CTA of kTileThreads threads
__device__ void cta_scan(const unsigned* in, unsigned* out, unsigned n) {
  __shared__ unsigned s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (unsigned base = 0; base < n; base += kTile) {
    unsigned v[kTileItems], sum = 0;
    const unsigned p0 = base + threadIdx.x * kTileItems;
#pragma unroll
    for (int i = 0; i < kTileItems; ++i) { v[i] = p0 + i < n ? in[p0 + i] : 0u; sum += v[i]; }
    unsigned tot;
    unsigned ex = block_excl_scan(sum, &tot) + s_carry;
#pragma unroll
    for (int i = 0; i < kTileItems; ++i) { if (p0 + i < n) out[p0 + i] = ex; ex += v[i]; }
    __syncthreads();
    if (threadIdx.x == 0) s_carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) out[n] = s_carry;
  __syncthreads();
}
__global__ void __launch_bounds__(kTileThreads)
k_sort_levels(const SortLevelsArgs a) {
  const unsigned nb = gridDim.x, gsz = nb * kTileThreads, gtid = blockIdx.x * kTileThreads + threadIdx.x;
  unsigned nseg = a.nseg0, levels = 0;
  int cur = 0;
  while (nseg > 0) {
    const unsigned* S = a.seg[cur]; const unsigned* E = S + a.maxLarge; const unsigned* D = S + 2 * a.maxLarge;
    unsigned* NS = a.seg[cur ^ 1]; unsigned* NE = NS + a.maxLarge; unsigned* ND = NS + 2 * a.maxLarge;
    for (unsigned g = gtid; g < nseg; g += gsz) d_pivot(g, a.A, S, E, a.tileCnt);
    grid_barrier(a.bar, nb);
    if (blockIdx.x == 0) { cta_scan(a.tileCnt, a.tileOff, nseg); if (threadIdx.x == 0) a.ctl->n_next = 0; }   // (all CTAs read n_next before the barrier above)
    grid_barrier(a.bar, nb);
    const unsigned ntiles = *(volatile unsigned*)&a.tileOff[nseg];
    for (unsigned t = blockIdx.x; t < ntiles; t += nb) d_count(t, a.A, S, E, a.tileOff, nseg, a.tL, a.tR);
    grid_barrier(a.bar, nb);
    if (blockIdx.x == 0) cta_scan(a.tL, a.gL, ntiles);
    if (blockIdx.x == nb - 1) cta_scan(a.tR, a.gR, ntiles);
    grid_barrier(a.bar, nb);
    for (unsigned t = blockIdx.x; t < ntiles; t += nb) d_scatter(t, a.A, S, E, a.tileOff, nseg, a.gL, a.gR, a.tR, a.Lpos, a.Rpos);
    grid_barrier(a.bar, nb);
    for (unsigned t = blockIdx.x; t < ntiles; t += nb) d_swap_tile(t, a.A, S, E, a.tileOff, nseg, a.gL, a.gR, a.Lpos, a.Rpos, a.cut);
    grid_barrier(a.bar, nb);
    for (unsigned g = gtid; g < nseg; g += gsz) d_children(g, S, E, D, a.cut, NS, NE, ND, a.smStart, a.smLenD, a.hpStart, a.hpEnd, a.ctl);
    grid_barrier(a.bar, nb);
    nseg = *(volatile unsigned*)&a.ctl->n_next;
    // n_next is re-armed by gtid 0 during the NEXT level's pivot phase (two barriers from here, and five before the next
    // children phase adds to it) - every CTA has long read it by then
    ++levels;
    cur ^= 1;
    if (nseg > 0 && gtid == 0) a.bar[3] = nseg;       // (kept for inspection: segments of the level about to start)
  }
  if (gtid == 0) a.bar[2] = levels;
}

// ------------------------------------------------------------------------------ replay pruning
// In BOTH sequential passes an edge whose (unordered) endpoint pair already occurred earlier in sorted order is a
// provable no-op: if the earlier copy joined its components this one finds a == b; if the earlier copy was rejected
// then (Kruskal) one of its components had threshold < w and is frozen for every later, heavier edge (a component's
// threshold only changes when it merges, which needs w <= threshold), or (small-segment pass) both components already
// had >= segMinVerts vertices and sizes only grow.  Self-loops are no-ops too.  Dropping them halves the host replay
// for a manifold mesh (every interior edge is emitted once per adjacent face) without changing a single id.
__global__ void k_pair_first(const Rec* __restrict__ rec, const unsigned* __restrict__ tri, const Edge12* __restrict__ src, size_t nE,
                             unsigned long long* __restrict__ tkeys, unsigned* __restrict__ tmin, unsigned tmask) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE) return;
  unsigned a, b;
  if (tri) edge_ends(tri, rec[j].i, a, b); else { a = (unsigned)src[rec[j].i].a; b = (unsigned)src[rec[j].i].b; }
  if (a == b) return;
  const unsigned lo = min(a, b), hi = max(a, b);
  const unsigned long long key = ((unsigned long long)hi << 32) | lo;
  unsigned h = (lo * 73856093u) ^ (hi * 19349669u); h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
  unsigned slot = h & tmask;
  for (;;) {
    const unsigned long long k = tkeys[slot];
    if (k == key) break;
    if (k == ~0ull) { const unsigned long long old = atomicCAS(&tkeys[slot], ~0ull, key); if (old == ~0ull || old == key) break; }
    slot = (slot + 1) & tmask;
  }
  atomicMin(&tmin[slot], (unsigned)j);
}
__global__ void k_pair_keep(const Rec* __restrict__ rec, const unsigned* __restrict__ tri, const Edge12* __restrict__ src, size_t nE,
                            const unsigned long long* __restrict__ tkeys, const unsigned* __restrict__ tmin, unsigned tmask,
                            unsigned* __restrict__ keep) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE) return;
  unsigned a, b;
  if (tri) edge_ends(tri, rec[j].i, a, b); else { a = (unsigned)src[rec[j].i].a; b = (unsigned)src[rec[j].i].b; }
  unsigned kp = 0;
  if (a != b) {
    const unsigned lo = min(a, b), hi = max(a, b);
    const unsigned long long key = ((unsigned long long)hi << 32) | lo;
    unsigned h = (lo * 73856093u) ^ (hi * 19349669u); h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
    unsigned slot = h & tmask;
    while (tkeys[slot] != key) slot = (slot + 1) & tmask;
    kp = tmin[slot] == (unsigned)j;
  }
  keep[j] = kp;
}
__global__ void k_compact_edges(const Rec* __restrict__ rec, const unsigned* __restrict__ tri, const Edge12* __restrict__ src, size_t nE,
                                const unsigned* __restrict__ keep, const unsigned* __restrict__ pos, Edge12* __restrict__ out) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nE || !keep[j]) return;
  const Rec r = rec[j];
  unsigned a, b;
  if (tri) edge_ends(tri, r.i, a, b); else { a = (unsigned)src[r.i].a; b = (unsigned)src[r.i].b; }
  Edge12 e; e.w = r.w; e.a = (int)a; e.b = (int)b;
  out[pos[j]] = e;
}

// ------------------------------------------------------------------------------ host side
// Workspace: a per-thread cached device arena (bump allocator).  cudaMalloc/cudaFree cost ~0.1-1 ms each and
// synchronise the device; with ~25 buffers per call they dominated small meshes.  The arena is reset at the start of
// every top-level call and regrown to a single chunk when a call overflowed it.
struct Arena {
  struct Chunk { char* p; size_t cap; };
  std::vector<Chunk> chunks; size_t used = 0, total_req = 0, last_total = 0; int dev = -1;
  void release() { for (Chunk& c : chunks) cudaFree(c.p); chunks.clear(); used = 0; }
  void reset() {
    int d = 0; cudaGetDevice(&d);
    if (d != dev || chunks.size() > 1) { release(); dev = d; }     // a call that overflowed its chunk: start over with one big enough
    last_total = total_req; used = 0; total_req = 0;
  }
  // make room for `bytes` more in one chunk (called once per top-level call, right after reset(), with an upper bound of its
  // needs); the chunk is kept across calls, so steady-state calls of similar size never touch cudaMalloc
  void reserve(size_t bytes) {
    bytes = std::max(bytes, last_total + (last_total >> 3));
    if (!chunks.empty() && used + bytes <= chunks.back().cap) return;
    if (used == 0) release();                                       // nothing live yet: replace rather than accumulate
    Chunk c{nullptr, bytes + (1u << 20)};
    if (cudaMalloc(&c.p, c.cap) != cudaSuccess) { cudaGetLastError(); return; }   // fall back to piecemeal chunks
    chunks.push_back(c); used = 0;
  }
  void* alloc(size_t bytes) {
    bytes = (bytes + 255) & ~size_t(255); if (!bytes) bytes = 256;
    total_req += bytes;
    if (!chunks.empty() && used + bytes <= chunks.back().cap) { void* r = chunks.back().p + used; used += bytes; return r; }
    Chunk c{nullptr, std::max(bytes, size_t(8) << 20)};
    if (cudaMalloc(&c.p, c.cap) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    chunks.push_back(c); used = bytes;
    return c.p;
  }
};
thread_local Arena g_arena;
struct PinnedBuf { void* p = nullptr; size_t cap = 0; void* get(size_t n) { if (n > cap) { if (p) cudaFreeHost(p); p = nullptr; cap = 0; if (cudaHostAlloc(&p, n + (n >> 3), cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); p = nullptr; return nullptr; } cap = n + (n >> 3); } return p; } };
thread_local PinnedBuf g_pinned, g_pinned_in;

struct DevBuf {
  void* p = nullptr;
  template <typename T> T* as() { return (T*)p; }
  int alloc(size_t bytes) { p = g_arena.alloc(bytes); return p ? 0 : -1; }
};

thread_local float g_timings[8] = {0, 0, 0, 0, 0, 0, 0, 0};
thread_local unsigned g_sort_launches = 0;

// Sorts A[0..n) (device) exactly like libstdc++ std::sort with the `w`-only comparator.
int device_introsort(Rec* A, size_t n, cudaStream_t st, int forced_depth = 0) {
  g_sort_launches = 0;
  if (n < 2) return SCN_OK;
  if (n > 0x7FFFFFFFull) return scn::fail(SCN_ERR_ARG, "too many edges");
  int lg = 0; for (size_t t = n; t > 1; t >>= 1) ++lg;
  const unsigned depth0 = forced_depth > 0 ? (unsigned)forced_depth : 2u * (unsigned)lg;   // std::__lg(n) * 2
  const size_t maxLarge = n / (kSmall + 1) + 2, maxSmall = n / 2 + 2, maxTiles = n / kTile + maxLarge + 2;
  DevBuf bSeg[2], bCut, bTileCnt, bTileOff, bTL, bTR, bGL, bGR, bLpos, bRpos, bSm, bHp, bCtl, bScr;
  for (int i = 0; i < 2; ++i) if (bSeg[i].alloc(maxLarge * 3 * 4)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc");
  if (bCut.alloc(maxLarge * 4) || bTileCnt.alloc(maxLarge * 4) || bTileOff.alloc((maxLarge + 1) * 4) || bTL.alloc(maxTiles * 4) ||
      bTR.alloc(maxTiles * 4) || bGL.alloc((maxTiles + 1) * 4) || bGR.alloc((maxTiles + 1) * 4) || bLpos.alloc(n * 4) ||
      bRpos.alloc(n * 4) || bSm.alloc(maxSmall * 2 * 4) || bHp.alloc(maxLarge * 2 * 4) || bCtl.alloc(sizeof(SortCtl)) ||
      bScr.alloc(scn::scan_scratch_elems(std::max(maxTiles, maxLarge)) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (sort workspace)");
  unsigned* smStart = bSm.as<unsigned>(); unsigned* smLenD = smStart + maxSmall;
  unsigned* hpStart = bHp.as<unsigned>(); unsigned* hpEnd = hpStart + maxLarge;
  SortCtl* ctl = bCtl.as<SortCtl>();
  SCN_CUDA_TRY(cudaMemsetAsync(ctl, 0, sizeof(SortCtl), st));
  SortCtl h{};
  unsigned nseg = 0;
  int cur = 0;
  if (n <= (size_t)kSmall) {
    const unsigned s0 = 0, ld = ((unsigned)n << 8) | depth0;
    SCN_CUDA_TRY(cudaMemcpyAsync(smStart, &s0, 4, cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(smLenD, &ld, 4, cudaMemcpyHostToDevice, st));
    h.n_small = 1;
  } else {
    const unsigned init[3] = { 0u, (unsigned)n, depth0 };
    unsigned* S = bSeg[0].as<unsigned>();
    SCN_CUDA_TRY(cudaMemcpyAsync(S, &init[0], 4, cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(S + maxLarge, &init[1], 4, cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(S + 2 * maxLarge, &init[2], 4, cudaMemcpyHostToDevice, st));
    nseg = 1;
  }
  static const bool by_launches = getenv("SCN_SEG_SORT_LAUNCHES") != nullptr;      // the per-level launch sequence, kept for A/B timing
  // the persistent kernel wins on small inputs, where launches and host round trips dominate; on large inputs full-size grids
  // per phase hide memory latency better than the co-resident grid-stride CTAs
  if (nseg > 0 && !by_launches && n <= (size_t(2) << 20)) {
    // one cooperative launch runs every level (see k_sort_levels); grid = all co-resident CTAs
    static thread_local int coop_blocks = 0;
    if (!coop_blocks) {
      int dev = 0, sms = 0, occ = 0, coop = 0;
      SCN_CUDA_TRY(cudaGetDevice(&dev));
      SCN_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      SCN_CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
      SCN_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_sort_levels, kTileThreads, 0));
      coop_blocks = coop ? sms * std::max(1, std::min(occ, 2)) : -1;
    }
    if (coop_blocks > 0) {
      // no more CTAs than the first level has tiles: a barrier costs with the number of CTAs that poll it
      const int use_blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)coop_blocks, (n + kTile - 1) / kTile));
      DevBuf bBar;
      if (bBar.alloc(16)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc (sort barrier)");
      SCN_CUDA_TRY(cudaMemsetAsync(bBar.p, 0, 16, st));
      SortLevelsArgs a;
      a.A = A; a.seg[0] = bSeg[0].as<unsigned>(); a.seg[1] = bSeg[1].as<unsigned>(); a.maxLarge = (unsigned)maxLarge;
      a.cut = bCut.as<unsigned>(); a.tileCnt = bTileCnt.as<unsigned>(); a.tileOff = bTileOff.as<unsigned>();
      a.tL = bTL.as<unsigned>(); a.tR = bTR.as<unsigned>(); a.gL = bGL.as<unsigned>(); a.gR = bGR.as<unsigned>();
      a.Lpos = bLpos.as<unsigned>(); a.Rpos = bRpos.as<unsigned>(); a.smStart = smStart; a.smLenD = smLenD; a.hpStart = hpStart; a.hpEnd = hpEnd;
      a.ctl = ctl; a.bar = bBar.as<unsigned>(); a.nseg0 = nseg;
      void* params[] = { (void*)&a };
      SCN_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)k_sort_levels, dim3((unsigned)use_blocks), dim3(kTileThreads), params, 0, st));
      g_sort_launches += 1;
      SCN_CUDA_TRY(cudaMemcpyAsync(&h, ctl, sizeof(SortCtl), cudaMemcpyDeviceToHost, st));
      SCN_CUDA_TRY(cudaStreamSynchronize(st));
      nseg = 0;
    }
  }
  while (nseg > 0) {
    unsigned* S = bSeg[cur].as<unsigned>(); unsigned* E = S + maxLarge; unsigned* D = S + 2 * maxLarge;
    unsigned* NS = bSeg[cur ^ 1].as<unsigned>(); unsigned* NE = NS + maxLarge; unsigned* ND = NS + 2 * maxLarge;
    const unsigned gb = (nseg + 127) / 128;
    k_pivot<<<gb, 128, 0, st>>>(A, S, E, nseg, bTileCnt.as<unsigned>());
    g_sort_launches += 1 + scn::exclusive_scan_u32(bTileCnt.as<unsigned>(), bTileOff.as<unsigned>(), nseg, bScr.as<unsigned>(), st);
    unsigned ntiles = 0;
    SCN_CUDA_TRY(cudaMemcpyAsync(&ntiles, bTileOff.as<unsigned>() + nseg, 4, cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    k_count<<<ntiles, kTileThreads, 0, st>>>(A, S, E, bTileOff.as<unsigned>(), nseg, bTL.as<unsigned>(), bTR.as<unsigned>());
    g_sort_launches += 1 + scn::exclusive_scan_u32(bTL.as<unsigned>(), bGL.as<unsigned>(), ntiles, bScr.as<unsigned>(), st);
    g_sort_launches += scn::exclusive_scan_u32(bTR.as<unsigned>(), bGR.as<unsigned>(), ntiles, bScr.as<unsigned>(), st);
    k_scatter<<<ntiles, kTileThreads, 0, st>>>(A, S, E, bTileOff.as<unsigned>(), nseg, bGL.as<unsigned>(), bGR.as<unsigned>(),
                                                 bTR.as<unsigned>(), bLpos.as<unsigned>(), bRpos.as<unsigned>());
    k_swap<<<ntiles, kTileThreads, 0, st>>>(A, S, E, bTileOff.as<unsigned>(), nseg, bGL.as<unsigned>(), bGR.as<unsigned>(),
                                              bLpos.as<unsigned>(), bRpos.as<unsigned>(), bCut.as<unsigned>());
    k_children<<<gb, 128, 0, st>>>(S, E, D, bCut.as<unsigned>(), nseg, NS, NE, ND, smStart, smLenD, hpStart, hpEnd, ctl);
    g_sort_launches += 3;
    SCN_CUDA_TRY(cudaMemcpyAsync(&h, ctl, sizeof(SortCtl), cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    nseg = h.n_next;
    const unsigned zero = 0;
    SCN_CUDA_TRY(cudaMemcpyAsync(&ctl->n_next, &zero, 4, cudaMemcpyHostToDevice, st));
    cur ^= 1;
  }
  if (h.n_heap) { k_sort_heap_fallback<<<(h.n_heap + 63) / 64, 64, 0, st>>>(A, hpStart, hpEnd, h.n_heap); ++g_sort_launches; }
  if (h.n_small) { k_sort_small<<<(h.n_small + kSmallWarps - 1) / kSmallWarps, 32 * kSmallWarps, 0, st>>>(A, smStart, smLenD, h.n_small); ++g_sort_launches; }
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

// Sequential replay on the host (segmentator.cpp:71-91 Kruskal with adaptive threshold; :236-250) over the pruned
// records.  One 16-byte element per vertex (the threshold sits next to the root fields it is read with) and software
// prefetch of the endpoints a few edges ahead: the loop is bound by cache misses on random vertices.
struct UfElt { int rank, p, size; float thr; };
inline int uf_find(UfElt* u, int x) { int y = x; while (y != u[y].p) y = u[y].p; u[x].p = y; return y; }
inline void uf_join(UfElt* u, int x, int y) {
  if (u[x].rank > u[y].rank) { u[y].p = x; u[x].size += u[y].size; }
  else { u[x].p = y; u[y].size += u[x].size; if (u[x].rank == u[y].rank) u[y].rank++; }
}
// The replay is bound by dependent cache misses on the forest.  Measured on the GPU box's host (Xeon 8562Y+, 2 M-vertex mesh,
// 6 M records): plain find + prefetch 24 ahead 103 ms; prefetching the records 48 ahead and walking two parent links of the
// record 8 ahead (read-only) + full path compression 86 ms.  Path compression changes only parent pointers, never roots,
// ranks, sizes or thresholds, so the ids are the reference's.
inline int uf_find_full(UfElt* U, int x) {
  int y = x; while (y != U[y].p) y = U[y].p;
  while (U[x].p != y) { const int n = U[x].p; U[x].p = y; x = n; }
  return y;
}
// The forest is random-accessed 12 M times per 2 M-vertex mesh: back it with transparent huge pages (a heap allocation of a
// long-lived process is usually 4 KB-paged, which cost ~40 % in TLB misses) and keep it between calls.
template <typename T> struct HugeAlloc {
  using value_type = T;
  HugeAlloc() = default;
  template <typename U> HugeAlloc(const HugeAlloc<U>&) {}
  T* allocate(size_t n) {
    const size_t bytes = ((n * sizeof(T)) + (size_t(2) << 20) - 1) & ~((size_t(2) << 20) - 1);
    void* p = aligned_alloc(size_t(2) << 20, bytes ? bytes : (size_t(2) << 20));
    if (!p) throw std::bad_alloc();
    madvise(p, bytes, MADV_HUGEPAGE);
    return (T*)p;
  }
  void deallocate(T* p, size_t) { free(p); }
  template <typename U> bool operator==(const HugeAlloc<U>&) const { return true; }
  template <typename U> bool operator!=(const HugeAlloc<U>&) const { return false; }
};
using Forest = std::vector<UfElt, HugeAlloc<UfElt>>;
thread_local Forest g_forest;

void host_kruskal(const Edge12* e, size_t nE, size_t nV, float c, Forest& u) {
  u.resize(nV);
  for (size_t i = 0; i < nV; ++i) { u[i].rank = 0; u[i].size = 1; u[i].p = (int)i; u[i].thr = c; }
  UfElt* U = u.data();
  // (the prefetch walk is written out here on purpose: factored into a helper taking `const UfElt*` the same statements
  //  compiled into a loop that ran 120 ms instead of 84 ms on the 2 M-vertex mesh)
  for (size_t i = 0; i < nE; ++i) {
    if (i + 48 < nE) { __builtin_prefetch(U + e[i + 48].a); __builtin_prefetch(U + e[i + 48].b); }
    if (i + 8 < nE) { int y = e[i + 8].a; y = U[y].p; y = U[y].p; __builtin_prefetch(U + y); y = e[i + 8].b; y = U[y].p; y = U[y].p; __builtin_prefetch(U + y); }
    int a = uf_find_full(U, e[i].a), b = uf_find_full(U, e[i].b);
    if (a != b && e[i].w <= U[a].thr && e[i].w <= U[b].thr) { uf_join(U, a, b); a = uf_find_full(U, a); U[a].thr = e[i].w + (c / (float)U[a].size); }
  }
}
void host_small_merge(const Edge12* e, size_t nE, int min_verts, Forest& u) {
  UfElt* U = u.data();
  for (size_t j = 0; j < nE; ++j) {
    if (j + 48 < nE) { __builtin_prefetch(U + e[j + 48].a); __builtin_prefetch(U + e[j + 48].b); }
    const int a = uf_find_full(U, e[j].a), b = uf_find_full(U, e[j].b);
    if (a != b && (U[a].size < min_verts || U[b].size < min_verts)) uf_join(U, a, b);
  }
}

// ---- S5 on the device: speculative-window replay of Kruskal-with-threshold (segmentator.cpp:71-91) -----------------------
// One CTA keeps a window of up to 1024 pending edges in weight order (shared memory) and repeats rounds:
//   1. every pending edge resolves the roots of its ends (read-only find with path compression; the forest lives in global
//      memory, L2-resident) and registers itself on both components with atomicMin(owner[root], position);
//   2. an edge whose ends share a root is a no-op for good (components only merge) and retires;
//      a component whose EARLIEST pending edge is heavier than its threshold is frozen - a threshold only changes in a
//      merge, a merge needs w <= threshold, and every pending or future edge is at least as heavy - so every edge touching
//      it retires as rejected, in bulk;
//      an edge that is the earliest pending edge of BOTH its components sees exactly the forest the sequential loop would
//      show it, so it is decided now: it passed the two threshold tests above, so it joins (union by rank with the
//      reference's argument order and tie rule, threshold = w + c / size);
//      every other edge stays pending;
//   3. the window is compacted in order and refilled from the sorted stream.
// Merges decided in one round touch disjoint pairs of components, so they commute.  Identical forest (parents up to path
// compression, ranks, sizes, thresholds, root identities) to the sequential loop; what limits it is the dependency chain of
// merges into one growing component - one merge per component per round - see DESIGN.md §5 for the measured comparison
// with the host loop, which stays the default.
constexpr int kUfWindow = 1024;
__device__ __forceinline__ int uf_find_dev(UfElt* U, int x) {
  int y = x;
  for (;;) { const int p = U[y].p; if (p == y) break; y = p; }
  while (x != y) { const int n = U[x].p; if (n != y) U[x].p = y; x = n; }       // concurrent finds only ever write ancestors: benign
  return y;
}
__global__ void __launch_bounds__(kUfWindow, 1)
k_kruskal_window(const Edge12* __restrict__ e, unsigned nE, UfElt* U, int* owner, float c, unsigned long long* rounds_out) {
  __shared__ Edge12 s_e[2][kUfWindow];
  __shared__ unsigned s_warp[kUfWindow / 32];
  __shared__ unsigned s_total;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  unsigned n_pend = 0, next = 0, cur = 0;
  unsigned long long rounds = 0;
  for (;;) {
    const unsigned fill = min((unsigned)kUfWindow - n_pend, nE - next);
    if ((unsigned)t < fill) s_e[cur][n_pend + t] = e[next + t];
    n_pend += fill; next += fill;
    if (n_pend == 0) break;
    __syncthreads();
    ++rounds;
    Edge12 ed = {0.f, 0, 0};
    int ra = 0, rb = 0; bool cand = false;
    if ((unsigned)t < n_pend) {
      ed = s_e[cur][t];
      ra = uf_find_dev(U, ed.a); rb = uf_find_dev(U, ed.b);
      cand = ra != rb;
      if (cand) { atomicMin(&owner[ra], t); atomicMin(&owner[rb], t); }
    }
    __syncthreads();
    bool keep = false, merge = false;
    if (cand) {
      const int fa = owner[ra], fb = owner[rb];
      const float tha = U[ra].thr, thb = U[rb].thr;
      if (s_e[cur][fa].w > tha || s_e[cur][fb].w > thb) { /* a frozen component: rejected for good */ }
      else if (fa == t && fb == t) merge = ed.w <= tha && ed.w <= thb;      // the loop's own test (false for a NaN weight: rejected, retired)
      else keep = true;
    }
    __syncthreads();                                        // every read of the forest / owners precedes the writes below
    if (cand) { owner[ra] = 0x7FFFFFFF; owner[rb] = 0x7FFFFFFF; }
    if (merge) {                                            // universe::join(a, b) + the threshold update, segmentator.cpp:46-58,84-87
      const int rka = U[ra].rank, rkb = U[rb].rank;
      int root;
      if (rka > rkb) { U[rb].p = ra; U[ra].size += U[rb].size; root = ra; }
      else { U[ra].p = rb; U[rb].size += U[ra].size; if (rka == rkb) U[rb].rank = rkb + 1; root = rb; }
      U[root].thr = __fadd_rn(ed.w, __fdiv_rn(c, (float)U[root].size));
    }
    // stable compaction of the edges that stay pending
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
      unsigned v = s_warp[lane], inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned q = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += q; }
      s_warp[lane] = inc - v;
      if (lane == 31) s_total = inc;
    }
    __syncthreads();
    if (keep) s_e[cur ^ 1][s_warp[warp] + __popc(bal & ((1u << lane) - 1u))] = ed;
    n_pend = s_total;
    cur ^= 1;
    __syncthreads();
  }
  if (t == 0 && rounds_out) *rounds_out = rounds;
}
__global__ void k_uf_init(UfElt* U, int* owner, size_t nV, float c) {
  const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (v >= nV) return;
  UfElt u; u.rank = 0; u.p = (int)v; u.size = 1; u.thr = c;
  U[v] = u; owner[v] = 0x7FFFFFFF;
}
thread_local unsigned long long g_uf_rounds = 0;
// Kruskal pass on the device over the pruned, sorted, still-resident records; the forest comes back to the host for the
// small-segment pass and the labels (same structure as host_kruskal leaves).
int device_kruskal(const Edge12* dE, size_t nK, size_t nV, float c, Forest& u, cudaStream_t st) {
  u.resize(nV);
  g_uf_rounds = 0;
  if (!nV) return SCN_OK;
  DevBuf dU, dOwner, dRounds;
  if (dU.alloc(nV * sizeof(UfElt)) || dOwner.alloc(nV * 4) || dRounds.alloc(8)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc (device union-find)");
  k_uf_init<<<(unsigned)((nV + 255) / 256), 256, 0, st>>>(dU.as<UfElt>(), dOwner.as<int>(), nV, c);
  k_kruskal_window<<<1, kUfWindow, 0, st>>>(dE, (unsigned)nK, dU.as<UfElt>(), dOwner.as<int>(), c, dRounds.as<unsigned long long>());
  SCN_CUDA_TRY(cudaMemcpyAsync(u.data(), dU.p, nV * sizeof(UfElt), cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(&g_uf_rounds, dRounds.p, 8, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

// Device: drop provable no-op records (see k_pair_first), copy the survivors to pinned host memory.  Returns the
// pruned, still weight-sorted records in *out (pointer into a cached pinned buffer) and their count.
int prune_and_download(const Rec* dRec, const unsigned* dTri, const Edge12* dSrc, size_t nE, cudaStream_t st, const Edge12** out, size_t* n_out,
                       const Edge12** d_out = nullptr) {
  *out = nullptr; *n_out = 0; if (d_out) *d_out = nullptr;
  if (!nE) return SCN_OK;
  size_t cap = 1; while (cap < 2 * nE) cap <<= 1;
  DevBuf dK, dM, dKeep, dPos, dOut, dScr;
  if (dK.alloc(cap * 8) || dM.alloc(cap * 4) || dKeep.alloc(nE * 4) || dPos.alloc((nE + 1) * 4) || dOut.alloc(nE * 12) || dScr.alloc(scn::scan_scratch_elems(nE) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (replay pruning workspace)");
  SCN_CUDA_TRY(cudaMemsetAsync(dK.p, 0xFF, cap * 8, st));
  SCN_CUDA_TRY(cudaMemsetAsync(dM.p, 0xFF, cap * 4, st));
  const unsigned g = (unsigned)((nE + 255) / 256);
  k_pair_first<<<g, 256, 0, st>>>(dRec, dTri, dSrc, nE, dK.as<unsigned long long>(), dM.as<unsigned>(), (unsigned)(cap - 1));
  k_pair_keep<<<g, 256, 0, st>>>(dRec, dTri, dSrc, nE, dK.as<unsigned long long>(), dM.as<unsigned>(), (unsigned)(cap - 1), dKeep.as<unsigned>());
  scn::exclusive_scan_u32(dKeep.as<unsigned>(), dPos.as<unsigned>(), nE, dScr.as<unsigned>(), st);
  k_compact_edges<<<g, 256, 0, st>>>(dRec, dTri, dSrc, nE, dKeep.as<unsigned>(), dPos.as<unsigned>(), dOut.as<Edge12>());
  unsigned nk = 0;
  SCN_CUDA_TRY(cudaMemcpyAsync(&nk, dPos.as<unsigned>() + nE, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  void* h = g_pinned.get((size_t)nk * 12 + 16);
  if (!h) return scn::fail(SCN_ERR_CUDA, "cudaHostAlloc (%u records)", nk);
  SCN_CUDA_TRY(cudaMemcpyAsync(h, dOut.p, (size_t)nk * 12, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  SCN_CUDA_TRY(cudaGetLastError());
  *out = (const Edge12*)h; *n_out = nk; if (d_out) *d_out = dOut.as<Edge12>();
  return SCN_OK;
}

// Small-segment pass (segmentator.cpp:237-243) pre-filter.  After the Kruskal pass an edge whose ends already share a root,
// or whose two components both have >= segMinVerts vertices, can never act in the second pass (components only merge and
// sizes only grow), so only the few edges between a small component and a neighbour need the sequential replay.  The forest
// (parent, size) goes to the device, every vertex resolves its root, the still-resident pruned edge array is filtered and
// compacted in order, and the survivors come back.
__global__ void k_uf_roots(const int2* __restrict__ ps, size_t nV, int* __restrict__ root) {
  const size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (v >= nV) return;
  int y = (int)v;
  for (;;) { const int p = ps[y].x; if (p == y) break; y = p; }
  root[v] = y;
}
__global__ void k_small_keep(const Edge12* __restrict__ e, size_t nK, const int* __restrict__ root, const int2* __restrict__ ps, int min_verts,
                             unsigned* __restrict__ keep) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= nK) return;
  const int ra = root[e[j].a], rb = root[e[j].b];
  keep[j] = (ra != rb && (ps[ra].y < min_verts || ps[rb].y < min_verts)) ? 1u : 0u;
}
__global__ void k_compact12(const Edge12* __restrict__ e, size_t nK, const unsigned* __restrict__ keep, const unsigned* __restrict__ pos,
                            Edge12* __restrict__ out) {
  const size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j < nK && keep[j]) out[pos[j]] = e[j];
}
int filter_small_merge(const Edge12* dE, size_t nK, const Forest& u, int min_verts, cudaStream_t st, const Edge12** out, size_t* n_out) {
  const size_t nV = u.size();
  int2* hps = (int2*)g_pinned_in.get(nV * 8);
  if (!hps) return scn::fail(SCN_ERR_CUDA, "cudaHostAlloc (forest upload)");
  for (size_t v = 0; v < nV; ++v) hps[v] = make_int2(u[v].p, u[v].size);
  DevBuf dPs, dRoot, dKeep, dPos, dOut, dScr;
  if (dPs.alloc(nV * 8) || dRoot.alloc(nV * 4) || dKeep.alloc(nK * 4) || dPos.alloc((nK + 1) * 4) || dOut.alloc(nK * 12) || dScr.alloc(scn::scan_scratch_elems(nK) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (small-segment filter workspace)");
  SCN_CUDA_TRY(cudaMemcpyAsync(dPs.p, hps, nV * 8, cudaMemcpyHostToDevice, st));
  k_uf_roots<<<(unsigned)((nV + 255) / 256), 256, 0, st>>>(dPs.as<int2>(), nV, dRoot.as<int>());
  const unsigned g = (unsigned)((nK + 255) / 256);
  k_small_keep<<<g, 256, 0, st>>>(dE, nK, dRoot.as<int>(), dPs.as<int2>(), min_verts, dKeep.as<unsigned>());
  scn::exclusive_scan_u32(dKeep.as<unsigned>(), dPos.as<unsigned>(), nK, dScr.as<unsigned>(), st);
  k_compact12<<<g, 256, 0, st>>>(dE, nK, dKeep.as<unsigned>(), dPos.as<unsigned>(), dOut.as<Edge12>());
  unsigned n2 = 0;
  SCN_CUDA_TRY(cudaMemcpyAsync(&n2, dPos.as<unsigned>() + nK, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  void* h = g_pinned.get((size_t)n2 * 12 + 16);                 // the Kruskal pass is done with the previous contents
  if (!h) return scn::fail(SCN_ERR_CUDA, "cudaHostAlloc (%u records)", n2);
  SCN_CUDA_TRY(cudaMemcpyAsync(h, dOut.p, (size_t)n2 * 12, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  SCN_CUDA_TRY(cudaGetLastError());
  *out = (const Edge12*)h; *n_out = n2;
  return SCN_OK;
}
constexpr size_t kSmallFilterMin = 200000;      // below this the sequential pass is cheaper than the round trip

struct Timer {
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  float lap() { auto t1 = std::chrono::steady_clock::now(); float ms = std::chrono::duration<float, std::milli>(t1 - t0).count(); t0 = t1; return ms; }
};

int segment_impl(const float* xyz, uint64_t nV, const uint32_t* tri, uint64_t nF, float kthr, int32_t min_verts,
                 int32_t* seg_out, int flags, Edge12* edges_presort, Edge12* edges_sorted, float* normals_out,
                 int32_t* roots_after_kruskal) {
  if ((!xyz && nV) || (!tri && nF) || !seg_out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (nV > 0x7FFFFFFFull || 3 * nF > 0x7FFFFFFFull) return scn::fail(SCN_ERR_ARG, "mesh too large for 32-bit ids");
  for (int i = 0; i < 8; ++i) g_timings[i] = 0;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return scn::fail(SCN_ERR_CUDA, "no CUDA device: the Segmentator kernels have no CPU fallback");
  Timer total, lapt;
  g_arena.reset();
  const size_t nE = 3 * nF;
  g_arena.reserve(104 * nE + 80 * (size_t)nV + (size_t(32) << 20));      // upper bound of every buffer below incl. sort + pruning
  // Inputs are usually pageable: a plain cudaMemcpy of the 72 MB of a 2 M-vertex mesh took ~60 ms.  A few host threads copy
  // slices into a cached pinned buffer (checking the indices on the way), then one DMA per array moves them.
  const size_t xyz_bytes = nV * 12, tri_bytes = nF * 12;
  char* stage = (xyz_bytes + tri_bytes >= (size_t(4) << 20)) ? (char*)g_pinned_in.get(xyz_bytes + tri_bytes) : nullptr;
  std::atomic<uint64_t> bad{~0ull};
  if (stage) {
    const unsigned nt = std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
    auto work = [&](unsigned t) {
      const size_t x0 = xyz_bytes * t / nt, x1 = xyz_bytes * (t + 1) / nt;
      memcpy(stage + x0, (const char*)xyz + x0, x1 - x0);
      const size_t i0 = 3 * nF * t / nt, i1 = 3 * nF * (t + 1) / nt;
      uint32_t* dst = (uint32_t*)(stage + xyz_bytes);
      uint32_t mx = 0;
      for (size_t i = i0; i < i1; ++i) { const uint32_t v = tri[i]; dst[i] = v; mx = v > mx ? v : mx; }
      if (mx >= nV) for (size_t i = i0; i < i1; ++i) if (tri[i] >= nV) { uint64_t cur = bad.load(); while (i < cur && !bad.compare_exchange_weak(cur, i)) {} break; }
    };
    std::vector<std::thread> pool;
    for (unsigned t = 1; t < nt; ++t) pool.emplace_back(work, t);
    work(0);
    for (auto& th : pool) th.join();
  } else {
    for (uint64_t i = 0; i < 3 * nF; ++i) if (tri[i] >= nV) { bad = i; break; }
  }
  if (bad.load() != ~0ull) { const uint64_t i = bad.load(); return scn::fail(SCN_ERR_FORMAT, "face %llu references vertex %u >= %llu", (unsigned long long)(i / 3), tri[i], (unsigned long long)nV); }
  const void* src_xyz = stage ? (const void*)stage : (const void*)xyz;
  const void* src_tri = stage ? (const void*)(stage + xyz_bytes) : (const void*)tri;
  cudaStream_t st = nullptr;
  DevBuf dXyz, dTri, dFn, dDeg, dOff, dCur, dCsr, dNrm, dRec, dE12, dScr;
  if (dXyz.alloc(nV * 12) || dTri.alloc(nF * 12) || dFn.alloc(nF * 16) || dDeg.alloc((nV + 1) * 4) || dOff.alloc((nV + 2) * 4) ||
      dCur.alloc((nV + 1) * 4) || dCsr.alloc(nE * 4) || dNrm.alloc(nV * 12) || dRec.alloc(nE * 8) || dE12.alloc(nE * 12) ||
      dScr.alloc(scn::scan_scratch_elems(nV + 1) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (segmentator workspace)");
  SCN_CUDA_TRY(cudaMemcpyAsync(dXyz.p, src_xyz, nV * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(dTri.p, src_tri, nF * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemsetAsync(dDeg.p, 0, (nV + 1) * 4, st));
  SCN_CUDA_TRY(cudaMemsetAsync(dCur.p, 0, (nV + 1) * 4, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  g_timings[0] = lapt.lap();
  const unsigned B = 256;
  if (nF) {
    k_face_normals<<<(unsigned)((nF + B - 1) / B), B, 0, st>>>(dXyz.as<float>(), dTri.as<unsigned>(), nF, nV, dFn.as<float4>(), dDeg.as<unsigned>());
  }
  scn::exclusive_scan_u32(dDeg.as<unsigned>(), dOff.as<unsigned>(), nV, dScr.as<unsigned>(), st);
  if (nF) k_fill_csr<<<(unsigned)((nE + B - 1) / B), B, 0, st>>>(dTri.as<unsigned>(), nF, dOff.as<unsigned>(), dCur.as<unsigned>(), dCsr.as<unsigned>());
  if (nV) k_vertex_normals<<<(unsigned)((nV + 127) / 128), 128, 0, st>>>(dOff.as<unsigned>(), dCsr.as<unsigned>(), dFn.as<float4>(), nV, dNrm.as<float>());
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  g_timings[1] = lapt.lap();
  if (nE) k_edge_weights<<<(unsigned)((nE + B - 1) / B), B, 0, st>>>(dXyz.as<float>(), dTri.as<unsigned>(), dNrm.as<float>(), nE, dRec.as<Rec>());
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  g_timings[2] = lapt.lap();
  if (normals_out && nV) SCN_CUDA_TRY(cudaMemcpy(normals_out, dNrm.p, nV * 12, cudaMemcpyDeviceToHost));
  if (edges_presort && nE) {
    k_gather_edges<<<(unsigned)((nE + B - 1) / B), B, 0, st>>>(dRec.as<Rec>(), dTri.as<unsigned>(), nE, dE12.as<Edge12>());
    SCN_CUDA_TRY(cudaMemcpy(edges_presort, dE12.p, nE * 12, cudaMemcpyDeviceToHost));
    lapt.lap();
  }
  int rc = device_introsort(dRec.as<Rec>(), nE, st);
  if (rc) return rc;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  g_timings[3] = lapt.lap();
  if (edges_sorted && nE) {                            // full sorted array: parity tests only
    k_gather_edges<<<(unsigned)((nE + B - 1) / B), B, 0, st>>>(dRec.as<Rec>(), dTri.as<unsigned>(), nE, dE12.as<Edge12>());
    SCN_CUDA_TRY(cudaMemcpy(edges_sorted, dE12.p, nE * 12, cudaMemcpyDeviceToHost));
    lapt.lap();
  }
  const Edge12* hE = nullptr; const Edge12* dE = nullptr; size_t nK = 0;
  rc = prune_and_download(dRec.as<Rec>(), dTri.as<unsigned>(), nullptr, nE, st, &hE, &nK, &dE);
  if (rc) return rc;
  g_timings[6] = lapt.lap();
  Forest& u = g_forest;
  if (flags & SCN_SEG_DEVICE_UNIONFIND) { rc = device_kruskal(dE, nK, nV, kthr, u, st); if (rc) return rc; }
  else host_kruskal(hE, nK, nV, kthr, u);
  g_timings[4] = lapt.lap();
  if (roots_after_kruskal) for (size_t q = 0; q < nV; ++q) { int y = (int)q; while (y != u[y].p) y = u[y].p; roots_after_kruskal[q] = y; }
  lapt.lap();
  if (nK >= kSmallFilterMin) { rc = filter_small_merge(dE, nK, u, min_verts, st, &hE, &nK); if (rc) return rc; }
  host_small_merge(hE, nK, min_verts, u);
  g_timings[5] = lapt.lap();
  for (size_t q = 0; q < nV; ++q) seg_out[q] = uf_find(u.data(), (int)q);
  g_timings[6] += lapt.lap();
  g_timings[7] = total.lap();
  return SCN_OK;
}

}  // namespace

extern "C" {

int scn_segment_mesh(const float* xyz, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces, float k_thresh,
                     int32_t seg_min_verts, int32_t* seg_out, int flags) {
  return segment_impl(xyz, n_verts, tri, n_faces, k_thresh, seg_min_verts, seg_out, flags, nullptr, nullptr, nullptr, nullptr);
}

int scn_segment_mesh_debug(const float* xyz, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces, float k_thresh,
                           int32_t seg_min_verts, int32_t* seg_out, int flags, void* edges_presort, void* edges_sorted,
                           float* vertex_normals, int32_t* roots_after_kruskal) {
  return segment_impl(xyz, n_verts, tri, n_faces, k_thresh, seg_min_verts, seg_out, flags, (Edge12*)edges_presort,
                      (Edge12*)edges_sorted, vertex_normals, roots_after_kruskal);
}

int scn_segment_graph(int32_t n_verts, int64_t n_edges, void* edges, float c, int32_t* roots_out, int32_t* sizes_out, int flags) {
  if (n_verts < 0 || n_edges < 0 || (!edges && n_edges)) return scn::fail(SCN_ERR_ARG, "bad argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return scn::fail(SCN_ERR_CUDA, "no CUDA device");
  Edge12* he = (Edge12*)edges;
  for (int64_t i = 0; i < n_edges; ++i)
    if (he[i].a < 0 || he[i].a >= n_verts || he[i].b < 0 || he[i].b >= n_verts) return scn::fail(SCN_ERR_ARG, "edge %lld endpoint out of range", (long long)i);
  const size_t nE = (size_t)n_edges;
  g_arena.reset();
  g_arena.reserve(96 * nE + (size_t(32) << 20));
  DevBuf dSrc, dDst, dRec;
  if (dSrc.alloc(nE * 12) || dDst.alloc(nE * 12) || dRec.alloc(nE * 8)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc");
  cudaStream_t st = nullptr;
  if (nE) {
    SCN_CUDA_TRY(cudaMemcpyAsync(dSrc.p, he, nE * 12, cudaMemcpyHostToDevice, st));
    k_rec_from_edges12<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(dSrc.as<Edge12>(), nE, dRec.as<Rec>());
  }
  int rc = device_introsort(dRec.as<Rec>(), nE, st, (flags >> 8) & 0xFF);
  if (rc) return rc;
  if (nE) {
    k_gather_edges12<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(dRec.as<Rec>(), dSrc.as<Edge12>(), nE, dDst.as<Edge12>());
    SCN_CUDA_TRY(cudaMemcpy(he, dDst.p, nE * 12, cudaMemcpyDeviceToHost));
  }
  SCN_CUDA_TRY(cudaGetLastError());
  const Edge12* hK = nullptr; size_t nK = 0;
  rc = prune_and_download(dRec.as<Rec>(), nullptr, dSrc.as<Edge12>(), nE, st, &hK, &nK);
  if (rc) return rc;
  Forest& u = g_forest;
  host_kruskal(hK, nK, (size_t)n_verts, c, u);
  for (int v = 0; v < n_verts; ++v) {
    int y = v; while (y != u[y].p) y = u[y].p;
    if (roots_out) roots_out[v] = y;
    if (sizes_out) sizes_out[v] = u[y].size;
  }
  return SCN_OK;
}

int scn_segment_last_timings(float* ms8) {
  if (!ms8) return scn::fail(SCN_ERR_ARG, "null argument");
  for (int i = 0; i < 8; ++i) ms8[i] = g_timings[i];
  return (int)g_sort_launches;
}

/* rounds taken by the device union-find replay of the last scn_segment_mesh call on this thread (0 = host loop was used) */
uint64_t scn_segment_last_uf_rounds(void) {
  return g_uf_rounds;
}

}  // extern "C"
