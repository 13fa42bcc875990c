// Stable LSD radix sort of (uint32 key, uint32 value) pairs (hand-written: per-tile digit histograms, one device-wide scan,
// rank-preserving scatter), 8 bits per pass, and the scratch its callers sort in.  Shared by segs.cu, meshclean.cu and
// meshsimplify.cu.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>

#include "scan.cuh"
#include "scn_common.h"

namespace scn {

constexpr int kRsThreads = 256, kRsItems = 8, kRsTile = kRsThreads * kRsItems;

static __global__ void __launch_bounds__(kRsThreads)
k_rs_hist(const unsigned* __restrict__ keys, size_t n, int shift, unsigned* __restrict__ hist, unsigned nblk) {
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const size_t base = (size_t)blockIdx.x * kRsTile;
#pragma unroll
  for (int r = 0; r < kRsItems; ++r) {
    const size_t i = base + (size_t)r * kRsThreads + threadIdx.x;
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];       // digit-major: one scan yields global offsets
}

// Round r of a tile handles elements base + r*256 + tid, so (round, warp, lane) order == input order: ranks computed as
// "tile offset of the digit + elements of earlier rounds/warps + earlier lanes with the same digit" keep the sort stable.
static __global__ void __launch_bounds__(kRsThreads)
k_rs_scatter(const unsigned* __restrict__ kin, const unsigned* __restrict__ vin, unsigned* __restrict__ kout,
             unsigned* __restrict__ vout, size_t n, int shift, const unsigned* __restrict__ offs, unsigned nblk) {
  __shared__ unsigned s_base[256];
  __shared__ unsigned s_wcnt[kRsThreads / 32][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  s_base[threadIdx.x] = offs[(size_t)threadIdx.x * nblk + blockIdx.x];
  const size_t base = (size_t)blockIdx.x * kRsTile;
  for (int r = 0; r < kRsItems; ++r) {
#pragma unroll
    for (int w = 0; w < kRsThreads / 32; ++w) s_wcnt[w][threadIdx.x] = 0;
    __syncthreads();
    const size_t i = base + (size_t)r * kRsThreads + threadIdx.x;
    const bool valid = i < n;
    unsigned k = 0, v = 0, d = 256u;
    if (valid) { k = kin[i]; v = vin[i]; d = (k >> shift) & 255u; }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) s_wcnt[warp][d] = __popc(peers);
    __syncthreads();
    {
      unsigned run = s_base[threadIdx.x];
#pragma unroll
      for (int w = 0; w < kRsThreads / 32; ++w) { const unsigned c = s_wcnt[w][threadIdx.x]; s_wcnt[w][threadIdx.x] = run; run += c; }
      s_base[threadIdx.x] = run;
    }
    __syncthreads();
    if (valid) { const unsigned pos = s_wcnt[warp][d] + rank; kout[pos] = k; vout[pos] = v; }
    __syncthreads();
  }
}

// Sorts (keys, vals) by the low `bits` bits of key, stable.  Result lands in (k0, v0) or (k1, v1): returns which (0/1).
inline int radix_sort_pairs(unsigned* k0, unsigned* v0, unsigned* k1, unsigned* v1, size_t n, int bits, unsigned* hist, unsigned* scratch,
                            cudaStream_t st) {
  const unsigned nblk = (unsigned)((n + kRsTile - 1) / kRsTile);
  int cur = 0;
  for (int shift = 0; shift < bits; shift += 8) {
    unsigned* ki = cur ? k1 : k0; unsigned* vi = cur ? v1 : v0; unsigned* ko = cur ? k0 : k1; unsigned* vo = cur ? v0 : v1;
    k_rs_hist<<<nblk, kRsThreads, 0, st>>>(ki, n, shift, hist, nblk);
    exclusive_scan_u32(hist, hist, (size_t)256 * nblk, scratch, st);
    k_rs_scatter<<<nblk, kRsThreads, 0, st>>>(ki, vi, ko, vo, n, shift, hist, nblk);
    cur ^= 1;
  }
  return cur;
}
inline size_t rs_hist_elems(size_t n) { return (size_t)256 * ((n + kRsTile - 1) / kRsTile) + 1; }
inline int bits_for(unsigned maxv) { int b = 1; while (b < 32 && (maxv >> b)) ++b; return b; }

static __global__ void k_iota(unsigned* v, size_t n) { const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; if (i < n) v[i] = (unsigned)i; }

struct Scratch {                      // radix-sort pairs and scan scratch, grown on demand
  DBuf k0, v0, k1, v1, hist, scr;
  size_t cap_pairs = 0, cap_scan = 0;
  int ensure(size_t n, size_t scan_n) {          // sorts of n pairs, scans of up to scan_n elements
    if (n > cap_pairs) {
      SCN_ALLOC(k0, n * 4); SCN_ALLOC(v0, n * 4); SCN_ALLOC(k1, n * 4); SCN_ALLOC(v1, n * 4); SCN_ALLOC(hist, rs_hist_elems(n) * 4);
      cap_pairs = n;
    }
    const size_t need = scan_scratch_elems(std::max(rs_hist_elems(cap_pairs), scan_n));
    if (need > cap_scan) { SCN_ALLOC(scr, need * 4); cap_scan = need; }
    return SCN_OK;
  }
};

// sorts `vals` (initially any permutation) stably by the keys staged in s.k0, leaving the result in (k0,v0) or (k1,v1);
// returns the value array
inline unsigned* sort_pass(Scratch& s, unsigned*& vals, size_t n, int bits, cudaStream_t st) {
  unsigned* k0 = s.k0.as<unsigned>(); unsigned* k1 = s.k1.as<unsigned>();
  unsigned* v0 = s.v0.as<unsigned>(); unsigned* v1 = s.v1.as<unsigned>();
  if (vals != v0) { cudaMemcpyAsync(v0, vals, n * 4, cudaMemcpyDeviceToDevice, st); }
  const int w = radix_sort_pairs(k0, v0, k1, v1, n, bits, s.hist.as<unsigned>(), s.scr.as<unsigned>(), st);
  vals = w ? v1 : v0;
  return vals;
}

}  // namespace scn
