// Counters and clocks of k_alloc's walk.  scripts/probes/alloc_walk_probe.py compiles a private copy of csrc/tsdf.cu with
// -DSCN_ALLOC_PROBE=1 (counters) or =2 (clock64 per phase; the counters' shared-memory atomics would distort the clocks)
// and -I to this directory; the shipped library never includes this file.
//
// Every hook accumulates into per-CTA shared-memory counters, added to g_alloc_probe by ap_end().  "Warp" below always
// means the lanes that execute the hook together (__activemask()): that is what the scheduler issues for.
#pragma once
#include <cuda_runtime.h>

enum AllocProbeCounter {
  AP_WARP_STEPS,        // note_cell executions, per converged group of lanes
  AP_WARP_STEPS_MISS,   // ... of which at least one lane left the fast path (key present, frame flag set)
  AP_LANE_STEPS,        // note_cell executions, per lane
  AP_LANE_MISS,         // ... that left the fast path
  AP_MISS_FLAG,         // lane outcome: key found present, frame flag clear -> flag set
  AP_MISS_CLAIM,        // lane outcome: slot claimed (CAS won) -> flag set
  AP_MISS_GLOBAL,       // lane outcome: 8 occupied slots in a row -> global table
  AP_COLLIDE,           // slot advances (slot held by another key)
  AP_FLAG_LANES,        // lanes that set a frame flag
  AP_FLAG_ADDRS,        // distinct slots among them, per converged group
  AP_WARP_FRAMES,       // (warp, frame) pairs with at least one walking lane
  AP_WARP_MAX_STEPS,    // sum over them of the largest lane step count
  AP_LANE_FRAMES,       // (lane, frame) pairs that walked
  AP_KEYS,              // occupied map slots at the flush
  AP_TOUCH,             // touch_block calls
  AP_CTAS,
  AP_HEAD_GROUPS,       // converged groups of lanes at the head of the group's frame j: AP_HEAD_GROUPS + j, j < 4
  AP_CLK_PROLOGUE = AP_HEAD_GROUPS + 4,
                        // clock64 ticks of lane 0 of every warp: map clear and frame staging
  AP_CLK_SETUP,         // frame head up to the first cell
  AP_CLK_WALK,          // the walk, up to the reconvergence at the next frame head
  AP_CLK_BARRIER,       // waiting for the CTA's other warps before the flush
  AP_CLK_FLUSH,
  AP_N
};

__device__ unsigned long long g_alloc_probe[AP_N];

__device__ __forceinline__ unsigned* ap_cta() { __shared__ unsigned s[AP_N]; return s; }
__device__ __forceinline__ unsigned& ap_my_steps() { __shared__ unsigned s[256]; return s[threadIdx.x]; }
__device__ __forceinline__ long long& ap_warp_clock() { __shared__ long long s[8]; return s[threadIdx.x >> 5]; }
__device__ __forceinline__ bool ap_leader(unsigned act) { return (int)(threadIdx.x & 31) == __ffs(act) - 1; }

#if SCN_ALLOC_PROBE == 1
__device__ __forceinline__ void ap_count(int c, unsigned n = 1) { atomicAdd(&ap_cta()[c], n); }
__device__ __forceinline__ void ap_mark(int) {}
#else
__device__ __forceinline__ void ap_count(int, unsigned = 1) {}
// closes the phase that was running (`done`) for this warp
__device__ __forceinline__ void ap_mark(int done) {
  if (threadIdx.x & 31) return;
  const long long now = clock64();
  atomicAdd(&ap_cta()[done], (unsigned)(now - ap_warp_clock()));
  ap_warp_clock() = now;
}
#endif

// before the kernel's first barrier
__device__ __forceinline__ void ap_begin() {
  if (threadIdx.x < AP_N) ap_cta()[threadIdx.x] = 0;
  ap_my_steps() = 0;
  if (!(threadIdx.x & 31)) ap_warp_clock() = clock64();
}

// one note_cell execution; hit = fast path
__device__ __forceinline__ void ap_step(bool hit) {
#if SCN_ALLOC_PROBE == 1
  const unsigned act = __activemask(), miss = __ballot_sync(act, !hit);
  ap_my_steps()++;
  if (ap_leader(act)) {
    ap_count(AP_WARP_STEPS); ap_count(AP_LANE_STEPS, __popc(act));
    if (miss) { ap_count(AP_WARP_STEPS_MISS); ap_count(AP_LANE_MISS, __popc(miss)); }
  }
#endif
}

// a lane sets its frame's flag in map slot h (outcome = AP_MISS_FLAG or AP_MISS_CLAIM)
__device__ __forceinline__ void ap_flag(unsigned h, int outcome) {
#if SCN_ALLOC_PROBE == 1
  const unsigned act = __activemask(), peers = __match_any_sync(act, h);
  ap_count(outcome); ap_count(AP_FLAG_LANES);
  if (ap_leader(peers)) ap_count(AP_FLAG_ADDRS);
#endif
}

// closes a frame's walk for the warp: at the head of the group's frame j (j = 0: nothing walked yet) and, with j < 0, after the last one
__device__ __forceinline__ void ap_frame(int j) {
#if SCN_ALLOC_PROBE == 1
  const unsigned act = __activemask(), s = ap_my_steps();
  ap_my_steps() = 0;
  const unsigned mx = __reduce_max_sync(act, s), walked = __ballot_sync(act, s != 0);
  if (ap_leader(act)) {
    if (j >= 0) ap_count(AP_HEAD_GROUPS + j);
    if (mx) { ap_count(AP_WARP_FRAMES); ap_count(AP_WARP_MAX_STEPS, mx); ap_count(AP_LANE_FRAMES, __popc(walked)); }
  }
#else
  ap_mark(j == 0 ? AP_CLK_PROLOGUE : AP_CLK_WALK);
#endif
}

// after the flush
__device__ __forceinline__ void ap_end() {
  ap_mark(AP_CLK_FLUSH);
  __syncthreads();
  if (threadIdx.x == 0) ap_cta()[AP_CTAS] = 1;
  __syncthreads();
  if (threadIdx.x < AP_N && ap_cta()[threadIdx.x]) atomicAdd(&g_alloc_probe[threadIdx.x], (unsigned long long)ap_cta()[threadIdx.x]);
}

// copies the counters out (n <= AP_N) and zeroes them
extern "C" int scn_alloc_probe_read(unsigned long long* out, int n) {
  unsigned long long h[AP_N] = {}, z[AP_N] = {};
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(h, g_alloc_probe, sizeof(h)) != cudaSuccess ||
      cudaMemcpyToSymbol(g_alloc_probe, z, sizeof(z)) != cudaSuccess) return -1;
  for (int i = 0; i < n && i < AP_N; ++i) out[i] = h[i];
  return AP_N;
}
