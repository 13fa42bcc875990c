// Internal: the device-resident mesh and the mesh-cleaning steps of meshclean.cu (DESIGN.md §6f), shared with the decimation
// in meshsimplify.cu (§6g), which runs the same duplicate-face and compaction code and then the script's clean filters on the
// mesh it already holds in device memory.  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>

#include "radix_sort.cuh"
#include "scn_common.h"

namespace scn::mc {

struct DBuf {                      // cudaMalloc with scope lifetime
  void* p = nullptr;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { if (p) cudaFree(p); }
  template <typename T> T* as() const { return (T*)p; }
  bool alloc(size_t bytes) { if (p) { cudaFree(p); p = nullptr; } return cudaMalloc(&p, bytes ? bytes : 4) == cudaSuccess; }
  void swap(DBuf& o) { std::swap(p, o.p); }
};
#define MC_ALLOC(buf, bytes) do { if (!(buf).alloc(bytes)) { cudaGetLastError(); return scn::fail(SCN_ERR_CUDA, "cudaMalloc(%zu) failed (%s:%d)", (size_t)(bytes), __FILE__, __LINE__); } } while (0)

struct Mesh {                         // the current mesh, in device memory
  DBuf xyz, rgb, tri;
  unsigned nV = 0, nF = 0;
  bool has_rgb = false;
};

struct Scratch {                      // radix-sort pairs and scan scratch, grown on demand
  DBuf k0, v0, k1, v1, hist, scr;
  size_t cap_pairs = 0, cap_scan = 0;
  int ensure(size_t n, size_t scan_n) {          // sorts of n pairs, scans of up to scan_n elements
    if (n > cap_pairs) {
      MC_ALLOC(k0, n * 4); MC_ALLOC(v0, n * 4); MC_ALLOC(k1, n * 4); MC_ALLOC(v1, n * 4); MC_ALLOC(hist, rs_hist_elems(n) * 4);
      cap_pairs = n;
    }
    const size_t need = scn::scan_scratch_elems(std::max(rs_hist_elems(cap_pairs), scan_n));
    if (need > cap_scan) { MC_ALLOC(scr, need * 4); cap_scan = need; }
    return SCN_OK;
  }
};

struct Stream {
  cudaStream_t s = nullptr;
  cudaEvent_t ev[8] = {};
  ~Stream() { for (auto e : ev) if (e) cudaEventDestroy(e); if (s) cudaStreamDestroy(s); }
};

inline unsigned grid_for(size_t n) { return (unsigned)((n + 255) / 256); }
inline float ms_between(cudaEvent_t a, cudaEvent_t b) { float ms = 0.f; return cudaEventElapsedTime(&ms, a, b) == cudaSuccess ? ms : 0.f; }
int read_u32(const unsigned* d, unsigned* h, size_t n, cudaStream_t st);
// sorts `vals` stably by the keys staged in s.k0, leaving the result in (k0,v0) or (k1,v1); returns the value array
unsigned* sort_pass(Scratch& s, unsigned*& vals, size_t n, int bits, cudaStream_t st);

// otri[pos[f]] = tri[f] for the faces with keep[f] (pos = exclusive scan of keep)
__global__ void k_compact_faces(const unsigned* __restrict__ tri, const unsigned* __restrict__ keep, const unsigned* __restrict__ pos,
                                unsigned nF, unsigned* __restrict__ otri);
// removeDuplicateFaces (§6f step 2): rep.duplicate_faces is set
int step_dedup(Mesh& m, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st);
// drops the vertices no face references; the survivors keep their order (ascending index), faces are renumbered
int drop_unreferenced(Mesh& m, Scratch& s, cudaStream_t st, unsigned* h_small);
// the three clean.mlx steps in order as `params` selects them (scn_mesh_clean after its upload); ev[0] is recorded by the caller
// before, ev[1..3] here after each step; the step counters and merge/dedup/pieces ms go into rep
int run_clean_steps(Mesh& m, const scn_mesh_clean_params& params, Scratch& s, scn_mesh_clean_report_t& rep, cudaStream_t st,
                    unsigned* d_err, unsigned* h_small, const cudaEvent_t* ev);

}  // namespace scn::mc
