// Internal: the device-resident mesh and the mesh-cleaning steps of meshclean.cu (DESIGN.md §6f), shared with the decimation
// in meshsimplify.cu (§6g), which runs the same duplicate-face and compaction code and then the script's clean filters on the
// mesh it already holds in device memory.  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

#include "radix_sort.cuh"
#include "scn_common.h"

namespace scn::mc {

struct Mesh {                         // the current mesh, in device memory
  DBuf xyz, rgb, tri;
  unsigned nV = 0, nF = 0;
  bool has_rgb = false;
};

inline float ms_between(const EventPtr& a, const EventPtr& b) { float ms = 0.f; return cudaEventElapsedTime(&ms, a.get(), b.get()) == cudaSuccess ? ms : 0.f; }
int read_u32(const unsigned* d, unsigned* h, size_t n, cudaStream_t st);

// allocates the pinned read-back words, the mesh (rgb if given) and the error word, records `start`, uploads the mesh and
// clears the error word
int upload_mesh(Mesh& m, const float* xyz, const uint8_t* rgb, uint64_t nV, const uint32_t* tri, uint64_t nF, PinnedPtr<unsigned>& h_small,
                DBuf& err, cudaEvent_t start, cudaStream_t st);
// copies the mesh into malloc'd arrays (colours if the mesh has them and `rgb` is given), records `done` after the copies, waits
// for them and only then hands the arrays to the caller; the error texts name `who`
int download_mesh(const Mesh& m, float** xyz, uint8_t** rgb, uint32_t** tri, cudaEvent_t done, cudaStream_t st, const char* who);

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
                    unsigned* d_err, unsigned* h_small, const EventPtr* ev);

}  // namespace scn::mc
