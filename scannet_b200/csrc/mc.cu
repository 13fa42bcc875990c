// Marching-cubes surface extraction from the hashed TSDF volume (SURVEY.md §8(f)1; stage contract
// `<id>.sens -> <id>_vh.ply`, /root/reference/Server/config/scan_stages.json:33-37).  The reference does this
// inside the external DepthSensing/FriedLiver binaries (no source in the tree), so the spec is this repo's own
// (DESIGN.md §6) and parity is against oracle/tsdf_oracle.c.
//
// Spec.  Voxel v is *usable* iff weight>0 and |sdf| <= mc_thresh_factor*voxel_size (s_SDFMarchingCubeThreshFactor,
// zParametersScanNet.txt:48).  Cube at voxel g has corners g+(c&1,(c>>1)&1,(c>>2)&1), c=0..7, and is valid iff all 8
// are usable; corner c is inside iff sdf<0.  Lattice edge (g,a) carries a vertex iff both ends are usable and exactly
// one is inside: t = s0/(s0-s1), position ((g_a + t)*vs on axis a, g*vs elsewhere), colour u8(fma(t, c1-c0, c0)+0.5).
// Triangulation table (256 cases, generated at start-up, identical construction in the oracle): on each cube face
// (corners counter-clockwise seen from outside) every maximal run of inside corners contributes one directed segment
// from the edge entering the run to the edge leaving it (ambiguous faces separate the inside corners); the segments
// chain into closed loops; each loop, started at its lowest edge id, is fanned (v0,vi,vi+1).  Normals point to sdf>0.
// Order: blocks by packed key, voxels by lx+8ly+64lz, edges by axis, triangles by table order; vertices no triangle
// references are dropped, order preserved.  Output is therefore deterministic although heap indices are not.
#include <algorithm>
#include <numeric>
#include <vector>

#include "scan.cuh"
#include "tsdf_internal.cuh"

using namespace scn_tsdf_detail;

namespace {

struct McTable { uint8_t ntri[256]; uint8_t tri[256][36]; };

int mc_edge_id(int c0, int c1) {
  const int d = c0 ^ c1, a = d == 1 ? 0 : (d == 2 ? 1 : 2), lo = c0 & ~d;
  const int x = lo & 1, y = (lo >> 1) & 1, z = (lo >> 2) & 1;
  const int u = a == 0 ? y : x, v = a == 2 ? y : z;
  return a * 4 + (u | (v << 1));
}

void build_mc_table(McTable& T) {
  memset(&T, 0, sizeof(T));
  for (int cs = 0; cs < 256; ++cs) {
    int next[12];
    for (int& n : next) n = -1;
    for (int a = 0; a < 3; ++a) for (int s = 0; s < 2; ++s) {
      const int b = (a + 1) % 3, c = (a + 2) % 3;
      auto mk = [&](int vb, int vc) { int off[3]; off[a] = s; off[b] = vb; off[c] = vc; return off[0] | (off[1] << 1) | (off[2] << 2); };
      int p[4];
      if (s == 1) { p[0] = mk(0, 0); p[1] = mk(1, 0); p[2] = mk(1, 1); p[3] = mk(0, 1); }
      else        { p[0] = mk(0, 0); p[1] = mk(0, 1); p[2] = mk(1, 1); p[3] = mk(1, 0); }
      bool in[4];
      for (int k = 0; k < 4; ++k) in[k] = (cs >> p[k]) & 1;
      for (int k = 0; k < 4; ++k) if (!in[(k + 3) & 3] && in[k]) {
        int m = k;
        while (in[(m + 1) & 3]) m = (m + 1) & 3;
        const int E = mc_edge_id(p[(k + 3) & 3], p[k]), X = mc_edge_id(p[m], p[(m + 1) & 3]);
        next[E] = X;
      }
    }
    bool seen[12] = {false};
    int nt = 0;
    for (int e0 = 0; e0 < 12; ++e0) if (next[e0] >= 0 && !seen[e0]) {
      int loop[12], n = 0;
      for (int e = e0; !seen[e]; e = next[e]) { seen[e] = true; loop[n++] = e; }
      for (int i = 1; i + 1 < n; ++i) { T.tri[cs][3 * nt] = (uint8_t)loop[0]; T.tri[cs][3 * nt + 1] = (uint8_t)loop[i]; T.tri[cs][3 * nt + 2] = (uint8_t)loop[i + 1]; ++nt; }
    }
    T.ntri[cs] = (uint8_t)nt;
  }
}

constexpr int H9 = 9 * 9 * 9;

struct McCtx {
  Tables tb; const unsigned* order; const unsigned* inv_order; unsigned n_blocks; float thr, vs;
};

// loads the 9^3 halo (own block + the +1 faces/edges/corner from up to 7 neighbours) of sorted block j
__device__ __forceinline__ void load_halo(const McCtx& c, unsigned j, float* s_sdf, unsigned* s_cw, int* s_nb, int* bxyz) {
  const unsigned heap_idx = c.order[j];
  int bx, by, bz;
  unpack_key(c.tb.block_keys[heap_idx], bx, by, bz);
  if (threadIdx.x < 8) {
    const int dx = threadIdx.x & 1, dy = (threadIdx.x >> 1) & 1, dz = threadIdx.x >> 2;
    s_nb[threadIdx.x] = threadIdx.x == 0 ? (int)heap_idx : lookup_block(c.tb, bx + dx, by + dy, bz + dz);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < H9; i += blockDim.x) {
    const int x = i % 9, y = (i / 9) % 9, z = i / 81;
    const int nb = s_nb[(x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2)];
    float sd = 0.f; unsigned cw = 0u;
    if (nb >= 0) { const uint2 v = c.tb.heap[(size_t)nb * 512 + ((x & 7) | ((y & 7) << 3) | ((z & 7) << 6))]; sd = __uint_as_float(v.x); cw = v.y; }
    s_sdf[i] = sd; s_cw[i] = cw;
  }
  __syncthreads();
  bxyz[0] = bx; bxyz[1] = by; bxyz[2] = bz;
}
__device__ __forceinline__ bool usable(float sd, unsigned cw, float thr) { return (cw >> 24) != 0u && fabsf(sd) <= thr; }

// pass A: per voxel, which of its 3 owned edges carry a vertex, and how many triangles its cube emits
__global__ void __launch_bounds__(512)
k_mc_count(const McCtx c, const McTable* __restrict__ tab, uint8_t* __restrict__ eflags, unsigned* __restrict__ vcnt, unsigned* __restrict__ tcnt) {
  __shared__ float s_sdf[H9]; __shared__ unsigned s_cw[H9]; __shared__ int s_nb[8];
  int b[3];
  load_halo(c, blockIdx.x, s_sdf, s_cw, s_nb, b);
  const int l = threadIdx.x, x = l & 7, y = (l >> 3) & 7, z = l >> 6;
  const int h0 = x + 9 * y + 81 * z;
  const int hoff[3] = {1, 9, 81};
  const bool u0 = usable(s_sdf[h0], s_cw[h0], c.thr), in0 = s_sdf[h0] < 0.f;
  unsigned fl = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int h1 = h0 + hoff[a];
    if (u0 && usable(s_sdf[h1], s_cw[h1], c.thr) && (in0 != (s_sdf[h1] < 0.f))) fl |= 1u << a;
  }
  bool valid = true; unsigned cs = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int h = h0 + (k & 1) + 9 * ((k >> 1) & 1) + 81 * (k >> 2);
    valid = valid && usable(s_sdf[h], s_cw[h], c.thr);
    cs |= (unsigned)(s_sdf[h] < 0.f) << k;
  }
  const size_t o = (size_t)blockIdx.x * 512 + l;
  eflags[o] = (uint8_t)fl; vcnt[o] = __popc(fl); tcnt[o] = valid ? tab->ntri[cs] : 0u;
}

// pass C: emit vertices and triangles (pre-compaction vertex ids), mark referenced vertices
__global__ void __launch_bounds__(512)
k_mc_emit(const McCtx c, const McTable* __restrict__ tab, const uint8_t* __restrict__ eflags, const unsigned* __restrict__ vbase,
          const unsigned* __restrict__ tbase, float* __restrict__ vpos, uint8_t* __restrict__ vrgb, unsigned* __restrict__ tri,
          unsigned* __restrict__ used) {
  __shared__ float s_sdf[H9]; __shared__ unsigned s_cw[H9]; __shared__ int s_nb[8];
  int b[3];
  load_halo(c, blockIdx.x, s_sdf, s_cw, s_nb, b);
  const int l = threadIdx.x, x = l & 7, y = (l >> 3) & 7, z = l >> 6;
  const int h0 = x + 9 * y + 81 * z;
  const int hoff[3] = {1, 9, 81};
  const size_t o = (size_t)blockIdx.x * 512 + l;
  const unsigned fl = eflags[o];
  const int g[3] = {8 * b[0] + x, 8 * b[1] + y, 8 * b[2] + z};
  unsigned vid = vbase[o];
#pragma unroll
  for (int a = 0; a < 3; ++a) if (fl & (1u << a)) {
    const int h1 = h0 + hoff[a];
    const float s0 = s_sdf[h0], s1 = s_sdf[h1];
    const float t = __fdiv_rn(s0, __fsub_rn(s0, s1));
    float p[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] = __fmul_rn(i == a ? __fadd_rn((float)g[i], t) : (float)g[i], c.vs);
    vpos[3 * (size_t)vid] = p[0]; vpos[3 * (size_t)vid + 1] = p[1]; vpos[3 * (size_t)vid + 2] = p[2];
    const unsigned c0 = s_cw[h0], c1 = s_cw[h1];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float a0 = (float)((c0 >> (8 * ch)) & 0xFFu), a1 = (float)((c1 >> (8 * ch)) & 0xFFu);
      vrgb[3 * (size_t)vid + ch] = (uint8_t)__float2int_rz(__fadd_rn(__fmaf_rn(t, __fsub_rn(a1, a0), a0), 0.5f));
    }
    ++vid;
  }
  bool valid = true; unsigned cs = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int h = h0 + (k & 1) + 9 * ((k >> 1) & 1) + 81 * (k >> 2);
    valid = valid && usable(s_sdf[h], s_cw[h], c.thr);
    cs |= (unsigned)(s_sdf[h] < 0.f) << k;
  }
  if (!valid) return;
  const int nt = tab->ntri[cs];
  unsigned tid = tbase[o];
  for (int i = 0; i < 3 * nt; ++i) {
    const int e = tab->tri[cs][i], a = e >> 2, jj = e & 3, u = jj & 1, v = jj >> 1;
    const int ox = a == 0 ? 0 : u, oy = a == 0 ? u : (a == 1 ? 0 : v), oz = a == 2 ? 0 : v;      // owner voxel offset
    const int X = x + ox, Y = y + oy, Z = z + oz;
    const int nb = s_nb[(X >> 3) | ((Y >> 3) << 1) | ((Z >> 3) << 2)];
    const size_t oo = (size_t)c.inv_order[nb] * 512 + ((X & 7) | ((Y & 7) << 3) | ((Z & 7) << 6));
    const unsigned f2 = eflags[oo];
    const unsigned id = vbase[oo] + __popc(f2 & ((1u << a) - 1u));
    tri[(size_t)tid * 3 + (i % 3)] = id;
    used[id] = 1u;
    if (i % 3 == 2) ++tid;
  }
}

__global__ void k_mc_remap(unsigned* __restrict__ tri, size_t n, const unsigned* __restrict__ newid) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) tri[i] = newid[tri[i]];
}
__global__ void k_mc_compact(const float* __restrict__ vpos, const uint8_t* __restrict__ vrgb, const unsigned* __restrict__ used,
                             const unsigned* __restrict__ newid, size_t n, float* __restrict__ opos, uint8_t* __restrict__ orgb) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || !used[i]) return;
  const size_t k = newid[i];
  for (int q = 0; q < 3; ++q) { opos[3 * k + q] = vpos[3 * i + q]; orgb[3 * k + q] = vrgb[3 * i + q]; }
}

}  // namespace

extern "C" int scn_tsdf_extract_mesh(scn_tsdf* t, float** xyz, uint8_t** rgb, uint32_t** tri, uint64_t* n_verts, uint64_t* n_faces) {
  if (!t || !xyz || !tri || !n_verts || !n_faces) return scn::fail(SCN_ERR_ARG, "null argument");
  SCN_CUDA_TRY(cudaSetDevice(t->device));
  SCN_CUDA_TRY(cudaStreamSynchronize(t->stream));
  cudaStream_t st = t->stream;
  Counters cnt;
  { int rc = read_counters(t, cnt); if (rc) return rc; }
  const size_t N = (size_t)cnt.blocks;
  *n_verts = *n_faces = 0; *xyz = nullptr; *tri = nullptr; if (rgb) *rgb = nullptr;
  if (N == 0) { *xyz = (float*)malloc(16); *tri = (uint32_t*)malloc(16); if (rgb) *rgb = (uint8_t*)malloc(16); return SCN_OK; }
  // deterministic block order: ascending packed key
  std::vector<unsigned long long> keys(N);
  SCN_CUDA_TRY(cudaMemcpy(keys.data(), t->tb.block_keys, N * 8, cudaMemcpyDeviceToHost));
  std::vector<unsigned> order(N), inv(N);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), [&](unsigned a, unsigned b) { return keys[a] < keys[b]; });
  for (size_t j = 0; j < N; ++j) inv[order[j]] = (unsigned)j;
  McTable tab; build_mc_table(tab);
  const size_t NV = N * 512;
  scn::DBuf dOrder, dInv, dTab, dFl, dVc, dTc, dVb, dTb, dScr;
  if (!dOrder.alloc(N * 4) || !dInv.alloc(N * 4) || !dTab.alloc(sizeof(McTable)) || !dFl.alloc(NV) || !dVc.alloc(NV * 4) || !dTc.alloc(NV * 4) ||
      !dVb.alloc((NV + 1) * 4) || !dTb.alloc((NV + 1) * 4) || !dScr.alloc(scn::scan_scratch_elems(NV) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (marching cubes workspace, %zu blocks)", N);
  SCN_CUDA_TRY(cudaMemcpyAsync(dOrder.p, order.data(), N * 4, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(dInv.p, inv.data(), N * 4, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(dTab.p, &tab, sizeof(tab), cudaMemcpyHostToDevice, st));
  McCtx c; c.tb = t->tb; c.order = dOrder.as<unsigned>(); c.inv_order = dInv.as<unsigned>(); c.n_blocks = (unsigned)N;
  { volatile float th = t->mc_thresh_factor * t->vp.vs; c.thr = th; } c.vs = t->vp.vs;
  k_mc_count<<<(unsigned)N, 512, 0, st>>>(c, dTab.as<McTable>(), dFl.as<uint8_t>(), dVc.as<unsigned>(), dTc.as<unsigned>());
  scn::exclusive_scan_u32(dVc.as<unsigned>(), dVb.as<unsigned>(), NV, dScr.as<unsigned>(), st);
  scn::exclusive_scan_u32(dTc.as<unsigned>(), dTb.as<unsigned>(), NV, dScr.as<unsigned>(), st);
  unsigned nV0 = 0, nT = 0;
  SCN_CUDA_TRY(cudaMemcpyAsync(&nV0, dVb.as<unsigned>() + NV, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(&nT, dTb.as<unsigned>() + NV, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  scn::DBuf dPos, dRgb, dTri, dUsed, dNew, dPos2, dRgb2;
  if (!dPos.alloc((size_t)nV0 * 12) || !dRgb.alloc((size_t)nV0 * 3) || !dTri.alloc((size_t)nT * 12) || !dUsed.alloc((size_t)nV0 * 4) || !dNew.alloc(((size_t)nV0 + 1) * 4))
    return scn::fail(SCN_ERR_CUDA, "cudaMalloc (mesh buffers: %u vertices, %u triangles)", nV0, nT);
  SCN_CUDA_TRY(cudaMemsetAsync(dUsed.p, 0, (size_t)nV0 * 4, st));
  k_mc_emit<<<(unsigned)N, 512, 0, st>>>(c, dTab.as<McTable>(), dFl.as<uint8_t>(), dVb.as<unsigned>(), dTb.as<unsigned>(), dPos.as<float>(),
                                          dRgb.as<uint8_t>(), dTri.as<unsigned>(), dUsed.as<unsigned>());
  scn::DBuf dScr2; if (!dScr2.alloc(scn::scan_scratch_elems(nV0) * 4)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc");
  scn::exclusive_scan_u32(dUsed.as<unsigned>(), dNew.as<unsigned>(), nV0, dScr2.as<unsigned>(), st);
  unsigned nV = 0;
  SCN_CUDA_TRY(cudaMemcpyAsync(&nV, dNew.as<unsigned>() + nV0, 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  if (!dPos2.alloc((size_t)nV * 12) || !dRgb2.alloc((size_t)nV * 3)) return scn::fail(SCN_ERR_CUDA, "cudaMalloc");
  if (nT) k_mc_remap<<<(unsigned)(((size_t)nT * 3 + 255) / 256), 256, 0, st>>>(dTri.as<unsigned>(), (size_t)nT * 3, dNew.as<unsigned>());
  if (nV0) k_mc_compact<<<(unsigned)(((size_t)nV0 + 255) / 256), 256, 0, st>>>(dPos.as<float>(), dRgb.as<uint8_t>(), dUsed.as<unsigned>(), dNew.as<unsigned>(), nV0,
                                                                                dPos2.as<float>(), dRgb2.as<uint8_t>());
  SCN_CUDA_TRY(cudaGetLastError());
  scn::MallocPtr<float> hxyz((float*)malloc(std::max<size_t>(16, (size_t)nV * 12)));
  scn::MallocPtr<uint32_t> htri((uint32_t*)malloc(std::max<size_t>(16, (size_t)nT * 12)));
  scn::MallocPtr<uint8_t> hrgb((uint8_t*)malloc(std::max<size_t>(16, (size_t)nV * 3)));
  if (!hxyz || !htri || !hrgb) return scn::fail(SCN_ERR_ARG, "out of host memory");
  SCN_CUDA_TRY(cudaMemcpy(hxyz.get(), dPos2.p, (size_t)nV * 12, cudaMemcpyDeviceToHost));
  SCN_CUDA_TRY(cudaMemcpy(hrgb.get(), dRgb2.p, (size_t)nV * 3, cudaMemcpyDeviceToHost));
  SCN_CUDA_TRY(cudaMemcpy(htri.get(), dTri.p, (size_t)nT * 12, cudaMemcpyDeviceToHost));
  *xyz = hxyz.release(); *tri = htri.release(); if (rgb) *rgb = hrgb.release();
  *n_verts = nV; *n_faces = nT;
  t->launches += 8;
  return SCN_OK;
}
