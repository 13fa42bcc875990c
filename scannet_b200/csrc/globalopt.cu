// Global optimisation of the keyframe trajectory (DESIGN.md §6k, "global optimisation spec v1"): the dense geometric term of
// BundleFusion's global stage, without sparse features, in the binary32 / binary64 operations and order of
// oracle/globalopt_oracle.c (the library is built with -fmad=false: no contraction), so that edges, sums and poses compare bit for bit.
//
// Keyframes: depth -> metres (-inf invalid) -> bilateral filter (when the volume filters) -> range test [depth_min, depth_max] ->
// 2x2 reductions to width x height -> vertex + normal maps (icp_common.cuh, §6j step 1), kept on the device for every keyframe.
// Solve, on the volume's stream:
//   go_overlap       every pair (i < j) at the initial poses: j's subsampled pixels associated against i's maps; one flag per pair.
//                    The flags go to the host once, which lists the edges in (i, j) order.
//   per solve (the host uploads the active edges, their CSR and the gauge, then launches without reading anything back):
//     nonlin_iters x [go_linearise (one CTA per 256 pixels of an edge: association, the 28 products, the §6j step-4 tree)
//                     -> go_edge_sums (slots in order) -> go_totals -> go_assemble (diagonal blocks, -g, damping, Cholesky of the
//                     preconditioner) -> go_pcg (one CTA: the whole PCG) -> go_update (Cayley, binary64)]
//     then go_linearise + go_edge_sums + go_verify at the final poses; the host reads one GoState and removes the worst edge or stops.
#include <algorithm>
#include <cmath>
#include <vector>

#include "icp_common.cuh"
#include "tsdf_internal.cuh"

namespace {

constexpr int kMaxNonlin = 16;
constexpr int kPcgThreads = 512;                   // leaves of the fixed dot-product tree
constexpr unsigned kOverlapNum = 1, kOverlapDen = 4;   // an overlap check passes when found / valid >= 1/4
constexpr int kEdgeChunk = 16384;                  // edges linearised per launch: bounds the partial sums to 16384 * slots * 224 B

struct GoState {                                   // device; one solve
  double rss_iter[kMaxNonlin + 1];
  unsigned long long pairs_iter[kMaxNonlin + 1];
  int chol_fail[kMaxNonlin];
  int nonfinite;
  unsigned lin_run;
  int worst;                                       // active-edge index of the worst failing edge, -1 when none fails
  double max_rms;
};

struct Edges {                                     // the active edges of a solve, in (i, j) order, and their incidence
  int ne;
  const int* ei; const int* ej;
  const int* nptr; const int* nedge;               // node k's edges: nedge[nptr[k] .. nptr[k+1]), in edge order
};

struct Sys {
  int n;
  Edges E;
  const double* esum; const unsigned* epairs;
  const int* fixed;
  double* Hd; double* Lc; double* rhs;             // n * 36, n * 36, 6 n
  int* fr;                                         // node moves in this iteration
  double *x, *r, *z, *p, *q;                       // 6 n each
  GoState* st;
};

// ---------------------------------------------------------------------------------------------------------------- residuals
// M = Ti^-1 Tj (3x4) in binary64 with Ti^-1 = [R^T | -R^T t], rounded once
__device__ void relative(const double* Di, const double* Dj, float* M) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double m = __dadd_rn(__dadd_rn(__dmul_rn(Di[r], Dj[c]), __dmul_rn(Di[4 + r], Dj[4 + c])), __dmul_rn(Di[8 + r], Dj[8 + c]));
      if (c == 3) m = __dsub_rn(m, __dadd_rn(__dadd_rn(__dmul_rn(Di[r], Di[3]), __dmul_rn(Di[4 + r], Di[7])), __dmul_rn(Di[8 + r], Di[11])));
      M[4 * r + c] = (float)m;
    }
}

__global__ void __launch_bounds__(kCta) go_overlap(const Level l, const Thresh th, int n, int f, const double* __restrict__ D,
                                                   const float4* __restrict__ V, const float4* __restrict__ N, unsigned char* __restrict__ flag) {
  const int j = blockIdx.x, i = blockIdx.y;
  if (i >= j) return;
  __shared__ float M[12];
  if (threadIdx.x == 0) relative(D + 12 * i, D + 12 * j, M);
  __syncthreads();
  float Mr[12];
#pragma unroll
  for (int q = 0; q < 12; ++q) Mr[q] = M[q];
  const size_t npx = (size_t)l.W * l.H;
  const int xs = (l.W + f - 1) / f, ys = (l.H + f - 1) / f;
  unsigned valid = 0, found = 0;
  for (int base = 0; base < xs * ys; base += kCta) {
    const int idx = base + threadIdx.x;
    bool v = false, fd = false;
    if (idx < xs * ys) {
      const int t = (idx / xs) * f * l.W + (idx % xs) * f;
      const float4 np = N[npx * j + t];
      Assoc a;
      v = np.w != 0.f;
      fd = associate(l, V + npx * i, N + npx * i, th, Mr, V[npx * j + t], np, a);
    }
    valid += __syncthreads_count(v);
    found += __syncthreads_count(fd);
  }
  if (threadIdx.x == 0) flag[(size_t)i * n + j] = valid > 0 && (unsigned long long)found * kOverlapDen >= (unsigned long long)valid * kOverlapNum;
}

// One CTA per 256 pixels (blockIdx.y) of j for active edge e0 + blockIdx.x: association against i, a = [(w_j x n^w), n^w], the 28 products, the tree
__global__ void __launch_bounds__(kCta) go_linearise(const Level l, const Thresh th, const Edges E, int e0, const double* __restrict__ D,
                                                     const float4* __restrict__ V, const float4* __restrict__ N, double* __restrict__ part,
                                                     unsigned* __restrict__ part_n) {
  __shared__ double s_w[kCta / 32][kNSum];
  __shared__ float s_m[36];                          // M, Tj, Ri
  const int e = e0 + blockIdx.x, i = E.ei[e], j = E.ej[e];
  if (threadIdx.x == 0) relative(D + 12 * i, D + 12 * j, s_m);
  if (threadIdx.x < 12) { s_m[12 + threadIdx.x] = (float)D[12 * j + threadIdx.x]; s_m[24 + threadIdx.x] = (float)D[12 * i + threadIdx.x]; }
  __syncthreads();
  const size_t npx = (size_t)l.W * l.H;
  const int px = blockIdx.y * kCta + threadIdx.x;
  double v[kNSum];
#pragma unroll
  for (int q = 0; q < kNSum; ++q) v[q] = 0.0;
  bool paired = false;
  if (px < (int)npx) {
    float M[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) M[q] = s_m[q];
    const float4 p = V[npx * j + px];
    Assoc as;
    paired = associate(l, V + npx * i, N + npx * i, th, M, p, N[npx * j + px], as);
    if (paired) {
      const float* Tj = s_m + 12; const float* Ri = s_m + 24;
      const float wx = __fadd_rn(dot3(Tj[0], Tj[1], Tj[2], p.x, p.y, p.z), Tj[3]);
      const float wy = __fadd_rn(dot3(Tj[4], Tj[5], Tj[6], p.x, p.y, p.z), Tj[7]);
      const float wz = __fadd_rn(dot3(Tj[8], Tj[9], Tj[10], p.x, p.y, p.z), Tj[11]);
      const float4 nq = as.nq;
      const float nx = dot3(Ri[0], Ri[1], Ri[2], nq.x, nq.y, nq.z);
      const float ny = dot3(Ri[4], Ri[5], Ri[6], nq.x, nq.y, nq.z);
      const float nz = dot3(Ri[8], Ri[9], Ri[10], nq.x, nq.y, nq.z);
      const float a[6] = {__fsub_rn(__fmul_rn(wy, nz), __fmul_rn(wz, ny)), __fsub_rn(__fmul_rn(wz, nx), __fmul_rn(wx, nz)),
                          __fsub_rn(__fmul_rn(wx, ny), __fmul_rn(wy, nx)), nx, ny, nz};
      products28(a, as.r, v);
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < kNSum; ++q) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v[q] = __dadd_rn(v[q], __shfl_down_sync(0xffffffffu, v[q], s));
    if (lane == 0) s_w[warp][q] = v[q];
  }
  const unsigned cnt = __syncthreads_count(paired);
  const size_t slot = (size_t)blockIdx.x * gridDim.y + blockIdx.y;       // within the chunk of edges from e0
  if (threadIdx.x < kNSum) {
    double a[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) a[w] = s_w[w][threadIdx.x];
#pragma unroll
    for (int s = 4; s > 0; s >>= 1)
#pragma unroll
      for (int t = 0; t < s; ++t) a[t] = __dadd_rn(a[t], a[t + s]);
    part[slot * kNSum + threadIdx.x] = a[0];
  }
  if (threadIdx.x == 0) part_n[slot] = cnt;
}

// one thread per active edge of a chunk: its slots in slot order
__global__ void go_edge_sums(int ne, int e0, int slots, const double* __restrict__ part, const unsigned* __restrict__ part_n,
                             double* __restrict__ esum, unsigned* __restrict__ epairs) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;              // within the chunk
  if (e >= ne) return;
  for (int q = 0; q < kNSum; ++q) {
    double s = 0.0;
    for (int c = 0; c < slots; ++c) s = __dadd_rn(s, part[((size_t)e * slots + c) * kNSum + q]);
    esum[(size_t)(e0 + e) * kNSum + q] = s;
  }
  unsigned n = 0;
  for (int c = 0; c < slots; ++c) n += part_n[(size_t)e * slots + c];
  epairs[e0 + e] = n;
}

// sum r^2 and pairs over the active edges in edge order
__global__ void go_totals(int ne, int it, const double* __restrict__ esum, const unsigned* __restrict__ epairs, GoState* st) {
  double rss = 0.0; unsigned long long pairs = 0;
  for (int e = 0; e < ne; ++e) { rss = __dadd_rn(rss, esum[(size_t)e * kNSum + 27]); pairs += epairs[e]; }
  st->rss_iter[it] = rss; st->pairs_iter[it] = pairs;
}

// ---------------------------------------------------------------------------------------------------------------- system
// one thread per node: H_kk = sum of S over its edges in edge order + 2^-13 * pairs, -g, the free flag, the preconditioner's factor
__global__ void go_assemble(const Sys S, int it) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= S.n) return;
  double H[6][6], g[6];
  for (int a = 0; a < 6; ++a) { g[a] = 0.0; for (int b = 0; b < 6; ++b) H[a][b] = 0.0; }
  unsigned pk = 0;
  for (int t = S.E.nptr[k]; t < S.E.nptr[k + 1]; ++t) {
    const int e = S.E.nedge[t];
    const double* s = S.esum + (size_t)e * kNSum;
    int q = 0;
    for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) { H[a][b] = __dadd_rn(H[a][b], s[q]); ++q; }
    const bool is_j = S.E.ej[e] == k;
    for (int a = 0; a < 6; ++a) g[a] = is_j ? __dadd_rn(g[a], s[21 + a]) : __dsub_rn(g[a], s[21 + a]);
    pk += S.epairs[e];
  }
  const double lambda = __dmul_rn(kDamp, (double)pk);
  for (int a = 0; a < 6; ++a) H[a][a] = __dadd_rn(H[a][a], lambda);
  for (int a = 0; a < 6; ++a) for (int b = 0; b < a; ++b) H[a][b] = H[b][a];
  const int fr = !S.fixed[k] && pk > 0;
  S.fr[k] = fr;
  for (int a = 0; a < 6; ++a) {
    S.rhs[6 * k + a] = fr ? -g[a] : 0.0;
    for (int b = 0; b < 6; ++b) S.Hd[36 * k + 6 * a + b] = H[a][b];
  }
  if (fr) {
    double L[6][6];
    if (!chol6(H, L)) S.st->chol_fail[it] = 1;
    for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) S.Lc[36 * k + 6 * a + b] = b <= a ? L[a][b] : 0.0;
  }
}

__device__ __forceinline__ double block_dot(const double* a, const double* b, int m, double* leaf) {
  double s = 0.0;
  for (int q = threadIdx.x; q < m; q += kPcgThreads) s = __dadd_rn(s, __dmul_rn(a[q], b[q]));
  leaf[threadIdx.x] = s;
  __syncthreads();
  for (int h = kPcgThreads / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) leaf[threadIdx.x] = __dadd_rn(leaf[threadIdx.x], leaf[threadIdx.x + h]);
    __syncthreads();
  }
  const double r = leaf[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ void precond(const Sys& S, const double* r, double* z) {
  for (int k = threadIdx.x; k < S.n; k += kPcgThreads) {
    if (!S.fr[k]) { for (int a = 0; a < 6; ++a) z[6 * k + a] = 0.0; continue; }
    double L[6][6];
    for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) L[a][b] = S.Lc[36 * k + 6 * a + b];
    chol6_solve(L, r + 6 * k, z + 6 * k);
  }
}

// y = H x: per row, the diagonal block first, then the node's edges in edge order (H_ij = -S)
__device__ __forceinline__ void matvec(const Sys& S, const double* x, double* y) {
  for (int row = threadIdx.x; row < 6 * S.n; row += kPcgThreads) {
    const int k = row / 6, a = row % 6;
    if (!S.fr[k]) { y[row] = 0.0; continue; }
    double acc = 0.0;
    for (int c = 0; c < 6; ++c) acc = __dadd_rn(acc, __dmul_rn(S.Hd[36 * k + 6 * a + c], x[6 * k + c]));
    for (int t = S.E.nptr[k]; t < S.E.nptr[k + 1]; ++t) {
      const int e = S.E.nedge[t];
      const int o = S.E.ei[e] == k ? S.E.ej[e] : S.E.ei[e];
      const double* s = S.esum + (size_t)e * kNSum;
      for (int c = 0; c < 6; ++c) {
        const int lo = a < c ? a : c, hi = a < c ? c : a;
        acc = __dsub_rn(acc, __dmul_rn(s[lo * 6 - lo * (lo - 1) / 2 + (hi - lo)], x[6 * o + c]));
      }
    }
    y[row] = acc;
  }
}

// PCG from x = 0 for `iters` iterations in one CTA, stopping early only when r.z is exactly 0
__global__ void __launch_bounds__(kPcgThreads) go_pcg(const Sys S, int it, int iters) {
  __shared__ double leaf[kPcgThreads];
  const int m = 6 * S.n;
  for (int a = threadIdx.x; a < m; a += kPcgThreads) { S.x[a] = 0.0; S.r[a] = S.rhs[a]; }
  if (S.st->chol_fail[it]) return;                 // written by go_assemble: the same for every thread; x stays 0
  __syncthreads();
  precond(S, S.r, S.z);
  __syncthreads();
  for (int a = threadIdx.x; a < m; a += kPcgThreads) S.p[a] = S.z[a];
  double rz = block_dot(S.r, S.z, m, leaf);
  unsigned run = 0;
  for (int i = 0; i < iters; ++i) {
    if (rz == 0.0) break;
    matvec(S, S.p, S.q);
    __syncthreads();
    const double alpha = __ddiv_rn(rz, block_dot(S.p, S.q, m, leaf));
    for (int a = threadIdx.x; a < m; a += kPcgThreads) {
      S.x[a] = __dadd_rn(S.x[a], __dmul_rn(alpha, S.p[a]));
      S.r[a] = __dsub_rn(S.r[a], __dmul_rn(alpha, S.q[a]));
    }
    __syncthreads();
    precond(S, S.r, S.z);
    __syncthreads();
    const double rzn = block_dot(S.r, S.z, m, leaf);
    const double beta = __ddiv_rn(rzn, rz);
    for (int a = threadIdx.x; a < m; a += kPcgThreads) S.p[a] = __dadd_rn(S.z[a], __dmul_rn(beta, S.p[a]));
    __syncthreads();
    rz = rzn;
    ++run;
  }
  if (threadIdx.x == 0) S.st->lin_run += run;
}

__global__ void go_update(const Sys S, double* D) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= S.n || !S.fr[k]) return;
  apply_update(D + 12 * k, S.x + 6 * k);
  bool fin = true;
  for (int q = 0; q < 12; ++q) fin = fin && isfinite(D[12 * k + q]);
  if (!fin) S.st->nonfinite = 1;
}

// at the final poses: every active edge's RMS, the largest, and the worst failing edge (fewer than kMinPairs pairs ranks above any
// RMS; ties go to the lowest (i, j))
__global__ void go_verify(int ne, double thresh, const double* __restrict__ esum, const unsigned* __restrict__ epairs, GoState* st) {
  int worst = -1; double ws = 0.0, mx = 0.0;
  for (int e = 0; e < ne; ++e) {
    const unsigned pe = epairs[e];
    const double rms = pe ? __dsqrt_rn(__ddiv_rn(esum[(size_t)e * kNSum + 27], (double)pe)) : 0.0;
    if (rms > mx) mx = rms;
    const double score = pe < kMinPairs ? INFINITY : rms;
    if ((pe < kMinPairs || rms > thresh) && (worst < 0 || score > ws)) { worst = e; ws = score; }
  }
  st->worst = worst; st->max_rms = mx;
  for (int it = 0; it < kMaxNonlin; ++it) if (st->chol_fail[it]) st->nonfinite = 1;
}

unsigned grid(int n) { return (unsigned)((n + kCta - 1) / kCta); }

}  // namespace

struct scn_globalopt {
  scn_globalopt_params p{};
  scn_tsdf* vol = nullptr;
  int s = 0;                                       // depth resolution = keyframe resolution * 2^s
  Level L{};
  float K[16]{};
  bool have_K = false;
  uint32_t n = 0;                                  // keyframes held
  std::vector<double> D0;                          // n * 12, the poses handed in
  scn::DBuf raw, metres, full, chain, depth, V, N;
  std::vector<float*> chain_ptr;
  scn::DBuf d_D0, d_D, flags, st;
  scn::DBuf ei, ej, nptr, nedge, fixed, part, part_n, esum, epairs, Hd, Lc, vec, fr;
  size_t cap_edges = 0, cap_nodes = 0;            // what the per-solve buffers below hold
  std::vector<scn_globalopt_edge_t> edges;         // the last solve's
  std::vector<scn::EventPtr> ev;                   // timing marks of the current call
  std::vector<int> ev_phase;                       // phase of the segment that ends at mark k
  double phase_ms[5] = {0, 0, 0, 0, 0};            // keyframe maps, overlap, linearise, PCG, verify
};

namespace {

enum { PH_MAPS = 0, PH_OVERLAP, PH_LINEARISE, PH_PCG, PH_VERIFY };

// records a mark; the segment from the previous mark to this one is timed as `phase` (-1: not timed)
int mark(scn_globalopt* g, int phase) {
  const size_t k = g->ev_phase.size();
  if (k == g->ev.size()) { g->ev.emplace_back(); SCN_CUDA_TRY(scn::create(g->ev.back())); }
  SCN_CUDA_TRY(cudaEventRecord(g->ev[k].get(), g->vol->stream));
  g->ev_phase.push_back(phase);
  return SCN_OK;
}

// adds the marks' segments to the phase times; the stream has been synchronised
int collect(scn_globalopt* g) {
  for (size_t k = 1; k < g->ev_phase.size(); ++k) {
    if (g->ev_phase[k] < 0) continue;              // a gap between timed phases
    float ms = 0.f;
    SCN_CUDA_TRY(cudaEventElapsedTime(&ms, g->ev[k - 1].get(), g->ev[k].get()));
    g->phase_ms[g->ev_phase[k]] += ms;
  }
  g->ev_phase.clear();
  return SCN_OK;
}

int root(std::vector<int>& par, int k) { while (par[k] != k) k = par[k] = par[par[k]]; return k; }

}  // namespace

extern "C" {

void scn_globalopt_default_params(scn_globalopt_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->submap_size = 10;                             // s_submapSize, zParametersBundlingScanNet.txt
  p->max_keyframes = 2000;                         // s_maxNumImages
  p->width = 80; p->height = 60;                   // s_downsampledWidth / Height
  p->dist_thresh = 0.15f;                          // s_denseDistThresh
  p->normal_thresh = 0.95f;                        // s_denseNormalThresh
  p->depth_min = 0.5f; p->depth_max = 4.0f;        // s_denseDepthMin / Max
  p->overlap_subsample = 4;                        // s_denseOverlapCheckSubsampleFactor
  p->nonlin_iters = 3;                             // s_numGlobalNonLinIterations
  p->lin_iters = 150;                              // s_numGlobalLinIterations
  p->verify_thresh = 0.05f;                        // s_verifyOptErrThresh
  p->max_removed = 10;                             // s_maxNumResidualsRemoved
}

int scn_globalopt_params_from_file(const char* path, scn_globalopt_params* p) {
  if (!path || !p) return scn::fail(SCN_ERR_ARG, "null argument");
  FILE* f = fopen(path, "rb");
  if (!f) return scn::fail(SCN_ERR_IO, "cannot open parameter file %s", path);
  char line[4096];
  while (fgets(line, sizeof(line), f)) {
    char* c = strstr(line, "//");
    if (c) *c = 0;
    char key[256]; char val[1024];
    if (sscanf(line, " %255[A-Za-z0-9_] = %1023[^;];", key, val) != 2) continue;
    const double v = atof(val);
    if (!strcmp(key, "s_submapSize")) p->submap_size = (uint32_t)v;
    else if (!strcmp(key, "s_maxNumImages")) p->max_keyframes = (uint32_t)v;
    else if (!strcmp(key, "s_downsampledWidth")) p->width = (uint32_t)v;
    else if (!strcmp(key, "s_downsampledHeight")) p->height = (uint32_t)v;
    else if (!strcmp(key, "s_denseDistThresh")) p->dist_thresh = (float)v;
    else if (!strcmp(key, "s_denseNormalThresh")) p->normal_thresh = (float)v;
    else if (!strcmp(key, "s_denseDepthMin")) p->depth_min = (float)v;
    else if (!strcmp(key, "s_denseDepthMax")) p->depth_max = (float)v;
    else if (!strcmp(key, "s_denseOverlapCheckSubsampleFactor")) p->overlap_subsample = (uint32_t)v;
    else if (!strcmp(key, "s_numGlobalNonLinIterations")) p->nonlin_iters = (uint32_t)v;
    else if (!strcmp(key, "s_numGlobalLinIterations")) p->lin_iters = (uint32_t)v;
    else if (!strcmp(key, "s_verifyOptErrThresh")) p->verify_thresh = (float)v;
    else if (!strcmp(key, "s_maxNumResidualsRemoved")) p->max_removed = (uint32_t)v;
  }
  fclose(f);
  return SCN_OK;
}

size_t scn_globalopt_report_sizeof(void) { return sizeof(scn_globalopt_report_t); }

int scn_globalopt_create(scn_tsdf* vol, const scn_globalopt_params* p, scn_globalopt** out) {
  if (!vol || !p || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  const uint32_t W = vol->p.width, H = vol->p.height;
  int s = 0;
  while (s < 16 && (W >> s) > p->width) ++s;
  if (!p->width || !p->height || (W >> s) != p->width || W % p->width || H % p->height || H / p->height != W / p->width)
    return scn::fail(SCN_ERR_ARG, "keyframe resolution %ux%u is not the depth resolution %ux%u divided by a power of two", p->width, p->height, W, H);
  if (p->width < 3 || p->height < 3) return scn::fail(SCN_ERR_ARG, "keyframe resolution %ux%u below 3x3", p->width, p->height);
  if (!p->max_keyframes || p->max_keyframes > 65535 || !p->submap_size || !p->overlap_subsample || p->nonlin_iters > kMaxNonlin || !(p->dist_thresh > 0.f) ||
      std::isnan(p->normal_thresh) || !(p->depth_max >= p->depth_min) || std::isnan(p->verify_thresh))
    return scn::fail(SCN_ERR_ARG, "invalid global optimisation parameters");
  SCN_CUDA_TRY(cudaSetDevice(vol->device));
  std::unique_ptr<scn_globalopt> g(new scn_globalopt());
  g->p = *p; g->vol = vol; g->s = s;
  const size_t px = (size_t)W * H, npx = (size_t)p->width * p->height;
  SCN_ALLOC(g->raw, px * 4); SCN_ALLOC(g->metres, px * 4); SCN_ALLOC(g->full, px * 4);
  size_t chain = 0;
  for (int k = 1; k < s; ++k) chain += (size_t)(W >> k) * (H >> k);
  SCN_ALLOC(g->chain, chain * 4);
  for (int k = 1, off = 0; k < s; ++k) { g->chain_ptr.push_back(g->chain.as<float>() + off); off += (W >> k) * (H >> k); }
  g->chain_ptr.push_back(nullptr);
  SCN_ALLOC(g->depth, npx * 4);
  SCN_ALLOC(g->V, npx * 16 * p->max_keyframes); SCN_ALLOC(g->N, npx * 16 * p->max_keyframes);
  SCN_ALLOC(g->st, sizeof(GoState));
  g->L.W = (int)p->width; g->L.H = (int)p->height;
  *out = g.release();
  return SCN_OK;
}

void scn_globalopt_destroy(scn_globalopt* g) {
  if (!g) return;
  cudaSetDevice(g->vol->device);
  cudaStreamSynchronize(g->vol->stream);
  delete g;
}

int scn_globalopt_add_keyframes(scn_globalopt* g, uint32_t n, const uint16_t* d_depth, const float* poses, const float K[16]) {
  if (!g || (n && (!d_depth || !poses || !K))) return scn::fail(SCN_ERR_ARG, "null argument");
  if ((uint64_t)g->n + n > g->p.max_keyframes)
    return scn::fail(SCN_ERR_CAPACITY, "%u keyframes exceed max_keyframes %u", g->n + n, g->p.max_keyframes);
  for (uint64_t i = 0; i < 16ull * n; ++i) if (!std::isfinite(poses[i])) return scn::fail(SCN_ERR_ARG, "keyframe %u has no finite pose", g->n + (uint32_t)(i / 16));
  if (n && g->have_K && memcmp(K, g->K, sizeof(g->K))) return scn::fail(SCN_ERR_ARG, "keyframes with different intrinsics");
  if (!n) return SCN_OK;
  scn_tsdf* v = g->vol;
  SCN_CUDA_TRY(cudaSetDevice(v->device));
  const cudaStream_t st = v->stream;
  const int W = (int)v->p.width, H = (int)v->p.height;
  const size_t px = (size_t)W * H, npx = (size_t)g->L.W * g->L.H;
  if (!g->have_K) { memcpy(g->K, K, sizeof(g->K)); level_intrinsics(g->L, K, g->s); g->have_K = true; }
  if (int rc = mark(g, -1)) return rc;
  for (uint32_t f = 0; f < n; ++f) {
    if (int rc = scn_depth_to_metres_device(d_depth + f * px, W, H, v->p.depth_shift, v->p.depth_filter != 0, v->p.depth_sigma_d, v->p.depth_sigma_r,
                                            g->raw.as<float>(), g->metres.as<float>(), st))
      return rc;
    k_range<<<grid(W * H), kCta, 0, st>>>(g->metres.as<float>(), W * H, g->p.depth_min, g->p.depth_max, g->full.as<float>());
    const float* src = g->full.as<float>();
    for (int k = 0; k < g->s; ++k) {
      float* dst = k + 1 == g->s ? g->depth.as<float>() : g->chain_ptr[k];
      k_reduce2<<<grid((W >> (k + 1)) * (H >> (k + 1))), kCta, 0, st>>>(src, W >> k, H >> k, dst);
      src = dst;
    }
    if (g->s == 0) SCN_CUDA_TRY(cudaMemcpyAsync(g->depth.p, src, px * 4, cudaMemcpyDeviceToDevice, st));
    const size_t k = g->n + f;
    k_vertex_normal<<<grid((int)npx), kCta, 0, st>>>(g->L, g->depth.as<float>(), g->V.as<float4>() + k * npx, g->N.as<float4>() + k * npx, nullptr);
    SCN_CUDA_TRY(cudaGetLastError());
  }
  if (int rc = mark(g, PH_MAPS)) return rc;
  SCN_CUDA_TRY(cudaStreamSynchronize(st));
  if (int rc = collect(g)) return rc;
  for (uint32_t f = 0; f < n; ++f)
    for (int q = 0; q < 12; ++q) g->D0.push_back((double)poses[16 * f + q]);
  g->n += n;
  return SCN_OK;
}

int scn_globalopt_solve(scn_globalopt* g, float* poses_out, scn_globalopt_report_t* report) {
  if (!g || (g->n && !poses_out)) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_tsdf* v = g->vol;
  SCN_CUDA_TRY(cudaSetDevice(v->device));
  const cudaStream_t st = v->stream;
  const int n = (int)g->n;
  scn_globalopt_report_t rep; memset(&rep, 0, sizeof(rep));
  rep.keyframes = g->n;
  g->edges.clear();
  for (int k = PH_OVERLAP; k <= PH_VERIFY; ++k) g->phase_ms[k] = 0.0;   // the keyframe maps' time accumulates over the adds
  const Thresh th{g->p.dist_thresh * g->p.dist_thresh, g->p.normal_thresh};
  const size_t npx = (size_t)g->L.W * g->L.H;
  const int slots = (int)((npx + kCta - 1) / kCta);
  // every pair at the initial poses
  std::vector<unsigned char> flags((size_t)n * n, 0);
  if (n > 1) {
    SCN_ALLOC(g->d_D0, sizeof(double) * 12 * n); SCN_ALLOC(g->d_D, sizeof(double) * 12 * n);
    SCN_CUDA_TRY(cudaMemcpyAsync(g->d_D0.p, g->D0.data(), sizeof(double) * 12 * n, cudaMemcpyHostToDevice, st));
    SCN_ALLOC(g->flags, (size_t)n * n);
    SCN_CUDA_TRY(cudaMemsetAsync(g->flags.p, 0, (size_t)n * n, st));
    if (int rc = mark(g, -1)) return rc;
    go_overlap<<<dim3(n, n), kCta, 0, st>>>(g->L, th, n, (int)g->p.overlap_subsample, g->d_D0.as<double>(), g->V.as<float4>(), g->N.as<float4>(),
                                            g->flags.as<unsigned char>());
    SCN_CUDA_TRY(cudaGetLastError());
    if (int rc = mark(g, PH_OVERLAP)) return rc;
    SCN_CUDA_TRY(cudaMemcpyAsync(flags.data(), g->flags.p, (size_t)n * n, cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
  }
  std::vector<int> ei, ej;
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j)
      if (j == i + 1 || flags[(size_t)i * n + j]) {
        ei.push_back(i); ej.push_back(j);
        scn_globalopt_edge_t e; memset(&e, 0, sizeof(e));
        e.i = (uint32_t)i; e.j = (uint32_t)j; e.loop = j != i + 1;
        g->edges.push_back(e);
        (j == i + 1 ? rep.edges_consecutive : rep.edges_loop)++;
      }
  const int ne_all = (int)ei.size();
  std::vector<char> active(ne_all, 1);
  std::vector<double> D((size_t)12 * n);
  memcpy(D.data(), g->D0.data(), sizeof(double) * 12 * n);
  GoState hs; memset(&hs, 0, sizeof(hs));
  std::vector<int> act;
  if ((size_t)ne_all > g->cap_edges) {               // the per-solve buffers grow to the largest solve so far
    const size_t chunk = std::min(kEdgeChunk, ne_all);
    g->cap_edges = 0;
    SCN_ALLOC(g->ei, 4 * (size_t)ne_all); SCN_ALLOC(g->ej, 4 * (size_t)ne_all); SCN_ALLOC(g->nedge, 8 * (size_t)ne_all);
    SCN_ALLOC(g->part, chunk * slots * kNSum * 8); SCN_ALLOC(g->part_n, chunk * slots * 4);
    SCN_ALLOC(g->esum, (size_t)ne_all * kNSum * 8); SCN_ALLOC(g->epairs, (size_t)ne_all * 4);
    g->cap_edges = (size_t)ne_all;
  }
  if (ne_all && (size_t)n > g->cap_nodes) {
    g->cap_nodes = 0;
    SCN_ALLOC(g->nptr, 4 * (size_t)(n + 1)); SCN_ALLOC(g->fixed, 4 * (size_t)n); SCN_ALLOC(g->fr, 4 * (size_t)n);
    SCN_ALLOC(g->Hd, (size_t)n * 36 * 8); SCN_ALLOC(g->Lc, (size_t)n * 36 * 8); SCN_ALLOC(g->vec, (size_t)n * 6 * 8 * 6);
    g->cap_nodes = (size_t)n;
  }
  bool first = true;
  while (ne_all) {
    // the active edges, their incidence and the gauge
    act.clear();
    for (int e = 0; e < ne_all; ++e) if (active[e]) act.push_back(e);
    const int ne = (int)act.size();
    std::vector<int> aei(ne), aej(ne), nptr(n + 1, 0), nedge(2 * (size_t)ne), fixed(n);
    for (int a = 0; a < ne; ++a) { aei[a] = ei[act[a]]; aej[a] = ej[act[a]]; ++nptr[aei[a] + 1]; ++nptr[aej[a] + 1]; }
    for (int k = 0; k < n; ++k) nptr[k + 1] += nptr[k];
    std::vector<int> fill(nptr.begin(), nptr.end() - 1);
    for (int a = 0; a < ne; ++a) { nedge[fill[aei[a]]++] = a; nedge[fill[aej[a]]++] = a; }
    std::vector<int> par(n);
    for (int k = 0; k < n; ++k) par[k] = k;
    for (int a = 0; a < ne; ++a) { const int x = root(par, aei[a]), y = root(par, aej[a]); if (x != y) { if (x < y) par[y] = x; else par[x] = y; } }
    for (int k = 0; k < n; ++k) fixed[k] = root(par, k) == k;
    if (ne) {
      SCN_CUDA_TRY(cudaMemcpyAsync(g->ei.p, aei.data(), 4 * ne, cudaMemcpyHostToDevice, st));
      SCN_CUDA_TRY(cudaMemcpyAsync(g->ej.p, aej.data(), 4 * ne, cudaMemcpyHostToDevice, st));
      SCN_CUDA_TRY(cudaMemcpyAsync(g->nedge.p, nedge.data(), 8 * (size_t)ne, cudaMemcpyHostToDevice, st));
    }
    SCN_CUDA_TRY(cudaMemcpyAsync(g->nptr.p, nptr.data(), 4 * (n + 1), cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(g->fixed.p, fixed.data(), 4 * n, cudaMemcpyHostToDevice, st));
    SCN_CUDA_TRY(cudaMemcpyAsync(g->d_D.p, g->d_D0.p, sizeof(double) * 12 * n, cudaMemcpyDeviceToDevice, st));
    SCN_CUDA_TRY(cudaMemsetAsync(g->st.p, 0, sizeof(GoState), st));
    const Edges E{ne, g->ei.as<int>(), g->ej.as<int>(), g->nptr.as<int>(), g->nedge.as<int>()};
    double* vec = g->vec.as<double>();
    const size_t m = (size_t)6 * n;
    const Sys S{n, E, g->esum.as<double>(), g->epairs.as<unsigned>(), g->fixed.as<int>(), g->Hd.as<double>(), g->Lc.as<double>(), vec, g->fr.as<int>(),
                vec + m, vec + 2 * m, vec + 3 * m, vec + 4 * m, vec + 5 * m, g->st.as<GoState>()};
    GoState* dst = g->st.as<GoState>();
    if (int rc = mark(g, -1)) return rc;
    for (int it = 0; it <= (int)g->p.nonlin_iters; ++it) {
      const bool last = it == (int)g->p.nonlin_iters;
      for (int e0 = 0; e0 < ne; e0 += kEdgeChunk) {
        const int nc = std::min(kEdgeChunk, ne - e0);
        go_linearise<<<dim3(nc, slots), kCta, 0, st>>>(g->L, th, E, e0, g->d_D.as<double>(), g->V.as<float4>(), g->N.as<float4>(),
                                                       g->part.as<double>(), g->part_n.as<unsigned>());
        go_edge_sums<<<grid(nc), kCta, 0, st>>>(nc, e0, slots, g->part.as<double>(), g->part_n.as<unsigned>(), g->esum.as<double>(),
                                                g->epairs.as<unsigned>());
      }
      go_totals<<<1, 1, 0, st>>>(ne, it, g->esum.as<double>(), g->epairs.as<unsigned>(), dst);
      if (last) {
        go_verify<<<1, 1, 0, st>>>(ne, (double)g->p.verify_thresh, g->esum.as<double>(), g->epairs.as<unsigned>(), dst);
        SCN_CUDA_TRY(cudaGetLastError());
        if (int rc = mark(g, PH_VERIFY)) return rc;
        break;
      }
      SCN_CUDA_TRY(cudaGetLastError());
      if (int rc = mark(g, PH_LINEARISE)) return rc;
      go_assemble<<<grid(n), kCta, 0, st>>>(S, it);
      go_pcg<<<1, kPcgThreads, 0, st>>>(S, it, (int)g->p.lin_iters);
      go_update<<<grid(n), kCta, 0, st>>>(S, g->d_D.as<double>());
      SCN_CUDA_TRY(cudaGetLastError());
      if (int rc = mark(g, PH_PCG)) return rc;
    }
    SCN_CUDA_TRY(cudaMemcpyAsync(&hs, g->st.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    if (int rc = collect(g)) return rc;
    ++rep.solves;
    rep.nonlin_iterations += g->p.nonlin_iters;
    rep.lin_iterations += hs.lin_run;
    if (first) { rep.rss_before = hs.rss_iter[0]; rep.pairs_before = hs.pairs_iter[0]; }
    first = false;
    rep.rss_after = hs.rss_iter[g->p.nonlin_iters]; rep.pairs_after = hs.pairs_iter[g->p.nonlin_iters];
    for (uint32_t it = 0; it < g->p.nonlin_iters; ++it) rep.rss_iter[it] = hs.rss_iter[it];
    rep.max_edge_rms = hs.max_rms;
    if (hs.nonfinite) { rep.rejected = 1; break; }
    if (hs.worst < 0) break;
    if (rep.edges_removed >= g->p.max_removed) { rep.rejected = 1; break; }
    active[act[hs.worst]] = 0;
    ++rep.edges_removed;
  }
  // the last solve's edges and poses
  if (ne_all) {
    const int ne = (int)act.size();
    std::vector<double> es((size_t)ne * kNSum);
    std::vector<unsigned> ep(ne);
    if (ne) {
      SCN_CUDA_TRY(cudaMemcpyAsync(es.data(), g->esum.p, es.size() * 8, cudaMemcpyDeviceToHost, st));
      SCN_CUDA_TRY(cudaMemcpyAsync(ep.data(), g->epairs.p, ep.size() * 4, cudaMemcpyDeviceToHost, st));
    }
    SCN_CUDA_TRY(cudaMemcpyAsync(D.data(), g->d_D.p, sizeof(double) * 12 * n, cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    for (int e = 0; e < ne_all; ++e) g->edges[e].removed = !active[e];
    for (int a = 0; a < ne; ++a) {
      scn_globalopt_edge_t& e = g->edges[act[a]];
      e.pairs = ep[a]; e.rss = es[(size_t)a * kNSum + 27];
      e.rms = e.pairs ? std::sqrt(e.rss / (double)e.pairs) : 0.0;
    }
  }
  rep.rms_before = rep.pairs_before ? std::sqrt(rep.rss_before / (double)rep.pairs_before) : 0.0;
  rep.rms_after = rep.pairs_after ? std::sqrt(rep.rss_after / (double)rep.pairs_after) : 0.0;
  for (int k = 0; k < n; ++k) {
    const double* P = rep.rejected ? g->D0.data() + 12 * k : D.data() + 12 * k;
    for (int q = 0; q < 12; ++q) poses_out[16 * k + q] = (float)P[q];
    poses_out[16 * k + 12] = 0.f; poses_out[16 * k + 13] = 0.f; poses_out[16 * k + 14] = 0.f; poses_out[16 * k + 15] = 1.f;
  }
  rep.keyframe_maps_ms = g->phase_ms[PH_MAPS];
  rep.overlap_ms = g->phase_ms[PH_OVERLAP]; rep.linearise_ms = g->phase_ms[PH_LINEARISE]; rep.pcg_ms = g->phase_ms[PH_PCG];
  rep.verify_ms = g->phase_ms[PH_VERIFY];
  if (report) *report = rep;
  return SCN_OK;
}

int scn_globalopt_edges(const scn_globalopt* g, scn_globalopt_edge_t* out, uint32_t cap, uint32_t* n) {
  if (!g || !n || (cap && !out)) return scn::fail(SCN_ERR_ARG, "null argument");
  *n = (uint32_t)g->edges.size();
  for (uint32_t e = 0; e < std::min<uint32_t>(cap, *n); ++e) out[e] = g->edges[e];
  return SCN_OK;
}

}  // extern "C"
