// Frame-to-model ICP camera tracking (DESIGN.md §6j, "tracking spec v1"): the tracker of the `recons` stage.  Not BundleFusion's
// trajectory (no features, no global optimisation): a dense point-to-plane ICP of the kind VoxelHashing's DepthSensing runs,
// against a raycast of the hashed TSDF volume, in the binary32 / binary64 operations and order of oracle/track_oracle.c (the
// library is built with -fmad=false: no contraction), so that poses, counters and the volume compare bit for bit.
//
// Per frame, on the volume's stream and without a host round trip inside the ICP:
//   depth -> metres (-inf invalid) -> bilateral filter (filter.cu, when the volume filters) -> range test -> 2x2 reductions to the
//   tracking resolution and two coarser levels -> vertex + normal maps;
//   per iteration one k_icp launch: association + the 28 exact binary64 products per pixel, a fixed tree per CTA into its slot, and
//   the last CTA to finish adds the slots in slot order and solves the 6x6 system (Cholesky, binary64) and applies the Cayley update;
//   k_finish composes the pose; one 104-byte copy to the host; the frame goes into the volume through scn_tsdf_integrate_device;
//   k_raycast + reductions + vertex / normal maps give the model of the next frame.
#include <cmath>

#include "icp_common.cuh"
#include "tsdf_internal.cuh"

using namespace scn_tsdf_detail;

namespace {

constexpr int kLevels = 3;
constexpr int kIters[kLevels] = {4, 5, 10};        // finest (0) to coarsest (2)
constexpr double kExitStep = 1e-5;
constexpr double kMaxRms = 0.02;

struct State {                                     // device; one frame's ICP
  double D[12];                                    // current estimate: frame camera -> model camera, 3x4
  float Df[12];
  int level_done[kLevels];
  int lost;
  unsigned iters[kLevels];
  unsigned pairs, valid, ticket;
  double rss;
};

struct Pose { float T[16]; };

// ---------------------------------------------------------------------------------------------------------------- raycast
__device__ __forceinline__ float lerpf(float p, float q, float a) { return __fadd_rn(__fmul_rn(p, __fsub_rn(1.0f, a)), __fmul_rn(q, a)); }

__device__ __forceinline__ bool sample_sdf(const Tables& tb, const float g[3], float& f) {
#pragma unroll
  for (int i = 0; i < 3; ++i) if (!(fabsf(g[i]) < 8388608.0f)) return false;
  const float fl[3] = {floorf(g[0]), floorf(g[1]), floorf(g[2])};
  const int b[3] = {(int)fl[0], (int)fl[1], (int)fl[2]};
  const float a[3] = {__fsub_rn(g[0], fl[0]), __fsub_rn(g[1], fl[1]), __fsub_rn(g[2], fl[2])};
  const int bx = b[0] >> 3, by = b[1] >> 3, bz = b[2] >> 3;
  const int home = lookup_block(tb, bx, by, bz);
  if (home < 0) return false;
  float c[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int x = b[0] + (k & 1), y = b[1] + ((k >> 1) & 1), z = b[2] + (k >> 2);
    const int blk = ((x >> 3) == bx && (y >> 3) == by && (z >> 3) == bz) ? home : lookup_block(tb, x >> 3, y >> 3, z >> 3);
    if (blk < 0) return false;
    const uint2 v = tb.heap[(size_t)blk * 512 + ((x & 7) | ((y & 7) << 3) | ((z & 7) << 6))];
    if ((v.y >> 24) == 0) return false;
    c[k] = __uint_as_float(v.x);
  }
  const float e0 = lerpf(c[0], c[1], a[0]), e1 = lerpf(c[2], c[3], a[0]), e2 = lerpf(c[4], c[5], a[0]), e3 = lerpf(c[6], c[7], a[0]);
  f = lerpf(lerpf(e0, e1, a[1]), lerpf(e2, e3, a[1]), a[2]);
  return true;
}

__global__ void k_raycast(const Level l, const Tables tb, const Pose P, float dmin, float step, float t_end, float inv_vs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= l.W * l.H) return;
  const int x = i % l.W, y = i / l.W;
  const float* T = P.T;
  const float rx = __fmul_rn(__fsub_rn((float)x, l.cx), l.ifx), ry = __fmul_rn(__fsub_rn((float)y, l.cy), l.ify);
  float res = -INFINITY, tp = 0.f, fp = 0.f;
  bool prev = false;
  for (int s = 0;; ++s) {
    const float tc = __fadd_rn(dmin, __fmul_rn((float)s, step));
    if (!(tc <= t_end)) break;
    const float pc[3] = {__fmul_rn(rx, tc), __fmul_rn(ry, tc), tc};
    float g[3], f = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      g[k] = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * k], pc[0]), __fmul_rn(T[4 * k + 1], pc[1])), __fmul_rn(T[4 * k + 2], pc[2])), T[4 * k + 3]), inv_vs);
    const bool ok = sample_sdf(tb, g, f);
    if (ok && prev && fp > 0.f && f < 0.f) { res = __fadd_rn(tp, __fmul_rn(__fsub_rn(tc, tp), __fdiv_rn(fp, __fsub_rn(fp, f)))); break; }
    prev = ok; tp = tc; fp = f;
  }
  l.mdepth[i] = res;
}

// ---------------------------------------------------------------------------------------------------------------- ICP
__device__ bool pair_terms(const Level& l, const Thresh th, const float* Df, int i, double* out) {
#pragma unroll
  for (int k = 0; k < kNSum; ++k) out[k] = 0.0;
  Assoc a;
  if (!associate(l, l.mv, l.mn, th, Df, l.v[i], l.n[i], a)) return false;
  const float4 nq = a.nq;
  const float J[6] = {__fsub_rn(__fmul_rn(a.ty, nq.z), __fmul_rn(a.tz, nq.y)), __fsub_rn(__fmul_rn(a.tz, nq.x), __fmul_rn(a.tx, nq.z)),
                      __fsub_rn(__fmul_rn(a.tx, nq.y), __fmul_rn(a.ty, nq.x)), nq.x, nq.y, nq.z};
  products28(J, a.r, out);
  return true;
}



// One Gauss-Newton iteration at level k.  Slot c = the 256 pixels [256c, 256c + 256): warps of 32 by a halving tree, the 8 warp sums
// by a halving tree; the last CTA adds the slots in slot order and solves.
__global__ void __launch_bounds__(kCta) k_icp(const Level l, int k, const Thresh th, State* st, double* __restrict__ part, unsigned* __restrict__ part_n) {
  __shared__ double s_w[kCta / 32][kNSum];
  __shared__ double s_sum[kNSum];
  __shared__ unsigned s_pairs;
  __shared__ bool s_last;
  if (st->lost || st->level_done[k]) return;                     // written by an earlier launch: the same for every thread
  float Df[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) Df[i] = st->Df[i];
  const int i = blockIdx.x * kCta + threadIdx.x;
  double v[kNSum];
  bool paired = false;
  if (i < l.W * l.H) paired = pair_terms(l, th, Df, i, v);
  else {
#pragma unroll
    for (int q = 0; q < kNSum; ++q) v[q] = 0.0;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < kNSum; ++q) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v[q] = __dadd_rn(v[q], __shfl_down_sync(0xffffffffu, v[q], s));
    if (lane == 0) s_w[warp][q] = v[q];
  }
  const unsigned cnt = __syncthreads_count(paired);
  if (threadIdx.x < kNSum) {
    double a[8];
#pragma unroll
    for (int w = 0; w < 8; ++w) a[w] = s_w[w][threadIdx.x];
#pragma unroll
    for (int s = 4; s > 0; s >>= 1)
#pragma unroll
      for (int t = 0; t < s; ++t) a[t] = __dadd_rn(a[t], a[t + s]);
    part[(size_t)blockIdx.x * kNSum + threadIdx.x] = a[0];
  }
  if (threadIdx.x == 0) part_n[blockIdx.x] = cnt;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x < kNSum) {
    double s = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) s = __dadd_rn(s, __ldcg(part + (size_t)c * kNSum + threadIdx.x));
    s_sum[threadIdx.x] = s;
  } else if (threadIdx.x == kNSum) {
    unsigned n = 0;
    for (unsigned c = 0; c < gridDim.x; ++c) n += __ldcg(part_n + c);
    s_pairs = n;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  st->ticket = 0;
  st->iters[k]++;
  st->pairs = s_pairs; st->rss = s_sum[27];
  double x[6];
  if (s_pairs < kMinPairs || !solve6(s_sum, s_pairs, x)) { st->lost = 1; return; }
  apply_update(st->D, x);
  for (int q = 0; q < 12; ++q) st->Df[q] = (float)st->D[q];
  double mx = 0.0;
  for (int q = 0; q < 6; ++q) mx = fmax(mx, fabs(x[q]));
  if (mx < kExitStep) st->level_done[k] = 1;
}

// pose of a tracked frame = ref * D, rounded once; the loss rule
__global__ void k_finish(const State* st, const Pose ref, scn_track_frame_t* out) {
  scn_track_frame_t r;
  memset(&r, 0, sizeof(r));
  for (int k = 0; k < kLevels; ++k) r.iterations[k] = st->iters[k];
  r.pairs = st->pairs; r.valid_pixels = st->valid; r.residual_ss = st->rss;
  r.rms = r.pairs ? __dsqrt_rn(__ddiv_rn(r.residual_ss, (double)r.pairs)) : 0.0;
  bool lost = st->lost != 0;
  if (!lost && ((unsigned long long)r.pairs * 4 < r.valid_pixels || r.rms > kMaxRms)) lost = true;
  if (lost) {
    r.lost = 1;
    for (int i = 0; i < 16; ++i) r.cam2world[i] = -INFINITY;
  } else {
    const double* D = st->D;
    for (int i = 0; i < 3; ++i) {
      const double r0 = ref.T[4 * i], r1 = ref.T[4 * i + 1], r2 = ref.T[4 * i + 2];
      for (int j = 0; j < 3; ++j) r.cam2world[4 * i + j] = (float)__dadd_rn(__dadd_rn(__dmul_rn(r0, D[j]), __dmul_rn(r1, D[4 + j])), __dmul_rn(r2, D[8 + j]));
      r.cam2world[4 * i + 3] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, D[3]), __dmul_rn(r1, D[7])), __dmul_rn(r2, D[11])), (double)ref.T[4 * i + 3]);
    }
    r.cam2world[12] = 0.f; r.cam2world[13] = 0.f; r.cam2world[14] = 0.f; r.cam2world[15] = 1.f;
  }
  *out = r;
}

__global__ void k_reset_state(State* st) {
  const double I[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  for (int i = 0; i < 12; ++i) { st->D[i] = I[i]; st->Df[i] = (float)I[i]; }
  for (int k = 0; k < kLevels; ++k) { st->level_done[k] = 0; st->iters[k] = 0; }
  st->lost = 0; st->pairs = 0; st->valid = 0; st->ticket = 0; st->rss = 0.0;
}

}  // namespace

struct scn_track {
  scn_track_params p{};
  scn_tsdf* vol = nullptr;
  int s = 0;                                       // depth resolution = tracking resolution * 2^s
  Level L[kLevels]{};
  scn::DBuf raw, metres, full, chain, lv[kLevels * 6], state, part, part_n, out;
  std::vector<float*> chain_ptr;                   // the reductions between the depth resolution and level 0
  bool have_model = false;
  Pose ref{};
  uint64_t frames = 0, launches = 0;
  scn::EventPtr ev[2][5];                          // per frame: start, frame maps, pose, integrated, model maps (two frames in flight)
  bool ev_pending[2] = {false, false};
  int ev_set = 0;
  double phase_ms[4] = {0, 0, 0, 0};               // frame maps, ICP + pose, integration, raycast + model maps
};

namespace {

unsigned grid(int n) { return (unsigned)((n + kCta - 1) / kCta); }

// adds the phase times of event set e, whose frame has completed
int collect_phases(scn_track* t, int e) {
  if (!t->ev_pending[e]) return SCN_OK;
  for (int k = 0; k < 4; ++k) {
    float ms = 0.f;
    SCN_CUDA_TRY(cudaEventElapsedTime(&ms, t->ev[e][k].get(), t->ev[e][k + 1].get()));
    t->phase_ms[k] += ms;
  }
  t->ev_pending[e] = false;
  return SCN_OK;
}

// frame maps of every level; the valid pixels of level 0 are counted into st->valid
int frame_maps(scn_track* t, const uint16_t* d_depth, const float K[16]) {
  scn_tsdf* v = t->vol;
  const cudaStream_t st = v->stream;
  const int W = (int)v->p.width, H = (int)v->p.height;
  if (int rc = scn_depth_to_metres_device(d_depth, W, H, v->p.depth_shift, v->p.depth_filter != 0, v->p.depth_sigma_d, v->p.depth_sigma_r,
                                          t->raw.as<float>(), t->metres.as<float>(), st))
    return rc;
  t->launches += v->p.depth_filter ? 2 : 1;
  k_range<<<grid(W * H), kCta, 0, st>>>(t->metres.as<float>(), W * H, v->p.depth_min, v->p.depth_max, t->full.as<float>());
  const float* src = t->full.as<float>();
  for (int k = 0; k < t->s; ++k) {
    float* dst = k + 1 == t->s ? t->L[0].depth : t->chain_ptr[k];
    k_reduce2<<<grid((W >> (k + 1)) * (H >> (k + 1))), kCta, 0, st>>>(src, W >> k, H >> k, dst);
    src = dst;
  }
  if (t->s == 0) SCN_CUDA_TRY(cudaMemcpyAsync(t->L[0].depth, src, (size_t)W * H * 4, cudaMemcpyDeviceToDevice, st));
  for (int k = 1; k < kLevels; ++k) k_reduce2<<<grid(t->L[k].W * t->L[k].H), kCta, 0, st>>>(t->L[k - 1].depth, t->L[k - 1].W, t->L[k - 1].H, t->L[k].depth);
  for (int k = 0; k < kLevels; ++k) {
    Level& l = t->L[k];
    level_intrinsics(l, K, t->s + k);
    k_vertex_normal<<<grid(l.W * l.H), kCta, 0, st>>>(l, l.depth, l.v, l.n, k == 0 ? &t->state.as<State>()->valid : nullptr);
  }
  t->launches += 1 + t->s + (kLevels - 1) + kLevels;
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

int model_maps(scn_track* t, const Pose& P) {
  scn_tsdf* v = t->vol;
  const cudaStream_t st = v->stream;
  Level& l0 = t->L[0];
  volatile float step = t->p.ray_increment_factor * v->p.trunc_base;
  const float t_end = std::fmin(v->p.depth_max, v->p.max_integration_distance);
  volatile float inv_vs = 1.0f / v->p.voxel_size;
  k_raycast<<<grid(l0.W * l0.H), kCta, 0, st>>>(l0, v->tb, P, v->p.depth_min, step, t_end, inv_vs);
  for (int k = 1; k < kLevels; ++k) k_reduce2<<<grid(t->L[k].W * t->L[k].H), kCta, 0, st>>>(t->L[k - 1].mdepth, t->L[k - 1].W, t->L[k - 1].H, t->L[k].mdepth);
  for (int k = 0; k < kLevels; ++k) k_vertex_normal<<<grid(t->L[k].W * t->L[k].H), kCta, 0, st>>>(t->L[k], t->L[k].mdepth, t->L[k].mv, t->L[k].mn, nullptr);
  t->launches += 1 + (kLevels - 1) + kLevels;
  SCN_CUDA_TRY(cudaGetLastError());
  return SCN_OK;
}

}  // namespace

extern "C" {

void scn_track_default_params(scn_track_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->width = 320; p->height = 240;                 // s_rayCastWidth / Height, zParametersScanNet.txt:22-23
  p->dist_thresh = 0.15f;                          // s_projCorrDistThres, zParametersBundlingScanNet.txt:55
  p->normal_thresh = 0.95f;                        // s_projCorrNormalThres, :56
  p->ray_increment_factor = 0.8f;                  // s_SDFRayIncrementFactor, zParametersScanNet.txt:61
}

int scn_track_params_from_file(const char* path, scn_track_params* p) {
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
    if (!strcmp(key, "s_rayCastWidth")) p->width = (uint32_t)v;
    else if (!strcmp(key, "s_rayCastHeight")) p->height = (uint32_t)v;
    else if (!strcmp(key, "s_projCorrDistThres")) p->dist_thresh = (float)v;
    else if (!strcmp(key, "s_projCorrNormalThres")) p->normal_thresh = (float)v;
    else if (!strcmp(key, "s_SDFRayIncrementFactor")) p->ray_increment_factor = (float)v;
  }
  fclose(f);
  return SCN_OK;
}

size_t scn_track_frame_sizeof(void) { return sizeof(scn_track_frame_t); }

int scn_track_create(scn_tsdf* vol, const scn_track_params* p, scn_track** out) {
  if (!vol || !p || !out) return scn::fail(SCN_ERR_ARG, "null argument");
  const uint32_t W = vol->p.width, H = vol->p.height;
  int s = 0;
  while (s < 16 && (W >> s) > p->width) ++s;
  if (!p->width || !p->height || (W >> s) != p->width || W % p->width || H % p->height || H / p->height != W / p->width)
    return scn::fail(SCN_ERR_ARG, "tracking resolution %ux%u is not the depth resolution %ux%u divided by a power of two", p->width, p->height, W, H);
  if ((p->width >> (kLevels - 1)) < 3 || (p->height >> (kLevels - 1)) < 3)
    return scn::fail(SCN_ERR_ARG, "tracking resolution %ux%u too small for %d levels", p->width, p->height, kLevels);
  if (!(p->dist_thresh > 0.f) || !(p->ray_increment_factor > 0.f) || !(vol->p.trunc_base > 0.f) || std::isnan(p->normal_thresh))
    return scn::fail(SCN_ERR_ARG, "invalid tracking parameters");
  SCN_CUDA_TRY(cudaSetDevice(vol->device));
  std::unique_ptr<scn_track> t(new scn_track());
  t->p = *p; t->vol = vol; t->s = s;
  const size_t px = (size_t)W * H;
  SCN_ALLOC(t->raw, px * 4); SCN_ALLOC(t->metres, px * 4); SCN_ALLOC(t->full, px * 4);
  size_t chain = 0;
  for (int k = 1; k < s; ++k) chain += (size_t)(W >> k) * (H >> k);
  SCN_ALLOC(t->chain, chain * 4);
  for (int k = 1, off = 0; k < s; ++k) { t->chain_ptr.push_back(t->chain.as<float>() + off); off += (W >> k) * (H >> k); }
  t->chain_ptr.push_back(nullptr);
  for (int k = 0; k < kLevels; ++k) {
    Level& l = t->L[k];
    l.W = (int)p->width >> k; l.H = (int)p->height >> k;
    const size_t n = (size_t)l.W * l.H;
    scn::DBuf* b = &t->lv[6 * k];
    SCN_ALLOC(b[0], n * 4); SCN_ALLOC(b[1], n * 16); SCN_ALLOC(b[2], n * 16);
    SCN_ALLOC(b[3], n * 4); SCN_ALLOC(b[4], n * 16); SCN_ALLOC(b[5], n * 16);
    l.depth = b[0].as<float>(); l.v = b[1].as<float4>(); l.n = b[2].as<float4>();
    l.mdepth = b[3].as<float>(); l.mv = b[4].as<float4>(); l.mn = b[5].as<float4>();
  }
  SCN_ALLOC(t->state, sizeof(State));
  SCN_ALLOC(t->part, (size_t)grid(t->L[0].W * t->L[0].H) * kNSum * 8);
  SCN_ALLOC(t->part_n, (size_t)grid(t->L[0].W * t->L[0].H) * 4);
  SCN_ALLOC(t->out, sizeof(scn_track_frame_t));
  for (auto& set : t->ev) for (auto& e : set) SCN_CUDA_TRY(scn::create(e));
  *out = t.release();
  return SCN_OK;
}

void scn_track_destroy(scn_track* t) {
  if (!t) return;
  cudaSetDevice(t->vol->device);
  cudaStreamSynchronize(t->vol->stream);
  delete t;
}

int scn_track_frames(scn_track* t, uint32_t n, const uint16_t* d_depth, const uint8_t* d_rgb, const float K[16], const float first_pose[16],
                     scn_track_frame_t* out) {
  if (!t || (n && (!d_depth || !K || !out)) || (!t->have_model && n && !first_pose)) return scn::fail(SCN_ERR_ARG, "null argument");
  scn_tsdf* v = t->vol;
  SCN_CUDA_TRY(cudaSetDevice(v->device));
  const cudaStream_t st = v->stream;
  const size_t px = (size_t)v->p.width * v->p.height;
  const Thresh th{t->p.dist_thresh * t->p.dist_thresh, t->p.normal_thresh};
  State* dst = t->state.as<State>();
  for (uint32_t f = 0; f < n; ++f) {
    const uint16_t* dd = d_depth + f * px;
    const uint8_t* dc = d_rgb ? d_rgb + f * px * 3 : nullptr;
    const int e = t->ev_set;
    if (int rc = collect_phases(t, e)) return rc;                  // recorded two frames ago, before the last synchronisation
    cudaEvent_t ev[5];
    for (int k = 0; k < 5; ++k) ev[k] = t->ev[e][k].get();
    SCN_CUDA_TRY(cudaEventRecord(ev[0], st));
    k_reset_state<<<1, 1, 0, st>>>(dst);
    ++t->launches;
    if (int rc = frame_maps(t, dd, K)) return rc;
    SCN_CUDA_TRY(cudaEventRecord(ev[1], st));
    scn_track_frame_t& r = out[f];
    if (!t->have_model) {
      k_finish<<<1, 1, 0, st>>>(dst, t->ref, t->out.as<scn_track_frame_t>());   // counters of the seed frame (valid pixels)
    } else {
      for (int k = kLevels - 1; k >= 0; --k) {
        const Level& l = t->L[k];
        for (int it = 0; it < kIters[k]; ++it)
          k_icp<<<grid(l.W * l.H), kCta, 0, st>>>(l, k, th, dst, t->part.as<double>(), t->part_n.as<unsigned>());
        t->launches += kIters[k];
      }
      k_finish<<<1, 1, 0, st>>>(dst, t->ref, t->out.as<scn_track_frame_t>());
    }
    ++t->launches;
    SCN_CUDA_TRY(cudaGetLastError());
    SCN_CUDA_TRY(cudaEventRecord(ev[2], st));
    SCN_CUDA_TRY(cudaMemcpyAsync(&r, t->out.p, sizeof(r), cudaMemcpyDeviceToHost, st));
    SCN_CUDA_TRY(cudaStreamSynchronize(st));
    if (!t->have_model) {
      // the seed: the first frame with at least kMinPairs valid pixels takes first_pose (identity when not finite); a frame before it
      // is lost, so that an empty first frame does not become a model nothing can track against
      const uint32_t valid = r.valid_pixels;
      memset(&r, 0, sizeof(r));
      r.valid_pixels = valid;
      bool finite = true;
      for (int i = 0; i < 16; ++i) finite = finite && std::isfinite(first_pose[i]);
      for (int i = 0; i < 16; ++i) r.cam2world[i] = valid < kMinPairs ? -INFINITY : finite ? first_pose[i] : (i % 5 == 0 ? 1.f : 0.f);
      r.lost = valid < kMinPairs ? 1u : 0u;
    }
    ++t->frames;
    if (!r.lost) {                                                  // a lost frame is not integrated; the next one tracks against the same model
      const uint64_t before = v->launches;
      if (int rc = scn_tsdf_integrate_device(v, 1, dd, dc, r.cam2world, K)) return rc;
      t->launches += v->launches - before;
    }
    SCN_CUDA_TRY(cudaEventRecord(ev[3], st));
    if (!r.lost) {
      Pose P;
      memcpy(P.T, r.cam2world, sizeof(P.T));
      if (int rc = model_maps(t, P)) return rc;
      t->ref = P;
      t->have_model = true;
    }
    SCN_CUDA_TRY(cudaEventRecord(ev[4], st));
    t->ev_pending[e] = true;
    t->ev_set ^= 1;
  }
  const int rc = scn_tsdf_sync(v);
  for (int e = 0; e < 2 && !rc; ++e) if (int q = collect_phases(t, e)) return q;
  return rc;
}

int scn_track_phase_ms(const scn_track* t, double* frame_maps_ms, double* icp_ms, double* integrate_ms, double* raycast_ms) {
  if (!t) return scn::fail(SCN_ERR_ARG, "null handle");
  double* o[4] = {frame_maps_ms, icp_ms, integrate_ms, raycast_ms};
  for (int k = 0; k < 4; ++k) if (o[k]) *o[k] = t->phase_ms[k];
  return SCN_OK;
}

int scn_track_stats(const scn_track* t, uint64_t* frames, uint64_t* kernel_launches) {
  if (!t) return scn::fail(SCN_ERR_ARG, "null handle");
  if (frames) *frames = t->frames;
  if (kernel_launches) *kernel_launches = t->launches;
  return SCN_OK;
}

}  // extern "C"
