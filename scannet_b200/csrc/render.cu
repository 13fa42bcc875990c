// Preview render on H100 (sm_90a): path-traced or ambient-occlusion images of a triangle mesh (DESIGN.md §6i, "render spec v1").
//
// Stands in for Server/mts_render.py (the `render` stage, `_vh_clean_2.ply` -> `_vh_clean_2.png`), which drives Mitsuba; Mitsuba
// is not in the reference tree, so the numerics are this repository's own spec and its scalar statement is
// oracle/render_oracle.c (test infrastructure, never linked here).  The camera comes from render_host.cpp.
//
// Every device operation is binary32 + - * / sqrt, round to nearest (the file is compiled with -fmad=false); what needs a
// transcendental (camera, sRGB tables, 2^exposure) is made on the host in binary64.
//
// Data layout in HBM:
//   tri4[3*leaf]   float4 v0 (w = face index), v1 (w = 1 when the face's normal is zero: never hit), v2, in leaf (Morton) order
//   leaf_rgb[leaf] uint4 the three vertex colours packed as r | g << 8 | b << 16 (w unused), present with vertex colours
//   nodes[i]       Node: the boxes of both children and their references (bit 31: a leaf), 64 B; node 0 is the root
//
// Kernels:
//   k_morton  per face: 30-bit Morton code of the centroid; (code, face) pairs are then sorted stably (radix_sort.cuh)
//   k_leaves  per leaf: the face's vertices copied into leaf order (exact copies), its box and colours
//   k_karras  per inner node: Karras (2012) radix-tree split of the sorted codes (face index breaks equal codes)
//   k_boxes   per leaf: climbs to the root; the second child to arrive at a node writes its boxes (min / max are exact)
//   k_trace   one thread per (view, pixel, sample); a CTA holds 256 / P pixels with P = the samples rounded up to a power of
//             two; per-thread stack traversal in local memory; the pixel sum is a fixed pairwise tree in shared memory, and
//             the pixel's thread writes the RGBA bytes.
#include <algorithm>
#include <cmath>
#include <vector>

#include "radix_sort.cuh"
#include "scn_common.h"

namespace {

constexpr int kTraceThreads = 256;
constexpr int kStack = 64;                   // >= tree depth: Karras inner nodes nest by strictly longer (30 + 32)-bit prefixes
constexpr unsigned kLeafBit = 0x80000000u;
constexpr uint32_t kMaxSamples = 256, kMaxDepth = 64, kMaxSide = 16384;
constexpr float kCoordMax = 268435456.f;     // 2^28: normals and their squared lengths stay finite

struct Node { float4 a, b, c, d; };          // a = (llo.xyz, lhi.x), b = (lhi.yz, rlo.xy), c = (rlo.z, rhi.xyz), d = (lref, rref, -, -)

struct Consts {
  float lin[256];                            // sRGB byte -> linear reflectance
  float thr[256];                            // thr[k] (k < 255): the linear value whose sRGB encoding is (k + 1/2) / 255
  float scale;                               // 2^exposure
  uint32_t W, H, spp, P, max_depth, n_views;
  int integrator, has_rgb;
  unsigned root;
};

// ------------------------------------------------------------------------------ spec arithmetic (device)
__device__ __forceinline__ float mnf(float a, float b) { return a < b ? a : b; }
__device__ __forceinline__ float mxf(float a, float b) { return a > b ? a : b; }

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ float unit(uint32_t h, uint32_t dim) { return (float)(mix32(h ^ dim) >> 8) * 5.9604644775390625e-8f; }

struct Ray {
  float o[3], d[3];
  float S[3];                                // Sx, Sy, Sz of the watertight test
  float okx, oky, okz;                       // o[kx], o[ky], o[kz]
  int kx, ky, kz;
};

__device__ __forceinline__ float sel(float x, float y, float z, int k) { return k == 0 ? x : (k == 1 ? y : z); }

__device__ __forceinline__ void ray_prep(Ray& r) {
  const float ax = fabsf(r.d[0]), ay = fabsf(r.d[1]), az = fabsf(r.d[2]);
  r.kz = ax >= ay ? (ax >= az ? 0 : 2) : (ay >= az ? 1 : 2);
  r.kx = r.kz == 2 ? 0 : r.kz + 1;
  r.ky = r.kx == 2 ? 0 : r.kx + 1;
  const float dkx = sel(r.d[0], r.d[1], r.d[2], r.kx), dky = sel(r.d[0], r.d[1], r.d[2], r.ky), dkz = sel(r.d[0], r.d[1], r.d[2], r.kz);
  r.S[0] = dkx / dkz; r.S[1] = dky / dkz; r.S[2] = 1.0f / dkz;
  r.okx = sel(r.o[0], r.o[1], r.o[2], r.kx); r.oky = sel(r.o[0], r.o[1], r.o[2], r.ky); r.okz = sel(r.o[0], r.o[1], r.o[2], r.kz);
}

__device__ __forceinline__ float comp(const float4& v, int k) { return sel(v.x, v.y, v.z, k); }

// The watertight ray-triangle test with the bounding-box clause and the clamp of spec §6i.  Returns false for a miss,
// else t and (U, V, W, det).
__device__ __forceinline__ bool tri_test(const Ray& r, const float4& v0, const float4& v1, const float4& v2, float& t, float& U, float& V,
                                         float& W, float& det) {
  const float Akx = comp(v0, r.kx) - r.okx, Aky = comp(v0, r.ky) - r.oky, Akz = comp(v0, r.kz) - r.okz;
  const float Bkx = comp(v1, r.kx) - r.okx, Bky = comp(v1, r.ky) - r.oky, Bkz = comp(v1, r.kz) - r.okz;
  const float Ckx = comp(v2, r.kx) - r.okx, Cky = comp(v2, r.ky) - r.oky, Ckz = comp(v2, r.kz) - r.okz;
  const float Ax = Akx - r.S[0] * Akz, Ay = Aky - r.S[1] * Akz;
  const float Bx = Bkx - r.S[0] * Bkz, By = Bky - r.S[1] * Bkz;
  const float Cx = Ckx - r.S[0] * Ckz, Cy = Cky - r.S[1] * Ckz;
  if (mnf(mnf(Ax, Bx), Cx) > 0.f || mxf(mxf(Ax, Bx), Cx) < 0.f || mnf(mnf(Ay, By), Cy) > 0.f || mxf(mxf(Ay, By), Cy) < 0.f) return false;
  U = Cx * By - Cy * Bx;
  V = Ax * Cy - Ay * Cx;
  W = Bx * Ay - By * Ax;
  if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) return false;
  det = (U + V) + W;
  if (det == 0.f) return false;
  const float Az = r.S[2] * Akz, Bz = r.S[2] * Bkz, Cz = r.S[2] * Ckz;
  const float T = (U * Az + V * Bz) + W * Cz;
  t = mxf(T / det, mnf(mnf(Az, Bz), Cz));
  t = mnf(t, mxf(mxf(Az, Bz), Cz));
  return true;
}

// Conservative box test in the triangle test's own sheared arithmetic: every operation is monotone in each vertex
// coordinate, so the box corners bound what any vertex inside gives (DESIGN.md §6i, "the cull").  best / tmin as in trace().
__device__ __forceinline__ bool box_test(const Ray& r, const float lo[3], const float hi[3], float tmin, float best, float& zmin) {
  const float lkx = sel(lo[0], lo[1], lo[2], r.kx) - r.okx, hkx = sel(hi[0], hi[1], hi[2], r.kx) - r.okx;
  const float lky = sel(lo[0], lo[1], lo[2], r.ky) - r.oky, hky = sel(hi[0], hi[1], hi[2], r.ky) - r.oky;
  const float lkz = sel(lo[0], lo[1], lo[2], r.kz) - r.okz, hkz = sel(hi[0], hi[1], hi[2], r.kz) - r.okz;
  const float gx0 = r.S[0] * lkz, gx1 = r.S[0] * hkz, gy0 = r.S[1] * lkz, gy1 = r.S[1] * hkz;
  if (lkx - mxf(gx0, gx1) > 0.f || hkx - mnf(gx0, gx1) < 0.f) return false;
  if (lky - mxf(gy0, gy1) > 0.f || hky - mnf(gy0, gy1) < 0.f) return false;
  const float z0 = r.S[2] * lkz, z1 = r.S[2] * hkz;
  zmin = mnf(z0, z1);
  return zmin <= best && mxf(z0, z1) > tmin;
}

// Closest hit with tmin < t <= tmax, smallest t then smallest face index, ignoring face `skip`.  Returns the leaf or -1.
__device__ int trace(const Ray& r, float tmin, float tmax, unsigned skip, const Node* __restrict__ nodes, const float4* __restrict__ tri4,
                     unsigned root, float& best_t, unsigned& n_nodes, unsigned& n_tris) {
  best_t = tmax;
  unsigned best_face = 0xffffffffu;
  int best_leaf = -1;
  unsigned stack[kStack];
  int sp = 0;
  unsigned cur = root;
  for (;;) {
    if (cur & kLeafBit) {
      const unsigned leaf = cur & ~kLeafBit;
      const float4 v0 = __ldg(tri4 + 3 * leaf), v1 = __ldg(tri4 + 3 * leaf + 1), v2 = __ldg(tri4 + 3 * leaf + 2);
      const unsigned face = __float_as_uint(v0.w);
      if (face != skip && __float_as_uint(v1.w) == 0u) {
        ++n_tris;
        float t, U, V, W, det;
        if (tri_test(r, v0, v1, v2, t, U, V, W, det) && t > tmin && (t < best_t || (t == best_t && face < best_face))) {
          best_t = t; best_face = face; best_leaf = (int)leaf;
        }
      }
    } else {
      ++n_nodes;
      const Node nd = nodes[cur];
      const float llo[3] = {nd.a.x, nd.a.y, nd.a.z}, lhi[3] = {nd.a.w, nd.b.x, nd.b.y};
      const float rlo[3] = {nd.b.z, nd.b.w, nd.c.x}, rhi[3] = {nd.c.y, nd.c.z, nd.c.w};
      float zl = 0.f, zr = 0.f;
      const bool hl = box_test(r, llo, lhi, tmin, best_t, zl), hr = box_test(r, rlo, rhi, tmin, best_t, zr);
      const unsigned cl = __float_as_uint(nd.d.x), cr = __float_as_uint(nd.d.y);
      if (hl && hr) {                        // nearer box first; the order changes the work, never the result
        const bool lfirst = zl <= zr;
        stack[sp++] = lfirst ? cr : cl;
        cur = lfirst ? cl : cr;
        continue;
      }
      if (hl) { cur = cl; continue; }
      if (hr) { cur = cr; continue; }
    }
    if (sp == 0) break;
    cur = stack[--sp];
  }
  return best_leaf;
}

// The recomputed test of the winning leaf: barycentric weights U/det, V/det, W/det
__device__ __forceinline__ void hit_weights(const Ray& r, const float4& v0, const float4& v1, const float4& v2, float b[3]) {
  float t, U, V, W, det;
  tri_test(r, v0, v1, v2, t, U, V, W, det);
  b[0] = U / det; b[1] = V / det; b[2] = W / det;
}

// Unit face normal turned against the incoming direction d
__device__ __forceinline__ void face_normal(const float4& v0, const float4& v1, const float4& v2, const float d[3], float n[3]) {
  const float e1[3] = {v1.x - v0.x, v1.y - v0.y, v1.z - v0.z}, e2[3] = {v2.x - v0.x, v2.y - v0.y, v2.z - v0.z};
  n[0] = e1[1] * e2[2] - e1[2] * e2[1];
  n[1] = e1[2] * e2[0] - e1[0] * e2[2];
  n[2] = e1[0] * e2[1] - e1[1] * e2[0];
  const float l = sqrtf((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  n[0] = n[0] / l; n[1] = n[1] / l; n[2] = n[2] / l;
  if ((n[0] * d[0] + n[1] * d[1]) + n[2] * d[2] > 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

// Cosine-weighted direction about n: normalize(n + s), s uniform on the sphere by rejection from the cube; try k draws dims
// 3k .. 3k+2 of hash h; 64 failed tries give n itself
__device__ __forceinline__ void cosine_dir(const float n[3], uint32_t h, float d[3]) {
  for (uint32_t k = 0; k < 64; ++k) {
    const float sx = 2.f * unit(h, 3 * k) - 1.f, sy = 2.f * unit(h, 3 * k + 1) - 1.f, sz = 2.f * unit(h, 3 * k + 2) - 1.f;
    const float q = (sx * sx + sy * sy) + sz * sz;
    if (q > 1.f || q < 9.5367431640625e-7f) continue;
    const float sl = sqrtf(q);
    const float w[3] = {n[0] + sx / sl, n[1] + sy / sl, n[2] + sz / sl};
    const float l2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2];
    if (l2 < 9.5367431640625e-7f) continue;
    const float l = sqrtf(l2);
    d[0] = w[0] / l; d[1] = w[1] / l; d[2] = w[2] / l;
    return;
  }
  d[0] = n[0]; d[1] = n[1]; d[2] = n[2];
}

// Reflectance at the hit: barycentric interpolation of the linear vertex colours, or 0.5 without colours
__device__ __forceinline__ void reflectance(const Consts& c, const float* s_lin, const uint4* __restrict__ leaf_rgb, int leaf, const float b[3],
                                            float rho[3]) {
  if (!c.has_rgb) { rho[0] = rho[1] = rho[2] = 0.5f; return; }
  const uint4 q = __ldg(leaf_rgb + leaf);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float c0 = s_lin[(q.x >> (8 * ch)) & 255u], c1 = s_lin[(q.y >> (8 * ch)) & 255u], c2 = s_lin[(q.z >> (8 * ch)) & 255u];
    rho[ch] = (b[0] * c0 + b[1] * c1) + b[2] * c2;
  }
}

__device__ __forceinline__ void hit_point(const Ray& r, float t, float p[3]) {
  p[0] = r.o[0] + t * r.d[0]; p[1] = r.o[1] + t * r.d[1]; p[2] = r.o[2] + t * r.d[2];
}

__global__ void __launch_bounds__(kTraceThreads)
k_trace(const __grid_constant__ Consts c, const scn_render_camera_t* __restrict__ cams, const Node* __restrict__ nodes,
        const float4* __restrict__ tri4, const uint4* __restrict__ leaf_rgb, uint8_t* __restrict__ rgba,
        unsigned long long* __restrict__ counters) {
  __shared__ float s_lin[256];
  __shared__ float s_thr[256];
  __shared__ float4 s_sum[kTraceThreads];
  s_lin[threadIdx.x] = c.lin[threadIdx.x];
  s_thr[threadIdx.x] = c.thr[threadIdx.x];
  __syncthreads();
  const unsigned P = c.P;
  const unsigned long long px_per_view = (unsigned long long)c.W * c.H;
  const unsigned long long gpix = (unsigned long long)blockIdx.x * (kTraceThreads / P) + threadIdx.x / P;
  const unsigned sample = threadIdx.x % P;
  const bool active = gpix < px_per_view * c.n_views && sample < c.spp;
  float L[3] = {0.f, 0.f, 0.f};
  float hit0 = 0.f;
  unsigned n_prim = 0, n_sec = 0, n_hit = 0, n_nodes = 0, n_tris = 0;
  if (active) {
    const unsigned view = (unsigned)(gpix / px_per_view);
    const unsigned pix = (unsigned)(gpix % px_per_view);
    const unsigned x = pix % c.W, y = pix / c.W;
    const scn_render_camera_t& cam = cams[view];
    const uint32_t hs = mix32(mix32(pix ^ 0x9e3779b9u) ^ sample);     // the view is not hashed: a view renders alike alone or in a batch
    const uint32_t h0 = mix32(hs);                                  // bounce 0
    const float fx = (float)x + unit(h0, 0), fy = (float)y + unit(h0, 1);
    Ray r;
#pragma unroll
    for (int i = 0; i < 3; ++i) { r.o[i] = cam.origin[i]; r.d[i] = (cam.p00[i] + fx * cam.du[i]) + fy * cam.dv[i]; }
    ray_prep(r);
    float t;
    int leaf = trace(r, cam.t_near, INFINITY, 0xffffffffu, nodes, tri4, c.root, t, n_nodes, n_tris);
    ++n_prim;
    if (leaf < 0) {
      L[0] = L[1] = L[2] = 1.f;
    } else {
      ++n_hit; hit0 = 1.f;
      float thr[3] = {1.f, 1.f, 1.f};
      for (uint32_t depth = 1;; ++depth) {
        const float4 v0 = __ldg(tri4 + 3 * leaf), v1 = __ldg(tri4 + 3 * leaf + 1), v2 = __ldg(tri4 + 3 * leaf + 2);
        const unsigned face = __float_as_uint(v0.w);
        if (c.integrator == SCN_RENDER_PATH) {
          float b[3], rho[3];
          hit_weights(r, v0, v1, v2, b);
          reflectance(c, s_lin, leaf_rgb, leaf, b, rho);
          thr[0] = thr[0] * rho[0]; thr[1] = thr[1] * rho[1]; thr[2] = thr[2] * rho[2];
          if (depth == c.max_depth) break;                          // L stays 0
        }
        float n[3], p[3];
        face_normal(v0, v1, v2, r.d, n);
        hit_point(r, t, p);
        Ray s;
#pragma unroll
        for (int i = 0; i < 3; ++i) s.o[i] = p[i];
        cosine_dir(n, mix32(hs ^ depth), s.d);
        ray_prep(s);
        const float tmax = c.integrator == SCN_RENDER_AO ? cam.ao_length : INFINITY;
        leaf = trace(s, cam.t_eps, tmax, face, nodes, tri4, c.root, t, n_nodes, n_tris);
        ++n_sec;
        if (leaf < 0) { L[0] = thr[0]; L[1] = thr[1]; L[2] = thr[2]; break; }
        if (c.integrator == SCN_RENDER_AO) break;                   // blocked: 0
        r = s;
      }
    }
  }
  // the pixel's samples, a fixed pairwise tree: for off = P/2 .. 1, s[i] += s[i + off] for i < off (samples >= spp are 0)
  s_sum[threadIdx.x] = make_float4(L[0], L[1], L[2], hit0);
  __syncthreads();
  for (unsigned off = P >> 1; off; off >>= 1) {
    if (sample < off) {
      const float4 a = s_sum[threadIdx.x], b = s_sum[threadIdx.x + off];
      s_sum[threadIdx.x] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    __syncthreads();
  }
  if (sample == 0 && gpix < px_per_view * c.n_views) {
    const float4 s = s_sum[threadIdx.x];
    const float sf = (float)c.spp;
    const float v[3] = {(s.x / sf) * c.scale, (s.y / sf) * c.scale, (s.z / sf) * c.scale};
    uint8_t out[4];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {                               // the number of thresholds <= v (thr is increasing)
      unsigned lo = 0, hi = 255;
      while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (s_thr[mid] <= v[ch]) lo = mid + 1; else hi = mid; }
      out[ch] = (uint8_t)lo;
    }
    const unsigned hits = (unsigned)s.w;                            // exact: a sum of at most 256 ones
    out[3] = (uint8_t)((510u * hits + c.spp) / (2u * c.spp));
    *reinterpret_cast<uchar4*>(rgba + 4 * gpix) = make_uchar4(out[0], out[1], out[2], out[3]);
  }
  const unsigned full = 0xffffffffu;
  n_prim = __reduce_add_sync(full, n_prim); n_sec = __reduce_add_sync(full, n_sec); n_hit = __reduce_add_sync(full, n_hit);
  n_nodes = __reduce_add_sync(full, n_nodes); n_tris = __reduce_add_sync(full, n_tris);
  if ((threadIdx.x & 31) == 0) {
    if (n_prim) atomicAdd(counters + 0, (unsigned long long)n_prim);
    if (n_sec) atomicAdd(counters + 1, (unsigned long long)n_sec);
    if (n_hit) atomicAdd(counters + 2, (unsigned long long)n_hit);
    if (n_nodes) atomicAdd(counters + 3, (unsigned long long)n_nodes);
    if (n_tris) atomicAdd(counters + 4, (unsigned long long)n_tris);
  }
}

// ------------------------------------------------------------------------------ BVH build
__device__ __forceinline__ unsigned spread10(unsigned v) {
  v = (v | (v << 16)) & 0x030000ffu; v = (v | (v << 8)) & 0x0300f00fu; v = (v | (v << 4)) & 0x030c30c3u; v = (v | (v << 2)) & 0x09249249u;
  return v;
}

// Morton code of the centroid's cell in a 1024^3 grid over the mesh box (the tree's shape only; no result depends on it)
__global__ void k_morton(const float* __restrict__ xyz, const uint32_t* __restrict__ tri, unsigned n, float3 lo, float3 inv,
                         unsigned* __restrict__ keys, unsigned* __restrict__ vals) {
  const unsigned f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const uint32_t a = tri[3 * f], b = tri[3 * f + 1], c = tri[3 * f + 2];
  unsigned q[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float m = (xyz[3 * a + k] + xyz[3 * b + k] + xyz[3 * c + k]) * (1.f / 3.f);
    const float s = (m - (&lo.x)[k]) * (&inv.x)[k];
    q[k] = (unsigned)fminf(fmaxf(s, 0.f), 1023.f);
  }
  keys[f] = (spread10(q[0]) << 2) | (spread10(q[1]) << 1) | spread10(q[2]);
  vals[f] = f;
}

__global__ void k_leaves(const float* __restrict__ xyz, const uint8_t* __restrict__ rgb, const uint32_t* __restrict__ tri,
                         const unsigned* __restrict__ order, unsigned n, float4* __restrict__ tri4, uint4* __restrict__ leaf_rgb,
                         float* __restrict__ leaf_box) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const unsigned f = order[k];
  const uint32_t id[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]};
  float v[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) v[j][i] = xyz[3 * (size_t)id[j] + i];
  const float e1[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]}, e2[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
  const float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
  const bool degenerate = !((nx * nx + ny * ny) + nz * nz > 0.f);
  tri4[3 * k] = make_float4(v[0][0], v[0][1], v[0][2], __uint_as_float(f));
  tri4[3 * k + 1] = make_float4(v[1][0], v[1][1], v[1][2], __uint_as_float(degenerate ? 1u : 0u));
  tri4[3 * k + 2] = make_float4(v[2][0], v[2][1], v[2][2], 0.f);
  if (rgb) {
    unsigned q[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) q[j] = rgb[3 * (size_t)id[j]] | (rgb[3 * (size_t)id[j] + 1] << 8) | (rgb[3 * (size_t)id[j] + 2] << 16);
    leaf_rgb[k] = make_uint4(q[0], q[1], q[2], 0u);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    leaf_box[6 * (size_t)k + i] = fminf(fminf(v[0][i], v[1][i]), v[2][i]);
    leaf_box[6 * (size_t)k + 3 + i] = fmaxf(fmaxf(v[0][i], v[1][i]), v[2][i]);
  }
}

// common-prefix length of sorted keys i and j over (code, index); -1 outside [0, n)
__device__ __forceinline__ int delta(const unsigned* __restrict__ code, int n, int i, int j) {
  if (j < 0 || j >= n) return -1;
  const unsigned a = code[i], b = code[j];
  return a == b ? 32 + __clz((unsigned)i ^ (unsigned)j) : __clz(a ^ b);
}

__global__ void k_karras(const unsigned* __restrict__ code, int n, Node* __restrict__ nodes, unsigned* __restrict__ parent_leaf,
                         unsigned* __restrict__ parent_inner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n - 1) return;
  const int d = delta(code, n, i, i + 1) - delta(code, n, i, i - 1) >= 0 ? 1 : -1;
  const int dmin = delta(code, n, i, i - d);
  int lmax = 2;
  while (delta(code, n, i, i + lmax * d) > dmin) lmax <<= 1;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (delta(code, n, i, i + (l + t) * d) > dmin) l += t;
  const int j = i + l * d;
  const int dnode = delta(code, n, i, j);
  int s = 0;
  for (int div = 2;; div <<= 1) {
    const int t = (l + div - 1) / div;
    if (delta(code, n, i, i + (s + t) * d) > dnode) s += t;
    if (t <= 1) break;
  }
  const int g = i + s * d + min(d, 0);
  const unsigned left = min(i, j) == g ? (kLeafBit | (unsigned)g) : (unsigned)g;
  const unsigned right = max(i, j) == g + 1 ? (kLeafBit | (unsigned)(g + 1)) : (unsigned)(g + 1);
  nodes[i].d = make_float4(__uint_as_float(left), __uint_as_float(right), 0.f, 0.f);
  if (left & kLeafBit) parent_leaf[g] = (unsigned)i; else parent_inner[g] = (unsigned)i;
  if (right & kLeafBit) parent_leaf[g + 1] = (unsigned)i; else parent_inner[g + 1] = (unsigned)i;
}

__device__ __forceinline__ void child_box(unsigned ref, const float* leaf_box, const float* inner_box, float b[6]) {
  const float* src = ref & kLeafBit ? leaf_box + 6 * (size_t)(ref & ~kLeafBit) : inner_box + 6 * (size_t)ref;
#pragma unroll
  for (int i = 0; i < 6; ++i) b[i] = __ldcg(src + i);
}

// Bottom-up boxes: each leaf climbs; at every inner node the first arrival stops and the second writes the node.
__global__ void k_boxes(int n, const unsigned* __restrict__ parent_leaf, const unsigned* __restrict__ parent_inner,
                        const float* __restrict__ leaf_box, float* inner_box, Node* nodes, unsigned* __restrict__ arrivals) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  unsigned p = parent_leaf[k];
  for (;;) {
    __threadfence();
    if (atomicAdd(arrivals + p, 1u) == 0u) return;
    __threadfence();
    const float4 dref = __ldcg(&nodes[p].d);
    float l[6], r[6];
    child_box(__float_as_uint(dref.x), leaf_box, inner_box, l);
    child_box(__float_as_uint(dref.y), leaf_box, inner_box, r);
    nodes[p].a = make_float4(l[0], l[1], l[2], l[3]);
    nodes[p].b = make_float4(l[4], l[5], r[0], r[1]);
    nodes[p].c = make_float4(r[2], r[3], r[4], r[5]);
#pragma unroll
    for (int i = 0; i < 3; ++i) { inner_box[6 * (size_t)p + i] = fminf(l[i], r[i]); inner_box[6 * (size_t)p + 3 + i] = fmaxf(l[3 + i], r[3 + i]); }
    if (p == 0) return;
    p = parent_inner[p];
  }
}

// ------------------------------------------------------------------------------ host
double srgb_decode(double x) { return x <= 0.04045 ? x / 12.92 : std::pow((x + 0.055) / 1.055, 2.4); }

int check_params(const scn_render_params* p) {
  if (!p) return scn::fail(SCN_ERR_ARG, "null params");
  if (p->width < 1 || p->height < 1 || p->width > kMaxSide || p->height > kMaxSide)
    return scn::fail(SCN_ERR_ARG, "film %ux%u: each side must be in 1 .. %u", p->width, p->height, kMaxSide);
  if (p->samples < 1 || p->samples > kMaxSamples) return scn::fail(SCN_ERR_ARG, "samples %u: must be in 1 .. %u", p->samples, kMaxSamples);
  if (p->integrator != SCN_RENDER_PATH && p->integrator != SCN_RENDER_AO) return scn::fail(SCN_ERR_ARG, "unknown integrator %d", p->integrator);
  if (p->max_depth < 1 || p->max_depth > kMaxDepth) return scn::fail(SCN_ERR_ARG, "max_depth %u: must be in 1 .. %u", p->max_depth, kMaxDepth);
  if (!std::isfinite(p->exposure) || std::fabs(p->exposure) > 64.f) return scn::fail(SCN_ERR_ARG, "exposure %g: must be finite, |e| <= 64", p->exposure);
  return SCN_OK;
}

}  // namespace

extern "C" {

void scn_render_default_params(scn_render_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->width = 640; p->height = 480;          // mts_render.py:145-150
  p->samples = 16;                          // :142
  p->integrator = SCN_RENDER_PATH;          // :139
  p->max_depth = 5;                         // no CLI flag in the script; DESIGN.md §6i
  p->exposure = 1.0f;                       // :157
  p->world_up[2] = 1.f;                     // :160
  p->camera_up[1] = 1.f;                    // :163
  p->bsphere_mult = 2.5f;                   // :169
}

size_t scn_render_report_sizeof(void) { return sizeof(scn_render_report_t); }

int scn_render_mesh(const float* xyz, const uint8_t* rgb, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                    const scn_render_params* params, const scn_render_camera_t* cams, uint32_t n_views, uint8_t* rgba_out,
                    scn_render_report_t* report) {
  const double t_start = scn::now_s();
  if (!xyz || !tri || !cams || !rgba_out) return scn::fail(SCN_ERR_ARG, "null argument");
  if (int rc = check_params(params)) return rc;
  if (n_faces == 0 || n_verts == 0) return scn::fail(SCN_ERR_ARG, "empty mesh (%llu vertices, %llu faces)", (unsigned long long)n_verts, (unsigned long long)n_faces);
  if (n_faces >= (1ull << 31) || n_verts >= (1ull << 32)) return scn::fail(SCN_ERR_ARG, "mesh too large (%llu faces)", (unsigned long long)n_faces);
  if (n_views == 0) return scn::fail(SCN_ERR_ARG, "no view");
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint64_t i = 0; i < 3 * n_verts; ++i) {
    const float v = xyz[i];
    if (!(std::fabs(v) <= kCoordMax)) return scn::fail(SCN_ERR_ARG, "vertex %llu: coordinate %g is not finite or exceeds 2^28", (unsigned long long)(i / 3), v);
    lo[i % 3] = std::min(lo[i % 3], v); hi[i % 3] = std::max(hi[i % 3], v);
  }
  for (uint64_t i = 0; i < 3 * n_faces; ++i)
    if (tri[i] >= n_verts) return scn::fail(SCN_ERR_ARG, "face %llu: vertex index %u >= %llu vertices", (unsigned long long)(i / 3), tri[i], (unsigned long long)n_verts);
  for (uint32_t v = 0; v < n_views; ++v) {
    const float* f = &cams[v].origin[0];
    for (int i = 0; i < (int)(sizeof(scn_render_camera_t) / 4); ++i)
      if (!std::isfinite(f[i])) return scn::fail(SCN_ERR_ARG, "camera %u: non-finite value", v);
  }
  const uint64_t px_per_view = (uint64_t)params->width * params->height, n_px = px_per_view * n_views;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { cudaGetLastError(); return scn::fail(SCN_ERR_CUDA, "no CUDA device"); }

  Consts c{};
  for (int k = 0; k < 256; ++k) c.lin[k] = (float)srgb_decode(k / 255.0);
  for (int k = 0; k < 255; ++k) c.thr[k] = (float)srgb_decode((k + 0.5) / 255.0);
  c.thr[255] = INFINITY;
  c.scale = (float)std::exp2((double)params->exposure);
  c.W = params->width; c.H = params->height; c.spp = params->samples; c.max_depth = params->max_depth; c.n_views = n_views;
  c.P = 1; while (c.P < c.spp) c.P <<= 1;
  c.integrator = params->integrator; c.has_rgb = rgb != nullptr;
  const unsigned n = (unsigned)n_faces;
  c.root = n == 1 ? kLeafBit : 0u;

  scn::StreamPtr stream;
  scn::EventPtr ev[5];
  SCN_CUDA_TRY(scn::create(stream, ev, 5));
  const cudaStream_t st = stream.get();
  scn::DBuf d_xyz, d_rgb, d_tri, d_cams, tri4, leaf_rgb, leaf_box, inner_box, nodes, par_leaf, par_inner, arrivals, d_rgba, counters;
  scn::Scratch sc;
  SCN_ALLOC(d_xyz, n_verts * 12);
  SCN_ALLOC(d_tri, n_faces * 12);
  SCN_ALLOC(d_cams, (size_t)n_views * sizeof(scn_render_camera_t));
  if (rgb) SCN_ALLOC(d_rgb, n_verts * 3);
  SCN_ALLOC(tri4, (size_t)n * 48);
  if (rgb) SCN_ALLOC(leaf_rgb, (size_t)n * 16);
  SCN_ALLOC(leaf_box, (size_t)n * 24);
  SCN_ALLOC(inner_box, (size_t)n * 24);
  SCN_ALLOC(nodes, (size_t)n * sizeof(Node));
  SCN_ALLOC(par_leaf, (size_t)n * 4);
  SCN_ALLOC(par_inner, (size_t)n * 4);
  SCN_ALLOC(arrivals, (size_t)n * 4);
  SCN_ALLOC(d_rgba, n_px * 4);
  SCN_ALLOC(counters, 5 * 8);
  if (int rc = sc.ensure(n, 0)) return rc;

  SCN_CUDA_TRY(cudaEventRecord(ev[0].get(), st));
  SCN_CUDA_TRY(cudaMemcpyAsync(d_xyz.p, xyz, n_verts * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(d_tri.p, tri, n_faces * 12, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(d_cams.p, cams, (size_t)n_views * sizeof(scn_render_camera_t), cudaMemcpyHostToDevice, st));
  if (rgb) SCN_CUDA_TRY(cudaMemcpyAsync(d_rgb.p, rgb, n_verts * 3, cudaMemcpyHostToDevice, st));
  SCN_CUDA_TRY(cudaMemsetAsync(counters.p, 0, 5 * 8, st));
  SCN_CUDA_TRY(cudaMemsetAsync(arrivals.p, 0, (size_t)n * 4, st));
  SCN_CUDA_TRY(cudaEventRecord(ev[1].get(), st));

  // BVH: Morton codes, stable sort of (code, face), leaves in sorted order, radix tree, boxes
  float3 blo = make_float3(lo[0], lo[1], lo[2]), inv;
  for (int k = 0; k < 3; ++k) { const float e = hi[k] - lo[k]; (&inv.x)[k] = e > 0.f ? 1024.f / e : 0.f; }
  k_morton<<<scn::grid_for(n), 256, 0, st>>>(d_xyz.as<float>(), d_tri.as<uint32_t>(), n, blo, inv, sc.k0.as<unsigned>(), sc.v0.as<unsigned>());
  SCN_CUDA_TRY(cudaGetLastError());
  unsigned* vals = sc.v0.as<unsigned>();
  scn::sort_pass(sc, vals, n, 30, st);
  const unsigned* keys = vals == sc.v0.as<unsigned>() ? sc.k0.as<unsigned>() : sc.k1.as<unsigned>();
  k_leaves<<<scn::grid_for(n), 256, 0, st>>>(d_xyz.as<float>(), rgb ? d_rgb.as<uint8_t>() : nullptr, d_tri.as<uint32_t>(), vals, n,
                                             tri4.as<float4>(), leaf_rgb.as<uint4>(), leaf_box.as<float>());
  SCN_CUDA_TRY(cudaGetLastError());
  if (n > 1) {
    k_karras<<<scn::grid_for(n - 1), 256, 0, st>>>(keys, (int)n, nodes.as<Node>(), par_leaf.as<unsigned>(), par_inner.as<unsigned>());
    SCN_CUDA_TRY(cudaGetLastError());
    k_boxes<<<scn::grid_for(n), 256, 0, st>>>((int)n, par_leaf.as<unsigned>(), par_inner.as<unsigned>(), leaf_box.as<float>(),
                                              inner_box.as<float>(), nodes.as<Node>(), arrivals.as<unsigned>());
    SCN_CUDA_TRY(cudaGetLastError());
  }
  SCN_CUDA_TRY(cudaEventRecord(ev[2].get(), st));

  const uint64_t px_per_cta = kTraceThreads / c.P, grid = (n_px + px_per_cta - 1) / px_per_cta;
  if (grid > 0x7fffffffull) return scn::fail(SCN_ERR_ARG, "%llu pixels in one call: too many", (unsigned long long)n_px);
  k_trace<<<(unsigned)grid, kTraceThreads, 0, st>>>(c, d_cams.as<scn_render_camera_t>(), nodes.as<Node>(), tri4.as<float4>(),
                                                    leaf_rgb.as<uint4>(), d_rgba.as<uint8_t>(), counters.as<unsigned long long>());
  SCN_CUDA_TRY(cudaGetLastError());
  SCN_CUDA_TRY(cudaEventRecord(ev[3].get(), st));
  unsigned long long cnt[5];
  SCN_CUDA_TRY(cudaMemcpyAsync(rgba_out, d_rgba.p, n_px * 4, cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaMemcpyAsync(cnt, counters.p, sizeof(cnt), cudaMemcpyDeviceToHost, st));
  SCN_CUDA_TRY(cudaEventRecord(ev[4].get(), st));
  SCN_CUDA_TRY(cudaEventSynchronize(ev[4].get()));
  if (report) {
    scn_render_report_t r{};
    r.views = n_views; r.pixels = n_px; r.samples = n_px * c.spp;
    r.primary_rays = cnt[0]; r.secondary_rays = cnt[1]; r.primary_hits = cnt[2]; r.node_visits = cnt[3]; r.triangle_tests = cnt[4];
    r.bvh_nodes = n - 1;
    float ms[4];
    for (int i = 0; i < 4; ++i) SCN_CUDA_TRY(cudaEventElapsedTime(&ms[i], ev[i].get(), ev[i + 1].get()));
    r.upload_ms = ms[0]; r.bvh_ms = ms[1]; r.trace_ms = ms[2]; r.download_ms = ms[3];
    r.total_ms = (scn::now_s() - t_start) * 1e3;
    *report = r;
  }
  return SCN_OK;
}

}  // extern "C"
