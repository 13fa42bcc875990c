// Device code shared by the tracker (track.cu, DESIGN.md §6j) and the global optimiser (globalopt.cu, §6k): the depth pyramid and
// vertex / normal maps of §6j step 1, the projective association of step 3, the Cholesky solve and the Cayley update of step 5.
// Every operation is an explicit correctly rounded intrinsic (and the library is built with -fmad=false), in the order of
// oracle/track_oracle.c, so both stages compare bit for bit with their oracles.  Not part of the public ABI.
#pragma once
#include <cmath>

#include "scn_common.h"

namespace {

constexpr int kCta = 256;
constexpr int kNSum = 28;                          // JtJ upper triangle (21), Jtr (6), sum r^2
constexpr unsigned kMinPairs = 64;
constexpr double kDamp = 0x1p-13;

struct Level {
  int W, H;
  float fx, fy, cx, cy, ifx, ify;
  float* depth; float4* v; float4* n;              // frame
  float* mdepth; float4* mv; float4* mn;           // model
};

struct Thresh { float dist2, normal; };

// level intrinsics from the depth intrinsic K at scale 2^-shift, rounded as the oracle's binary32 expressions
inline void level_intrinsics(Level& l, const float K[16], int shift) {
  const float sc = 1.0f / (float)(1 << shift);
  volatile float fx = K[0] * sc, fy = K[5] * sc, a = K[2] + 0.5f, b = K[6] + 0.5f;
  volatile float cx = a * sc, cy = b * sc;
  l.fx = fx; l.fy = fy; l.cx = cx - 0.5f; l.cy = cy - 0.5f;
  volatile float ifx = 1.0f / l.fx, ify = 1.0f / l.fy;
  l.ifx = ifx; l.ify = ify;
}

// ---------------------------------------------------------------------------------------------------------------- pyramid
__global__ void k_range(const float* __restrict__ m, int n, float dmin, float dmax, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = m[i];
  out[i] = (v >= dmin && v <= dmax) ? v : -INFINITY;
}

__global__ void k_reduce2(const float* __restrict__ in, int W, int H, float* __restrict__ out) {
  const int w = W / 2, h = H / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const int x = i % w, y = i / w;
  const float q[4] = {in[(2 * y) * W + 2 * x], in[(2 * y) * W + 2 * x + 1], in[(2 * y + 1) * W + 2 * x], in[(2 * y + 1) * W + 2 * x + 1]};
  float z[4]; int n = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) { const bool ok = q[k] != -INFINITY; z[k] = ok ? q[k] : 0.0f; n += ok; }
  out[i] = n ? __fdiv_rn(__fadd_rn(__fadd_rn(z[0], z[1]), __fadd_rn(z[2], z[3])), (float)n) : -INFINITY;
}

__device__ __forceinline__ float4 backproject(const Level& l, const float* D, int x, int y) {
  const float d = D[y * l.W + x];
  if (d == -INFINITY) return make_float4(0.f, 0.f, 0.f, 0.f);
  return make_float4(__fmul_rn(__fmul_rn(__fsub_rn((float)x, l.cx), l.ifx), d), __fmul_rn(__fmul_rn(__fsub_rn((float)y, l.cy), l.ify), d), d, 1.f);
}

__global__ void k_vertex_normal(const Level l, const float* __restrict__ D, float4* __restrict__ V, float4* __restrict__ N, unsigned* valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= l.W * l.H) return;
  const int x = i % l.W, y = i / l.W;
  const float4 c = backproject(l, D, x, y);
  float4 n = make_float4(0.f, 0.f, 0.f, 0.f);
  V[i] = c;
  if (c.w != 0.f && x > 0 && y > 0 && x + 1 < l.W && y + 1 < l.H) {
    const float4 r = backproject(l, D, x + 1, y), le = backproject(l, D, x - 1, y);
    const float4 dn = backproject(l, D, x, y + 1), up = backproject(l, D, x, y - 1);
    if (r.w != 0.f && le.w != 0.f && dn.w != 0.f && up.w != 0.f) {
      const float ux = __fsub_rn(r.x, le.x), uy = __fsub_rn(r.y, le.y), uz = __fsub_rn(r.z, le.z);
      const float vx = __fsub_rn(dn.x, up.x), vy = __fsub_rn(dn.y, up.y), vz = __fsub_rn(dn.z, up.z);
      const float cx = __fsub_rn(__fmul_rn(vy, uz), __fmul_rn(vz, uy));       // dv x du: towards the camera
      const float cy = __fsub_rn(__fmul_rn(vz, ux), __fmul_rn(vx, uz));
      const float cz = __fsub_rn(__fmul_rn(vx, uy), __fmul_rn(vy, ux));
      const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
      if (len > 0.f) {
        n = make_float4(__fdiv_rn(cx, len), __fdiv_rn(cy, len), __fdiv_rn(cz, len), 1.f);
        if (valid) atomicAdd(valid, 1u);
      }
    }
  }
  N[i] = n;
}

// ---------------------------------------------------------------------------------------------------------------- association
__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

struct Assoc { float tx, ty, tz, r; float4 nq; int j; };

// §6j step 3: the point p (normal np) of the source mapped by Df (3x4) into the target camera of level l, projected to the nearest
// pixel j of the target maps (mv, mn), kept when the distance and normal tests pass; r = n_q . (Df p - q)
__device__ __forceinline__ bool associate(const Level& l, const float4* __restrict__ mv, const float4* __restrict__ mn, const Thresh th,
                                          const float* Df, float4 p, float4 np, Assoc& a) {
  if (np.w == 0.f) return false;
  const float tx = __fadd_rn(dot3(Df[0], Df[1], Df[2], p.x, p.y, p.z), Df[3]);
  const float ty = __fadd_rn(dot3(Df[4], Df[5], Df[6], p.x, p.y, p.z), Df[7]);
  const float tz = __fadd_rn(dot3(Df[8], Df[9], Df[10], p.x, p.y, p.z), Df[11]);
  if (!(tz > 0.f)) return false;
  const float u = rintf(__fadd_rn(__fmul_rn(__fdiv_rn(tx, tz), l.fx), l.cx));
  const float v = rintf(__fadd_rn(__fmul_rn(__fdiv_rn(ty, tz), l.fy), l.cy));
  if (!(u >= 0.f && u <= (float)(l.W - 1) && v >= 0.f && v <= (float)(l.H - 1))) return false;
  const int j = (int)v * l.W + (int)u;
  const float4 q = mv[j], nq = mn[j];
  if (nq.w == 0.f) return false;
  const float dx = __fsub_rn(tx, q.x), dy = __fsub_rn(ty, q.y), dz = __fsub_rn(tz, q.z);
  if (!(dot3(dx, dy, dz, dx, dy, dz) <= th.dist2)) return false;
  const float rnx = dot3(Df[0], Df[1], Df[2], np.x, np.y, np.z);
  const float rny = dot3(Df[4], Df[5], Df[6], np.x, np.y, np.z);
  const float rnz = dot3(Df[8], Df[9], Df[10], np.x, np.y, np.z);
  if (!(dot3(rnx, rny, rnz, nq.x, nq.y, nq.z) >= th.normal)) return false;
  a.tx = tx; a.ty = ty; a.tz = tz; a.nq = nq; a.j = j;
  a.r = dot3(dx, dy, dz, nq.x, nq.y, nq.z);
  return true;
}

// the 28 exact binary64 products of a Jacobian row J (binary32) and residual r: J J^T upper triangle, J r, r^2
__device__ __forceinline__ void products28(const float* J, float r, double* out) {
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int b = a; b < 6; ++b) out[k++] = __dmul_rn((double)J[a], (double)J[b]);
#pragma unroll
  for (int a = 0; a < 6; ++a) out[k++] = __dmul_rn((double)J[a], (double)r);
  out[k] = __dmul_rn((double)r, (double)r);
}

// ---------------------------------------------------------------------------------------------------------------- solve, update
// Cholesky factor L of the symmetric 6x6 A; false when a pivot is not positive
__device__ bool chol6(const double (&A)[6][6], double (&L)[6][6]) {
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
    for (int m = 0; m < j; ++m) s = __dsub_rn(s, __dmul_rn(L[j][m], L[j][m]));
    if (!(s > 0.0)) return false;
    L[j][j] = __dsqrt_rn(s);
    for (int i = j + 1; i < 6; ++i) {
      double q = A[i][j];
      for (int m = 0; m < j; ++m) q = __dsub_rn(q, __dmul_rn(L[i][m], L[j][m]));
      L[i][j] = __ddiv_rn(q, L[j][j]);
    }
  }
  return true;
}

// x = (L L^T)^-1 b
__device__ void chol6_solve(const double (&L)[6][6], const double* b, double* x) {
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double q = b[i];
    for (int m = 0; m < i; ++m) q = __dsub_rn(q, __dmul_rn(L[i][m], y[m]));
    y[i] = __ddiv_rn(q, L[i][i]);
  }
  for (int i = 5; i >= 0; --i) {
    double q = y[i];
    for (int m = i + 1; m < 6; ++m) q = __dsub_rn(q, __dmul_rn(L[m][i], x[m]));
    x[i] = __ddiv_rn(q, L[i][i]);
  }
}

// Cholesky of (JtJ + kDamp * pairs * I) x = -Jtr; false when a pivot is not positive
__device__ bool solve6(const double* sum, unsigned pairs, double* x) {
  double A[6][6], L[6][6], b[6];
  const double lambda = __dmul_rn(kDamp, (double)pairs);
  int k = 0;
  for (int a = 0; a < 6; ++a) for (int c = a; c < 6; ++c) { A[a][c] = a == c ? __dadd_rn(sum[k], lambda) : sum[k]; A[c][a] = A[a][c]; ++k; }
  if (!chol6(A, L)) return false;
  for (int i = 0; i < 6; ++i) b[i] = -sum[21 + i];
  chol6_solve(L, b, x);
  return true;
}

// D <- [Cayley(x[0..2]) | x[3..5]] D, Cayley(w) = ((1 - g.g) I + 2 g g^T + 2 [g]x) / (1 + g.g), g = w / 2
__device__ void apply_update(double* D, const double* x) {
  const double g[3] = {__dmul_rn(x[0], 0.5), __dmul_rn(x[1], 0.5), __dmul_rn(x[2], 0.5)};
  const double gg = __dadd_rn(__dadd_rn(__dmul_rn(g[0], g[0]), __dmul_rn(g[1], g[1])), __dmul_rn(g[2], g[2]));
  const double den = __dadd_rn(1.0, gg);
  const double S[9] = {0.0, -g[2], g[1], g[2], 0.0, -g[0], -g[1], g[0], 0.0};
  double R[9], N[12];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
    R[3 * i + j] = __ddiv_rn(__dadd_rn(__dadd_rn((i == j) ? __dsub_rn(1.0, gg) : 0.0, __dmul_rn(__dmul_rn(2.0, g[i]), g[j])), __dmul_rn(2.0, S[3 * i + j])), den);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 4; ++j)
      N[4 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * i], D[j]), __dmul_rn(R[3 * i + 1], D[4 + j])), __dmul_rn(R[3 * i + 2], D[8 + j]));
    N[4 * i + 3] = __dadd_rn(N[4 * i + 3], x[3 + i]);
  }
  for (int i = 0; i < 12; ++i) D[i] = N[i];
}

}  // namespace
