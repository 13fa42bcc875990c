/* TEST INFRASTRUCTURE — not product code.
 *
 * Sequential CPU statement of quadric edge-collapse decimation, DESIGN.md §6g (this repository's own spec: MeshLab/VCG is not
 * in the reference tree, and a priority-queue decimation could not be reproduced in parallel anyway).  Round by round it makes
 * the same selection as the kernels and uses the same binary64 arithmetic, operation for operation (contraction off:
 * oracle/meshclean.mk passes -ffp-contract=off).  Positions are binary32.
 *
 * Mode 1 ("one collapse at a time") applies a round's selected edges one by one in ascending order and recomputes every edge,
 * cost and placement before each one.  It exists only to check that the collapses of a round commute (tests/). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* counters[]: the integer fields of scn_mesh_simplify_report_t after the four size fields, in order */
enum { C_TARGET, C_ROUNDS, C_COLLAPSES, C_FACES_COLLAPSED, C_AUTOCLEAN_DUP, C_MAX_VERTEX_FACES, C_N };

#define QUALITY_SCALE (2.0 * 1.7320508075688772)   /* 2*sqrt(3) in binary64: q = 4*sqrt(3)*area / sum l^2 = 2*sqrt(3)*|n| / sum l^2 */

typedef struct {
  int64_t nV, nF;
  float* xyz;          /* nV*3, vertex positions (dead vertices keep their last position) */
  double* Q;           /* nV*10: q00 q01 q02 q03 q11 q12 q13 q22 q23 q33 */
  uint32_t* tri;       /* nF*3 */
  uint8_t* falive;     /* nF */
  int64_t alive;
} State;

typedef struct {       /* one round's edges, ascending (a, b) */
  int64_t n;
  uint32_t *a, *b;
  double* cost;
  float* p;            /* n*3: placement */
  uint32_t* f;         /* alive faces containing both ends */
  int64_t *ring_start; /* nV+1 */
  uint32_t* ring;      /* corner indices of alive faces, grouped by vertex, ascending within a vertex */
} Round;

static void face_quadric(const float* p0, const float* p1, const float* p2, double* K) {
  const double x0 = p0[0], y0 = p0[1], z0 = p0[2];
  const double ux = (double)p1[0] - x0, uy = (double)p1[1] - y0, uz = (double)p1[2] - z0;
  const double vx = (double)p2[0] - x0, vy = (double)p2[1] - y0, vz = (double)p2[2] - z0;
  const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
  const double len = sqrt((nx * nx + ny * ny) + nz * nz);
  if (len == 0.0) { for (int i = 0; i < 10; ++i) K[i] = 0.0; return; }
  const double d = -((nx * x0 + ny * y0) + nz * z0);
  const double v[4] = {nx, ny, nz, d};
  int k = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = i; j < 4; ++j) K[k++] = (v[i] * v[j]) / len;
}

static double quality(const float* p0, const float* p1, const float* p2) {
  const double ux = (double)p1[0] - p0[0], uy = (double)p1[1] - p0[1], uz = (double)p1[2] - p0[2];
  const double vx = (double)p2[0] - p0[0], vy = (double)p2[1] - p0[1], vz = (double)p2[2] - p0[2];
  const double wx = (double)p2[0] - p1[0], wy = (double)p2[1] - p1[1], wz = (double)p2[2] - p1[2];
  const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
  const double len = sqrt((nx * nx + ny * ny) + nz * nz);
  const double s = (((ux * ux + uy * uy) + uz * uz) + ((wx * wx + wy * wy) + wz * wz)) + ((vx * vx + vy * vy) + vz * vz);
  return s > 0.0 ? (QUALITY_SCALE * len) / s : 0.0;
}

static double qerr(const double* q, const float* p) {
  const double x = p[0], y = p[1], z = p[2];
  return ((((((((q[0] * x * x + 2.0 * q[1] * x * y) + 2.0 * q[2] * x * z) + 2.0 * q[3] * x) + q[4] * y * y) + 2.0 * q[5] * y * z) +
            2.0 * q[6] * y) + q[7] * z * z) + 2.0 * q[8] * z) + q[9];
}

/* placement of edge (a, b) with Q = Q_a + Q_b; returns err at the placement */
static double place(const double* q, const float* pa, const float* pb, float* out) {
  const double c00 = q[4] * q[7] - q[5] * q[5], c01 = q[2] * q[5] - q[1] * q[7], c02 = q[1] * q[5] - q[2] * q[4];
  const double c11 = q[0] * q[7] - q[2] * q[2], c12 = q[1] * q[2] - q[0] * q[5], c22 = q[0] * q[4] - q[1] * q[1];
  const double det = (q[0] * c00 + q[1] * c01) + q[2] * c02;
  if (det > 1e-9 * q[0] * q[4] * q[7]) {
    const double b0 = -q[3], b1 = -q[6], b2 = -q[8];
    const float x[3] = {(float)(((c00 * b0 + c01 * b1) + c02 * b2) / det), (float)(((c01 * b0 + c11 * b1) + c12 * b2) / det),
                        (float)(((c02 * b0 + c12 * b1) + c22 * b2) / det)};
    if (isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2])) { memcpy(out, x, 12); return qerr(q, out); }
  }
  const float mid[3] = {(float)(0.5 * ((double)pa[0] + (double)pb[0])), (float)(0.5 * ((double)pa[1] + (double)pb[1])),
                        (float)(0.5 * ((double)pa[2] + (double)pb[2]))};
  const float* cand[3] = {pa, pb, mid};
  double best = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double e = qerr(q, cand[i]);
    if (i == 0 || e < best) { best = e; memcpy(out, cand[i], 12); }
  }
  return best;
}

static int has(const uint32_t* t, uint32_t v) { return t[0] == v || t[1] == v || t[2] == v; }

/* quality penalty and f(e) of edge (a, b) placed at p */
static double penalty_and_f(const State* s, const Round* r, uint32_t a, uint32_t b, const float* p, double thr, uint32_t* f_out) {
  double qmin = 1.0;
  uint32_t f = 0;
  const uint32_t ends[2] = {a, b};
  for (int k = 0; k < 2; ++k) {
    const uint32_t v = ends[k];
    for (int64_t i = r->ring_start[v]; i < r->ring_start[v + 1]; ++i) {
      const uint32_t face = r->ring[i] / 3;
      const uint32_t* t = s->tri + 3 * (size_t)face;
      if (has(t, a) && has(t, b)) {
        if (k == 0 && (i == r->ring_start[v] || r->ring[i - 1] / 3 != face)) ++f;    /* once per face */
        continue;
      }
      const float* c[3];
      for (int j = 0; j < 3; ++j) c[j] = (t[j] == a || t[j] == b) ? p : s->xyz + 3 * (size_t)t[j];
      const double q = quality(c[0], c[1], c[2]);
      if (q < qmin) qmin = q;
    }
  }
  *f_out = f;
  return qmin < thr ? thr / (qmin > 1e-6 ? qmin : 1e-6) : 1.0;
}

static int cmp_pair(const void* x, const void* y) {
  const uint64_t a = *(const uint64_t*)x, b = *(const uint64_t*)y;
  return a < b ? -1 : a > b;
}

static int cmp_pair16(const void* x, const void* y) {
  const uint64_t* a = (const uint64_t*)x; const uint64_t* b = (const uint64_t*)y;
  if (a[0] != b[0]) return a[0] < b[0] ? -1 : 1;
  return a[1] < b[1] ? -1 : a[1] > b[1];
}

static void round_free(Round* r) { free(r->a); free(r->b); free(r->cost); free(r->p); free(r->f); free(r->ring_start); free(r->ring); memset(r, 0, sizeof(*r)); }

/* edges, rings and costs of the current mesh; returns the largest ring (corners at one vertex) or -2 */
static int64_t build_round(const State* s, double thr, Round* r) {
  memset(r, 0, sizeof(*r));
  uint64_t* pairs = (uint64_t*)malloc((size_t)(3 * s->nF + 1) * 8);
  r->ring_start = (int64_t*)calloc((size_t)s->nV + 2, 8);
  r->ring = (uint32_t*)malloc((size_t)(3 * s->nF + 1) * 4);
  if (!pairs || !r->ring_start || !r->ring) { free(pairs); return -2; }
  int64_t np = 0;
  for (int64_t f = 0; f < s->nF; ++f) {
    if (!s->falive[f]) continue;
    const uint32_t* t = s->tri + 3 * f;
    for (int k = 0; k < 3; ++k) {
      uint32_t u = t[k], v = t[(k + 1) % 3];
      r->ring_start[u + 1]++;
      if (u == v) continue;
      if (u > v) { const uint32_t x = u; u = v; v = x; }
      pairs[np++] = ((uint64_t)u << 32) | v;
    }
  }
  int64_t big = 0;
  for (int64_t v = 0; v < s->nV; ++v) { if (r->ring_start[v + 1] > big) big = r->ring_start[v + 1]; r->ring_start[v + 1] += r->ring_start[v]; }
  int64_t* fill = (int64_t*)malloc((size_t)(s->nV + 1) * 8);
  if (!fill) { free(pairs); return -2; }
  memcpy(fill, r->ring_start, (size_t)(s->nV + 1) * 8);
  for (int64_t f = 0; f < s->nF; ++f)
    if (s->falive[f]) for (int k = 0; k < 3; ++k) r->ring[fill[s->tri[3 * f + k]]++] = (uint32_t)(3 * f + k);
  free(fill);
  qsort(pairs, (size_t)np, 8, cmp_pair);
  int64_t ne = 0;
  for (int64_t i = 0; i < np; ++i) if (i == 0 || pairs[i] != pairs[i - 1]) pairs[ne++] = pairs[i];
  r->n = ne;
  r->a = (uint32_t*)malloc((size_t)(ne + 1) * 4); r->b = (uint32_t*)malloc((size_t)(ne + 1) * 4); r->f = (uint32_t*)malloc((size_t)(ne + 1) * 4);
  r->cost = (double*)malloc((size_t)(ne + 1) * 8); r->p = (float*)malloc((size_t)(ne + 1) * 12);
  if (!r->a || !r->b || !r->f || !r->cost || !r->p) { free(pairs); return -2; }
  for (int64_t e = 0; e < ne; ++e) {
    const uint32_t a = (uint32_t)(pairs[e] >> 32), b = (uint32_t)pairs[e];
    double q[10];
    for (int i = 0; i < 10; ++i) q[i] = s->Q[10 * (size_t)a + i] + s->Q[10 * (size_t)b + i];
    float* p = r->p + 3 * e;
    const double err = place(q, s->xyz + 3 * (size_t)a, s->xyz + 3 * (size_t)b, p);
    const double pen = penalty_and_f(s, r, a, b, p, thr, &r->f[e]);
    r->a[e] = a; r->b[e] = b;
    r->cost[e] = (err > 1e-15 ? err : 1e-15) * pen;
  }
  free(pairs);
  return big;
}

static const Round* g_round;                       /* qsort has no context argument */
static int cmp_edge(const void* x, const void* y) {
  const int64_t i = *(const int64_t*)x, j = *(const int64_t*)y;
  const double ci = g_round->cost[i], cj = g_round->cost[j];
  if (ci != cj) return ci < cj ? -1 : 1;
  return i < j ? -1 : i > j;                         /* edges are in (a, b) order */
}

static void collapse(State* s, uint32_t a, uint32_t b, const float* p) {
  memcpy(s->xyz + 3 * (size_t)a, p, 12);
  for (int i = 0; i < 10; ++i) s->Q[10 * (size_t)a + i] = s->Q[10 * (size_t)a + i] + s->Q[10 * (size_t)b + i];
  for (int64_t f = 0; f < s->nF; ++f) {
    if (!s->falive[f]) continue;
    uint32_t* t = s->tri + 3 * f;
    if (!has(t, b)) continue;
    if (has(t, a)) { s->falive[f] = 0; s->alive--; continue; }
    for (int k = 0; k < 3; ++k) if (t[k] == b) t[k] = a;
  }
}

/* Returns 0, -1 for the inputs the library refuses with SCN_ERR_ARG, -2 out of memory, -3 a batched round differs from
 * applying its collapses one at a time (mode 1 only).
 * max_rounds < 0: the whole filter with AutoClean; outputs compacted (room for nV vertices and nF faces).
 * max_rounds >= 0: stops after that many rounds, before AutoClean, and writes the raw state: all nV positions, all nF faces,
 * falive_out[nF], quad_out[nV*10] (either may be NULL) and the cost of every applied collapse in order (cost_out, room for nF). */
int oracle_mesh_simplify(const float* xyz, const uint8_t* rgb, int64_t nV, const uint32_t* tri, int64_t nF, uint64_t target_faces,
                         double target_perc, double quality_thr, int mode, int64_t max_rounds, float* xyz_out, uint8_t* rgb_out,
                         uint32_t* tri_out, int64_t* nV_out, int64_t* nF_out, uint64_t* counters, uint8_t* falive_out, double* quad_out,
                         double* cost_out) {
  memset(counters, 0, C_N * sizeof(uint64_t));
  for (int64_t c = 0; c < 3 * nF; ++c) if ((int64_t)tri[c] >= nV) return -1;
  for (int64_t i = 0; i < 3 * nV; ++i) if (!isfinite(xyz[i])) return -1;
  if (!(target_perc >= 0.0 && target_perc <= 1.0) || !(quality_thr >= 0.0)) return -1;
  const uint64_t target = target_perc != 0.0 ? (uint64_t)floor((double)nF * target_perc) : target_faces;
  counters[C_TARGET] = target;
  State s = {nV, nF, NULL, NULL, NULL, NULL, nF};
  s.xyz = (float*)malloc((size_t)(nV + 1) * 12); s.Q = (double*)calloc((size_t)nV + 1, 80);
  s.tri = (uint32_t*)malloc((size_t)(nF + 1) * 12); s.falive = (uint8_t*)malloc((size_t)nF + 1);
  uint64_t* order = NULL; uint32_t* m = NULL; uint32_t* M = NULL; uint32_t* rank = NULL;
  int rc = 0;
  Round r = {0};
  if (!s.xyz || !s.Q || !s.tri || !s.falive) { rc = -2; goto out; }
  if (nV) memcpy(s.xyz, xyz, (size_t)nV * 12);
  if (nF) memcpy(s.tri, tri, (size_t)nF * 12);
  memset(s.falive, 1, (size_t)nF);
  /* vertex quadrics: every corner adds its face's quadric, faces ascending (a repeated corner adds K_f = 0 again) */
  for (int64_t f = 0; f < nF; ++f) {
    double K[10];
    const uint32_t* t = s.tri + 3 * f;
    face_quadric(s.xyz + 3 * (size_t)t[0], s.xyz + 3 * (size_t)t[1], s.xyz + 3 * (size_t)t[2], K);
    for (int k = 0; k < 3; ++k) for (int i = 0; i < 10; ++i) s.Q[10 * (size_t)t[k] + i] = s.Q[10 * (size_t)t[k] + i] + K[i];
  }
  int64_t ncost = 0;
  while ((uint64_t)s.alive > target && (max_rounds < 0 || (int64_t)counters[C_ROUNDS] < max_rounds)) {
    const int64_t big = build_round(&s, quality_thr, &r);
    if (big < 0) { rc = -2; goto out; }
    if ((uint64_t)big > counters[C_MAX_VERTEX_FACES]) counters[C_MAX_VERTEX_FACES] = (uint64_t)big;
    const int64_t ne = r.n;
    if (ne == 0) break;
    order = (uint64_t*)malloc((size_t)ne * 8); rank = (uint32_t*)malloc((size_t)ne * 4);
    m = (uint32_t*)malloc((size_t)nV * 4); M = (uint32_t*)malloc((size_t)nV * 4);
    if (!order || !rank || !m || !M) { rc = -2; goto out; }
    for (int64_t e = 0; e < ne; ++e) order[e] = (uint64_t)e;
    g_round = &r;
    qsort(order, (size_t)ne, 8, cmp_edge);
    for (int64_t i = 0; i < ne; ++i) rank[order[i]] = (uint32_t)i;
    for (int64_t v = 0; v < nV; ++v) m[v] = UINT32_MAX;
    for (int64_t e = 0; e < ne; ++e) {
      if (rank[e] < m[r.a[e]]) m[r.a[e]] = rank[e];
      if (rank[e] < m[r.b[e]]) m[r.b[e]] = rank[e];
    }
    memcpy(M, m, (size_t)nV * 4);
    for (int64_t e = 0; e < ne; ++e) {
      if (m[r.b[e]] < M[r.a[e]]) M[r.a[e]] = m[r.b[e]];
      if (m[r.a[e]] < M[r.b[e]]) M[r.b[e]] = m[r.a[e]];
    }
    /* the selected edges, in ascending order, while the target is not reached */
    int64_t nsel = 0;
    for (int64_t i = 0; i < ne; ++i) {
      const int64_t e = (int64_t)order[i];
      if (M[r.a[e]] == (uint32_t)i && M[r.b[e]] == (uint32_t)i) order[nsel++] = (uint64_t)e;
    }
    if (mode == 0) {
      /* the prefix, then all of it in one pass over the faces; m[] is reused as the rename table */
      int64_t left = s.alive, napp = 0;
      for (; napp < nsel && (uint64_t)left > target; ++napp) left -= r.f[order[napp]];
      for (int64_t v = 0; v < nV; ++v) m[v] = (uint32_t)v;
      for (int64_t k = 0; k < napp; ++k) {
        const int64_t e = (int64_t)order[k];
        const uint32_t a = r.a[e], b = r.b[e];
        memcpy(s.xyz + 3 * (size_t)a, r.p + 3 * e, 12);
        for (int i = 0; i < 10; ++i) s.Q[10 * (size_t)a + i] = s.Q[10 * (size_t)a + i] + s.Q[10 * (size_t)b + i];
        m[b] = a;
        counters[C_COLLAPSES]++; counters[C_FACES_COLLAPSED] += r.f[e];
        if (cost_out) cost_out[ncost] = r.cost[e];
        ++ncost;
      }
      for (int64_t f = 0; f < nF; ++f) {
        if (!s.falive[f]) continue;
        uint32_t* t = s.tri + 3 * f;
        for (int k = 0; k < 3; ++k) {
          if (m[t[k]] == t[k]) continue;
          const uint32_t a = m[t[k]], b = t[k];        /* a face meets at most one collapsed edge */
          if (has(t, a)) { s.falive[f] = 0; s.alive--; break; }
          for (int j = 0; j < 3; ++j) if (t[j] == b) t[j] = a;
          break;
        }
      }
      if (s.alive != left) { rc = -3; goto out; }
    } else {
      Round one = {0};
      const uint32_t* sa = r.a; const uint32_t* sb = r.b;
      for (int64_t k = 0; k < nsel && (uint64_t)s.alive > target; ++k) {
        const uint32_t a = sa[order[k]], b = sb[order[k]];
        if (build_round(&s, quality_thr, &one) < 0) { round_free(&one); rc = -2; goto out; }
        int64_t lo = 0, hi = one.n;                    /* the edge in the recomputed list */
        while (lo < hi) { const int64_t mid = (lo + hi) / 2; if (one.a[mid] < a || (one.a[mid] == a && one.b[mid] < b)) lo = mid + 1; else hi = mid; }
        if (lo == one.n || one.a[lo] != a || one.b[lo] != b) { round_free(&one); rc = -3; goto out; }
        const int64_t before = s.alive;
        collapse(&s, a, b, one.p + 3 * lo);
        if (before - s.alive != (int64_t)one.f[lo]) { round_free(&one); rc = -3; goto out; }
        counters[C_COLLAPSES]++; counters[C_FACES_COLLAPSED] += one.f[lo];
        if (cost_out) cost_out[ncost] = one.cost[lo];
        ++ncost;
        round_free(&one);
      }
    }
    counters[C_ROUNDS]++;
    free(order); free(rank); free(m); free(M); order = NULL; rank = NULL; m = M = NULL;
    round_free(&r);
  }
  if (max_rounds >= 0) {
    if (nV) memcpy(xyz_out, s.xyz, (size_t)nV * 12);
    if (nF) memcpy(tri_out, s.tri, (size_t)nF * 12);
    if (falive_out && nF) memcpy(falive_out, s.falive, (size_t)nF);
    if (quad_out && nV) memcpy(quad_out, s.Q, (size_t)nV * 80);
    *nV_out = nV; *nF_out = nF;
    goto out;
  }
  /* AutoClean: alive faces in order, duplicates dropped under mLib's rule (the first of each sorted index triple survives),
   * then unreferenced vertices dropped; survivors keep ascending order */
  {
    int64_t f2 = 0;
    uint64_t* key = (uint64_t*)malloc((size_t)(nF + 1) * 16);
    uint8_t* ref = (uint8_t*)calloc((size_t)nV + 1, 1);
    int64_t* newid = (int64_t*)malloc((size_t)(nV + 1) * 8);
    if (!key || !ref || !newid) { free(key); free(ref); free(newid); rc = -2; goto out; }
    int64_t na = 0;
    for (int64_t f = 0; f < nF; ++f) {
      if (!s.falive[f]) continue;
      uint64_t k[3] = {s.tri[3 * f], s.tri[3 * f + 1], s.tri[3 * f + 2]}, x;
      if (k[0] > k[1]) { x = k[0]; k[0] = k[1]; k[1] = x; }
      if (k[1] > k[2]) { x = k[1]; k[1] = k[2]; k[2] = x; }
      if (k[0] > k[1]) { x = k[0]; k[0] = k[1]; k[1] = x; }
      key[2 * na] = (k[0] << 32) | k[1]; key[2 * na + 1] = (k[2] << 32) | (uint64_t)f;
      ++na;
    }
    qsort(key, (size_t)na, 16, cmp_pair16);           /* by (triple, face): the first of each run is the lowest face index */
    uint8_t* keep = (uint8_t*)calloc((size_t)nF + 1, 1);
    if (!keep) { free(key); free(ref); free(newid); rc = -2; goto out; }
    for (int64_t i = 0; i < na; ++i)
      if (i == 0 || key[2 * i] != key[2 * i - 2] || (key[2 * i + 1] >> 32) != (key[2 * i - 1] >> 32)) keep[key[2 * i + 1] & 0xFFFFFFFFu] = 1;
    for (int64_t f = 0; f < nF; ++f) {
      if (!keep[f]) continue;
      memcpy(tri_out + 3 * f2, s.tri + 3 * f, 12);
      for (int k = 0; k < 3; ++k) ref[s.tri[3 * f + k]] = 1;
      ++f2;
    }
    counters[C_AUTOCLEAN_DUP] = (uint64_t)(na - f2);
    int64_t v2 = 0;
    for (int64_t v = 0; v < nV; ++v) {
      if (!ref[v]) continue;
      newid[v] = v2;
      memcpy(xyz_out + 3 * v2, s.xyz + 3 * v, 12);
      if (rgb && rgb_out) memcpy(rgb_out + 3 * v2, rgb + 3 * v, 3);
      ++v2;
    }
    for (int64_t c = 0; c < 3 * f2; ++c) tri_out[c] = (uint32_t)newid[tri_out[c]];
    *nV_out = v2; *nF_out = f2;
    free(key); free(ref); free(newid); free(keep);
  }
out:
  round_free(&r);
  free(order); free(rank); free(m); free(M);
  free(s.xyz); free(s.Q); free(s.tri); free(s.falive);
  return rc;
}
