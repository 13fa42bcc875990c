/* TEST INFRASTRUCTURE — scalar CPU statement of the dense global optimisation of the keyframe trajectory (DESIGN.md §6k,
 * "global optimisation spec v1").
 *
 * The reference's `recons` stage runs BundleFusion, whose global stage pairs sparse SIFT matches with a dense geometric term between
 * keyframes, solved by Gauss-Newton with PCG on the GPU.  Neither is in the reference tree.  This is the dense geometric term alone,
 * written down here and in scannet_b200/csrc/globalopt.cu in the same binary32 / binary64 operations in the same order (compile with
 * -ffp-contract=off: no contraction), so that the GPU result is compared bit for bit.
 *
 * It includes track_oracle.c (unchanged) for the §6j frame pipeline (range test, 2x2 reductions, vertex and normal maps), the
 * Cholesky solve and the Cayley update.  Only tests/, __graft_entry__.smoke() and scripts/bench_globalopt.py may load this library.
 */
#include "track_oracle.c"

#define GO_CTA 256                  /* pixels per partial sum (one CTA of the linearisation kernel) */
#define GO_PCG_THREADS 512          /* leaves of the fixed dot-product tree */
#define GO_MAX_NONLIN 16
#define GO_OVERLAP_NUM 1            /* an overlap check passes when found / valid >= GO_OVERLAP_NUM / GO_OVERLAP_DEN */
#define GO_OVERLAP_DEN 4

typedef struct {                    /* = scn_globalopt_params */
  uint32_t submap_size;             /* s_submapSize */
  uint32_t max_keyframes;           /* s_maxNumImages */
  uint32_t width, height;           /* s_downsampledWidth / Height: the depth resolution / 2^s */
  float dist_thresh;                /* s_denseDistThresh */
  float normal_thresh;              /* s_denseNormalThresh */
  float depth_min, depth_max;       /* s_denseDepthMin / Max */
  uint32_t overlap_subsample;       /* s_denseOverlapCheckSubsampleFactor */
  uint32_t nonlin_iters;            /* s_numGlobalNonLinIterations */
  uint32_t lin_iters;               /* s_numGlobalLinIterations */
  float verify_thresh;              /* s_verifyOptErrThresh */
  uint32_t max_removed;             /* s_maxNumResidualsRemoved */
} oracle_go_params;

typedef struct {                    /* the counters of scn_globalopt_report_t */
  uint32_t keyframes, edges_consecutive, edges_loop, edges_removed, rejected, solves;
  uint32_t nonlin_iterations, lin_iterations;
  uint64_t pairs_before, pairs_after;
  double rss_before, rss_after, rms_before, rms_after, max_edge_rms;
  double rss_iter[GO_MAX_NONLIN];   /* sum r^2 at the start of each Gauss-Newton iteration of the last solve */
} oracle_go_report;

typedef struct {
  oracle_go_params p;
  int W, H, s;                      /* depth resolution; keyframe resolution = depth / 2^s */
  trk_level L;                      /* keyframe level (intrinsics; v / n point at the keyframe being built) */
  float* full; float* half[16];
  int n;                            /* keyframes */
  f4* v; f4* nm;                    /* n * W * H each */
  double* D0;                       /* n * 12: the poses handed in */
  /* edges of the last solve, in (i, j) order */
  int ne;
  int* ei; int* ej; int* loop; int* active;
  double* esum;                     /* ne * 28 at the final poses */
  uint32_t* epairs;
  double* pcg_rz;                   /* rz before each PCG iteration of the first linear solve (lin_iters + 1) */
  double* pcg_x;                    /* the first linear solve's solution, 6 n */
} oracle_go;

/* ---- keyframes ----------------------------------------------------------------------------------------------------------- */
oracle_go* oracle_go_create(const oracle_go_params* p, uint32_t depth_width, uint32_t depth_height) {
  const uint32_t W = depth_width, H = depth_height;
  int s = 0;
  while (s < 16 && (W >> s) > p->width) ++s;
  if (!p->width || !p->height || (W >> s) != p->width || W % p->width || H % p->height || H / p->height != W / p->width ||
      p->width < 3 || p->height < 3 || !p->max_keyframes || !p->overlap_subsample || p->nonlin_iters > GO_MAX_NONLIN)
    return NULL;
  oracle_go* g = (oracle_go*)calloc(1, sizeof(oracle_go));
  g->p = *p; g->W = (int)W; g->H = (int)H; g->s = s;
  g->full = (float*)malloc((size_t)W * H * 4);
  for (int k = 0; k < s; ++k) g->half[k] = (float*)malloc((size_t)(W >> (k + 1)) * (H >> (k + 1)) * 4);
  g->L.W = (int)p->width; g->L.H = (int)p->height;
  const size_t npx = (size_t)p->width * p->height;
  g->L.depth = (float*)malloc(npx * 4);
  g->v = (f4*)malloc(npx * 16 * p->max_keyframes); g->nm = (f4*)malloc(npx * 16 * p->max_keyframes);
  g->D0 = (double*)malloc(sizeof(double) * 12 * p->max_keyframes);
  return g;
}

void oracle_go_destroy(oracle_go* g) {
  if (!g) return;
  free(g->full);
  for (int k = 0; k < g->s; ++k) free(g->half[k]);
  free(g->L.depth); free(g->v); free(g->nm); free(g->D0);
  free(g->ei); free(g->ej); free(g->loop); free(g->active); free(g->esum); free(g->epairs); free(g->pcg_rz); free(g->pcg_x);
  free(g);
}

/* One keyframe: metres = the (filtered) depth at the depth resolution, -inf invalid; K the depth intrinsic; T its cam2world.
 * Returns the pixels with a normal, or -1 when max_keyframes are already held. */
int oracle_go_add_keyframe(oracle_go* g, const float* metres, const float* K, const float* T) {
  if ((uint32_t)g->n >= g->p.max_keyframes) return -1;
  const int W = g->W, H = g->H;
  for (int i = 0; i < W * H; ++i) { const float m = metres[i]; g->full[i] = (m >= g->p.depth_min && m <= g->p.depth_max) ? m : -INFINITY; }
  const float* src = g->full;
  for (int k = 0; k < g->s; ++k) { reduce2(src, W >> k, H >> k, g->half[k]); src = g->half[k]; }
  trk_level* l = &g->L;
  memcpy(l->depth, src, (size_t)l->W * l->H * 4);
  const float sc = 1.0f / (float)(1 << g->s);
  l->fx = K[0] * sc; l->fy = K[5] * sc; l->cx = (K[2] + 0.5f) * sc - 0.5f; l->cy = (K[6] + 0.5f) * sc - 0.5f;
  l->ifx = 1.0f / l->fx; l->ify = 1.0f / l->fy;
  const size_t npx = (size_t)l->W * l->H;
  const uint32_t valid = vertex_normal(l, l->depth, g->v + npx * g->n, g->nm + npx * g->n);
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) g->D0[12 * g->n + 4 * r + c] = (double)T[4 * r + c];
  ++g->n;
  return (int)valid;
}

/* ---- one edge's residuals ------------------------------------------------------------------------------------------------ */
/* M = Ti^-1 Tj (3x4) in binary64 with Ti^-1 = [R^T | -R^T t], rounded once */
static void relative(const double* Di, const double* Dj, float* M) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 4; ++c) {
      double m = (Di[r] * Dj[c] + Di[4 + r] * Dj[4 + c]) + Di[8 + r] * Dj[8 + c];
      if (c == 3) m = m - ((Di[r] * Di[3] + Di[4 + r] * Di[7]) + Di[8 + r] * Di[11]);
      M[4 * r + c] = (float)m;
    }
  }
}

/* §6j step 3 against keyframe i's maps: r = n_i . (M p - v_i); returns 1 when associated */
static int associate(const trk_level* l, const f4* mv, const f4* mn, float dist2, float normal, const float* M, f4 p, f4 np,
                     float* t, f4* nq_out, float* r) {
  if (np.w == 0.f) return 0;
  const float tx = ((M[0] * p.x + M[1] * p.y) + M[2] * p.z) + M[3];
  const float ty = ((M[4] * p.x + M[5] * p.y) + M[6] * p.z) + M[7];
  const float tz = ((M[8] * p.x + M[9] * p.y) + M[10] * p.z) + M[11];
  if (!(tz > 0.f)) return 0;
  const float u = rintf((tx / tz) * l->fx + l->cx), v = rintf((ty / tz) * l->fy + l->cy);
  if (!(u >= 0.f && u <= (float)(l->W - 1) && v >= 0.f && v <= (float)(l->H - 1))) return 0;
  const int j = (int)v * l->W + (int)u;
  const f4 q = mv[j], nq = mn[j];
  if (nq.w == 0.f) return 0;
  const float dx = tx - q.x, dy = ty - q.y, dz = tz - q.z;
  if (!((dx * dx + dy * dy) + dz * dz <= dist2)) return 0;
  const float rnx = (M[0] * np.x + M[1] * np.y) + M[2] * np.z;
  const float rny = (M[4] * np.x + M[5] * np.y) + M[6] * np.z;
  const float rnz = (M[8] * np.x + M[9] * np.y) + M[10] * np.z;
  if (!((rnx * nq.x + rny * nq.y) + rnz * nq.z >= normal)) return 0;
  t[0] = tx; t[1] = ty; t[2] = tz; *nq_out = nq;
  *r = (dx * nq.x + dy * nq.y) + dz * nq.z;
  return 1;
}

/* pixel t of keyframe j against keyframe i: the 28 exact binary64 products of a = [(w_j x n^w), n^w] (w_j = Tj v_j, n^w = Ri n_i,
 * binary32) and r; zeros when unpaired */
static int edge_terms(const oracle_go* g, const double* D, int i, int j, const float* M, int t, double* out) {
  for (int k = 0; k < TRK_NSUM; ++k) out[k] = 0.0;
  const size_t npx = (size_t)g->L.W * g->L.H;
  float tp[3], r; f4 nq;
  const float d2 = g->p.dist_thresh * g->p.dist_thresh;
  const f4 p = g->v[npx * j + t];
  if (!associate(&g->L, g->v + npx * i, g->nm + npx * i, d2, g->p.normal_thresh, M, p, g->nm[npx * j + t], tp, &nq, &r)) return 0;
  float Tj[12], Ri[12];
  for (int k = 0; k < 12; ++k) { Tj[k] = (float)D[12 * j + k]; Ri[k] = (float)D[12 * i + k]; }
  const float wx = ((Tj[0] * p.x + Tj[1] * p.y) + Tj[2] * p.z) + Tj[3];
  const float wy = ((Tj[4] * p.x + Tj[5] * p.y) + Tj[6] * p.z) + Tj[7];
  const float wz = ((Tj[8] * p.x + Tj[9] * p.y) + Tj[10] * p.z) + Tj[11];
  const float nx = (Ri[0] * nq.x + Ri[1] * nq.y) + Ri[2] * nq.z;
  const float ny = (Ri[4] * nq.x + Ri[5] * nq.y) + Ri[6] * nq.z;
  const float nz = (Ri[8] * nq.x + Ri[9] * nq.y) + Ri[10] * nq.z;
  const float a[6] = { wy * nz - wz * ny, wz * nx - wx * nz, wx * ny - wy * nx, nx, ny, nz };
  int k = 0;
  for (int x = 0; x < 6; ++x) for (int y = x; y < 6; ++y) out[k++] = (double)a[x] * (double)a[y];
  for (int x = 0; x < 6; ++x) out[k++] = (double)a[x] * (double)r;
  out[k] = (double)r * (double)r;
  return 1;
}

/* the 28 sums of edge (i, j) at poses D by the §6j step-4 tree: slots of 256 pixels of j, warps of 32 by a halving tree, the 8 warp
 * sums by a halving tree, then the slots in slot order */
static void edge_system(const oracle_go* g, const double* D, int i, int j, double* sum, uint32_t* pairs) {
  float M[12];
  relative(D + 12 * i, D + 12 * j, M);
  const int npx = g->L.W * g->L.H, nslot = (npx + GO_CTA - 1) / GO_CTA;
  *pairs = 0;
  for (int k = 0; k < TRK_NSUM; ++k) sum[k] = 0.0;
  double (*v)[TRK_NSUM] = malloc(sizeof(double) * GO_CTA * TRK_NSUM);
  for (int c = 0; c < nslot; ++c) {
    double w[8][TRK_NSUM];
    for (int t = 0; t < GO_CTA; ++t) {
      const int px = c * GO_CTA + t;
      if (px < npx) *pairs += (uint32_t)edge_terms(g, D, i, j, M, px, v[t]);
      else for (int k = 0; k < TRK_NSUM; ++k) v[t][k] = 0.0;
    }
    for (int wp = 0; wp < 8; ++wp) {
      double* lane[32];
      for (int t = 0; t < 32; ++t) lane[t] = v[32 * wp + t];
      for (int s = 16; s > 0; s >>= 1) for (int t = 0; t < s; ++t) for (int k = 0; k < TRK_NSUM; ++k) lane[t][k] = lane[t][k] + lane[t + s][k];
      for (int k = 0; k < TRK_NSUM; ++k) w[wp][k] = lane[0][k];
    }
    for (int s = 4; s > 0; s >>= 1) for (int t = 0; t < s; ++t) for (int k = 0; k < TRK_NSUM; ++k) w[t][k] = w[t][k] + w[t + s][k];
    for (int k = 0; k < TRK_NSUM; ++k) sum[k] = sum[k] + w[0][k];
  }
  free(v);
}

/* the overlap check of (i, j) at poses D: j's pixels (x, y) with x and y multiples of the subsample factor */
static int overlaps(const oracle_go* g, const double* D, int i, int j) {
  float M[12];
  relative(D + 12 * i, D + 12 * j, M);
  const size_t npx = (size_t)g->L.W * g->L.H;
  const int f = (int)g->p.overlap_subsample;
  const float d2 = g->p.dist_thresh * g->p.dist_thresh;
  uint32_t valid = 0, found = 0;
  for (int y = 0; y < g->L.H; y += f) for (int x = 0; x < g->L.W; x += f) {
    const int t = y * g->L.W + x;
    float tp[3], r; f4 nq;
    valid += g->nm[npx * j + t].w != 0.f;
    found += (uint32_t)associate(&g->L, g->v + npx * i, g->nm + npx * i, d2, g->p.normal_thresh, M, g->v[npx * j + t], g->nm[npx * j + t], tp, &nq, &r);
  }
  return valid > 0 && (uint64_t)found * GO_OVERLAP_DEN >= (uint64_t)valid * GO_OVERLAP_NUM;
}

/* ---- the linear system and PCG --------------------------------------------------------------------------------------------- */
typedef struct {
  int n, ne;
  const int *ei, *ej, *act;
  const double* esum;               /* ne * 28 */
  double* Hd;                       /* n * 36: diagonal blocks, damped */
  double* rhs;                      /* 6 n: -g */
  int* free_;                       /* a node that moves in this iteration */
} go_sys;

/* H_ii += S, H_jj += S, H_ij -= S; g_j += b, g_i -= b; per node in edge order, then 2^-13 * (pairs touching k) on the diagonal */
static void assemble(go_sys* S, const uint32_t* epairs, const int* fixed) {
  for (int k = 0; k < S->n; ++k) {
    double H[36], gk[6];
    for (int q = 0; q < 36; ++q) H[q] = 0.0;
    for (int q = 0; q < 6; ++q) gk[q] = 0.0;
    uint32_t pk = 0;
    for (int e = 0; e < S->ne; ++e) {
      if (!S->act[e] || (S->ei[e] != k && S->ej[e] != k)) continue;
      const double* s = S->esum + (size_t)e * TRK_NSUM;
      int q = 0;
      for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) { H[6 * a + b] = H[6 * a + b] + s[q]; ++q; }
      for (int a = 0; a < 6; ++a) gk[a] = S->ej[e] == k ? gk[a] + s[21 + a] : gk[a] - s[21 + a];
      pk += epairs[e];
    }
    const double lambda = TRK_DAMP * (double)pk;
    for (int a = 0; a < 6; ++a) H[7 * a] = H[7 * a] + lambda;
    for (int a = 0; a < 6; ++a) for (int b = 0; b < a; ++b) H[6 * a + b] = H[6 * b + a];
    memcpy(S->Hd + 36 * k, H, sizeof(H));
    S->free_[k] = !fixed[k] && pk > 0;
    for (int a = 0; a < 6; ++a) S->rhs[6 * k + a] = S->free_[k] ? -gk[a] : 0.0;
  }
}

static void matvec(const go_sys* S, const double* x, double* y) {
  for (int k = 0; k < S->n; ++k) {
    for (int a = 0; a < 6; ++a) {
      if (!S->free_[k]) { y[6 * k + a] = 0.0; continue; }
      double acc = 0.0;
      for (int c = 0; c < 6; ++c) acc = acc + S->Hd[36 * k + 6 * a + c] * x[6 * k + c];
      for (int e = 0; e < S->ne; ++e) {
        if (!S->act[e] || (S->ei[e] != k && S->ej[e] != k)) continue;
        const int o = S->ei[e] == k ? S->ej[e] : S->ei[e];
        const double* s = S->esum + (size_t)e * TRK_NSUM;
        for (int c = 0; c < 6; ++c) {
          const int lo = a < c ? a : c, hi = a < c ? c : a;
          const double sac = s[lo * 6 - lo * (lo - 1) / 2 + (hi - lo)];      /* upper-triangle index of (lo, hi) */
          acc = acc - sac * x[6 * o + c];
        }
      }
      y[6 * k + a] = acc;
    }
  }
}

/* fixed tree: leaf t adds entries t, t + 512, ... in order; then a halving tree over the 512 leaves */
static double dot(const double* a, const double* b, int m) {
  double leaf[GO_PCG_THREADS];
  for (int t = 0; t < GO_PCG_THREADS; ++t) {
    double s = 0.0;
    for (int q = t; q < m; q += GO_PCG_THREADS) s = s + a[q] * b[q];
    leaf[t] = s;
  }
  for (int s = GO_PCG_THREADS / 2; s > 0; s >>= 1) for (int t = 0; t < s; ++t) leaf[t] = leaf[t] + leaf[t + s];
  return leaf[0];
}

/* block-Jacobi: z_k = H_kk^-1 r_k by Cholesky (track_oracle.c's solve with no damping and the right-hand side -(-r)) */
static int precond(const go_sys* S, const double* r, double* z) {
  for (int k = 0; k < S->n; ++k) {
    if (!S->free_[k]) { for (int a = 0; a < 6; ++a) z[6 * k + a] = 0.0; continue; }
    double sum[TRK_NSUM];
    int q = 0;
    for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) sum[q++] = S->Hd[36 * k + 6 * a + b];
    for (int a = 0; a < 6; ++a) sum[21 + a] = -r[6 * k + a];
    if (!oracle_track_solve(sum, 0, z + 6 * k)) return 0;
  }
  return 1;
}

/* PCG from x = 0 for lin_iters iterations, stopping early only when r.z is exactly 0.  Returns 0 when a preconditioner block is not
 * positive definite.  rz_hist (may be NULL) receives r.z before each iteration. */
static int pcg(const go_sys* S, uint32_t iters, double* x, uint32_t* run, double* rz_hist) {
  const int m = 6 * S->n;
  double* r = malloc(sizeof(double) * m * 4);
  double *z = r + m, *p = r + 2 * m, *q = r + 3 * m;
  int ok = 1;
  for (int a = 0; a < m; ++a) { x[a] = 0.0; r[a] = S->rhs[a]; }
  if (!precond(S, r, z)) { ok = 0; goto out; }
  memcpy(p, z, sizeof(double) * m);
  double rz = dot(r, z, m);
  *run = 0;
  for (uint32_t it = 0; it < iters; ++it) {
    if (rz_hist) rz_hist[it] = rz;
    if (rz == 0.0) break;
    matvec(S, p, q);
    const double alpha = rz / dot(p, q, m);
    for (int a = 0; a < m; ++a) { x[a] = x[a] + alpha * p[a]; r[a] = r[a] - alpha * q[a]; }
    if (!precond(S, r, z)) { ok = 0; goto out; }
    const double rzn = dot(r, z, m);
    const double beta = rzn / rz;
    for (int a = 0; a < m; ++a) p[a] = z[a] + beta * p[a];
    rz = rzn;
    ++*run;
  }
out:
  free(r);
  return ok;
}

/* ---- the solve ----------------------------------------------------------------------------------------------------------------- */
static int root(int* par, int k) { while (par[k] != k) k = par[k] = par[par[k]]; return k; }

/* the lowest-index keyframe of each connected component of the active edges is held fixed (a keyframe with no edge is its own) */
static void gauge(int n, int ne, const int* ei, const int* ej, const int* act, int* fixed) {
  int* par = malloc(sizeof(int) * (n ? n : 1));
  for (int k = 0; k < n; ++k) par[k] = k;
  for (int e = 0; e < ne; ++e) if (act[e]) {
    const int a = root(par, ei[e]), b = root(par, ej[e]);
    if (a != b) { if (a < b) par[b] = a; else par[a] = b; }
  }
  for (int k = 0; k < n; ++k) fixed[k] = root(par, k) == k;
  free(par);
}

static int finite12(const double* D) { for (int q = 0; q < 12; ++q) if (!isfinite(D[q])) return 0; return 1; }

/* Solves the keyframes held.  poses_out (n * 16): the optimised cam2world, or the poses handed in when the result is rejected. */
int oracle_go_solve(oracle_go* g, float* poses_out, oracle_go_report* rep) {
  const int n = g->n;
  memset(rep, 0, sizeof(*rep));
  rep->keyframes = (uint32_t)n;
  free(g->ei); free(g->ej); free(g->loop); free(g->active); free(g->esum); free(g->epairs); free(g->pcg_rz); free(g->pcg_x);
  const int cap = n > 1 ? n * (n - 1) / 2 : 1;
  g->ei = malloc(sizeof(int) * cap); g->ej = malloc(sizeof(int) * cap); g->loop = malloc(sizeof(int) * cap); g->active = malloc(sizeof(int) * cap);
  g->ne = 0;
  for (int i = 0; i < n; ++i) for (int j = i + 1; j < n; ++j) {
    const int ov = j == i + 1 || overlaps(g, g->D0, i, j);
    if (!ov) continue;
    g->ei[g->ne] = i; g->ej[g->ne] = j; g->loop[g->ne] = j != i + 1; g->active[g->ne] = 1; ++g->ne;
    if (j == i + 1) ++rep->edges_consecutive; else ++rep->edges_loop;
  }
  const int ne = g->ne;
  g->esum = malloc(sizeof(double) * TRK_NSUM * (ne ? ne : 1)); g->epairs = malloc(sizeof(uint32_t) * (ne ? ne : 1));
  g->pcg_rz = calloc(g->p.lin_iters + 1, sizeof(double)); g->pcg_x = calloc(6 * (size_t)(n ? n : 1), sizeof(double));
  double* D = malloc(sizeof(double) * 12 * (n ? n : 1));
  double* x = malloc(sizeof(double) * 6 * (n ? n : 1));
  int* fixed = malloc(sizeof(int) * (n ? n : 1)); int* fr = malloc(sizeof(int) * (n ? n : 1));
  double* Hd = malloc(sizeof(double) * 36 * (n ? n : 1)); double* rhs = malloc(sizeof(double) * 6 * (n ? n : 1));
  go_sys S = { n, ne, g->ei, g->ej, g->active, g->esum, Hd, rhs, fr };
  int first = 1;
  while (ne > 0) {
    gauge(n, ne, g->ei, g->ej, g->active, fixed);
    memcpy(D, g->D0, sizeof(double) * 12 * n);
    int nonfinite = 0;
    ++rep->solves;
    for (uint32_t it = 0; it <= g->p.nonlin_iters; ++it) {
      double rss = 0.0; uint64_t pairs = 0;
      for (int e = 0; e < ne; ++e) {
        if (!g->active[e]) continue;
        edge_system(g, D, g->ei[e], g->ej[e], g->esum + (size_t)e * TRK_NSUM, &g->epairs[e]);
        rss = rss + g->esum[(size_t)e * TRK_NSUM + 27]; pairs += g->epairs[e];
      }
      if (first && it == 0) { rep->rss_before = rss; rep->pairs_before = pairs; }
      if (it == g->p.nonlin_iters) { rep->rss_after = rss; rep->pairs_after = pairs; break; }
      rep->rss_iter[it] = rss;
      assemble(&S, g->epairs, fixed);
      uint32_t run = 0;
      if (!pcg(&S, g->p.lin_iters, x, &run, first && it == 0 ? g->pcg_rz : NULL)) nonfinite = 1;
      if (first && it == 0) memcpy(g->pcg_x, x, sizeof(double) * 6 * n);
      rep->lin_iterations += run; ++rep->nonlin_iterations;
      for (int k = 0; k < n; ++k) {
        if (!fr[k]) continue;
        apply_update(D + 12 * k, x + 6 * k);
        if (!finite12(D + 12 * k)) nonfinite = 1;
      }
    }
    first = 0;
    /* verification at the final poses */
    int worst = -1; double worst_score = 0.0; rep->max_edge_rms = 0.0;
    for (int e = 0; e < ne; ++e) {
      if (!g->active[e]) continue;
      const uint32_t pe = g->epairs[e];
      const double rms = pe ? sqrt(g->esum[(size_t)e * TRK_NSUM + 27] / (double)pe) : 0.0;
      if (rms > rep->max_edge_rms) rep->max_edge_rms = rms;
      const double score = pe < TRK_MIN_PAIRS ? INFINITY : rms;
      if ((pe < TRK_MIN_PAIRS || rms > g->p.verify_thresh) && (worst < 0 || score > worst_score)) { worst = e; worst_score = score; }
    }
    if (nonfinite) { rep->rejected = 1; break; }
    if (worst < 0) break;
    if (rep->edges_removed >= g->p.max_removed) { rep->rejected = 1; break; }
    g->active[worst] = 0;
    ++rep->edges_removed;
  }
  rep->rms_before = rep->pairs_before ? sqrt(rep->rss_before / (double)rep->pairs_before) : 0.0;
  rep->rms_after = rep->pairs_after ? sqrt(rep->rss_after / (double)rep->pairs_after) : 0.0;
  for (int k = 0; k < n; ++k) {
    const double* P = rep->rejected ? g->D0 + 12 * k : D + 12 * k;
    for (int q = 0; q < 12; ++q) poses_out[16 * k + q] = (float)P[q];
    poses_out[16 * k + 12] = 0.f; poses_out[16 * k + 13] = 0.f; poses_out[16 * k + 14] = 0.f; poses_out[16 * k + 15] = 1.f;
  }
  free(D); free(x); free(fixed); free(fr); free(Hd); free(rhs);
  return 0;
}

/* ---- test hooks ---------------------------------------------------------------------------------------------------------------- */
int oracle_go_num_edges(const oracle_go* g) { return g->ne; }
/* the last solve's edges in (i, j) order: i, j, loop flag, still active, pairs and the 28 sums at the final poses */
void oracle_go_edges(const oracle_go* g, int* ei, int* ej, int* loop, int* active, uint32_t* pairs, double* sums) {
  for (int e = 0; e < g->ne; ++e) {
    ei[e] = g->ei[e]; ej[e] = g->ej[e]; loop[e] = g->loop[e]; active[e] = g->active[e]; pairs[e] = g->epairs[e];
    if (sums) memcpy(sums + (size_t)e * TRK_NSUM, g->esum + (size_t)e * TRK_NSUM, sizeof(double) * TRK_NSUM);
  }
}
/* the 28 sums of (i, j) at the poses handed in */
void oracle_go_edge_system(const oracle_go* g, int i, int j, double* sum, uint32_t* pairs) { edge_system(g, g->D0, i, j, sum, pairs); }
/* the first linear system of a solve over every edge of the last solve (or, with ne_in >= 0, over the given edges) at the poses
 * handed in: the dense damped H (6n x 6n, free and fixed rows alike), the right-hand side -g (0 for a node that does not move), the
 * free flags, and PCG's solution after `iters` iterations */
void oracle_go_first_system(oracle_go* g, int ne_in, const int* ei_in, const int* ej_in, uint32_t iters, double* Hdense, double* rhs,
                            int* free_out, double* x) {
  const int n = g->n;
  const int ne = ne_in >= 0 ? ne_in : g->ne;
  const int* ei = ne_in >= 0 ? ei_in : g->ei;
  const int* ej = ne_in >= 0 ? ej_in : g->ej;
  int* act = malloc(sizeof(int) * (ne ? ne : 1));
  double* es = malloc(sizeof(double) * TRK_NSUM * (ne ? ne : 1));
  uint32_t* ep = malloc(sizeof(uint32_t) * (ne ? ne : 1));
  int* fixed = malloc(sizeof(int) * n);
  double* Hd = malloc(sizeof(double) * 36 * n);
  for (int e = 0; e < ne; ++e) { act[e] = 1; edge_system(g, g->D0, ei[e], ej[e], es + (size_t)e * TRK_NSUM, &ep[e]); }
  gauge(n, ne, ei, ej, act, fixed);
  go_sys S = { n, ne, ei, ej, act, es, Hd, rhs, free_out };
  assemble(&S, ep, fixed);
  const int m = 6 * n;
  for (int q = 0; q < m * m; ++q) Hdense[q] = 0.0;
  for (int k = 0; k < n; ++k) for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) Hdense[(size_t)(6 * k + a) * m + 6 * k + b] = Hd[36 * k + 6 * a + b];
  for (int e = 0; e < ne; ++e) {
    const double* s = es + (size_t)e * TRK_NSUM;
    int q = 0;
    for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) {
      const double v = -s[q++];
      Hdense[(size_t)(6 * ei[e] + a) * m + 6 * ej[e] + b] += v; Hdense[(size_t)(6 * ej[e] + b) * m + 6 * ei[e] + a] += v;
      if (a != b) { Hdense[(size_t)(6 * ei[e] + b) * m + 6 * ej[e] + a] += v; Hdense[(size_t)(6 * ej[e] + a) * m + 6 * ei[e] + b] += v; }
    }
  }
  uint32_t run = 0;
  pcg(&S, iters, x, &run, NULL);
  free(act); free(es); free(ep); free(fixed); free(Hd);
}
/* r.z before each PCG iteration and the solution of the first linear solve of the last oracle_go_solve */
void oracle_go_pcg_trace(const oracle_go* g, double* rz, double* x) {
  if (rz) memcpy(rz, g->pcg_rz, sizeof(double) * (g->p.lin_iters + 1));
  if (x) memcpy(x, g->pcg_x, sizeof(double) * 6 * g->n);
}
