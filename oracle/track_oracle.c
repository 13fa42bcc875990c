/* TEST INFRASTRUCTURE — scalar CPU statement of the frame-to-model ICP tracker (DESIGN.md §6j, "tracking spec v1").
 *
 * PARITY UNPINNED.  The reference's `recons` stage runs FriedLiver.exe (BundleFusion), which is not in the reference tree
 * (Server/scan_processor.py:27-29,123-126).  This is NOT BundleFusion's trajectory: no features, no global optimisation.
 * It is a frame-to-model dense point-to-plane ICP of the kind VoxelHashing's DepthSensing runs, written down here and in
 * scannet_b200/csrc/track.cu in the same binary32 / binary64 operations in the same order (compile with
 * -ffp-contract=off: no contraction), so that the GPU result is compared bit for bit.
 *
 * The volume is tsdf_oracle.c's (included below, unchanged): track -> integrate -> raycast -> next frame runs on the CPU.
 * Only tests/, __graft_entry__.smoke() and scripts/bench_recons.py may load this library.
 */
#include "tsdf_oracle.c"

#include <stdio.h>

#define TRK_LEVELS 3
#define TRK_CTA 256                 /* pixels per partial sum (one CTA of the association kernel) */
#define TRK_NSUM 28                 /* JtJ upper triangle (21), Jtr (6), sum r^2 */
static const int trk_iters[TRK_LEVELS] = { 4, 5, 10 };          /* iterations per level, finest (0) to coarsest (2) */
#define TRK_EXIT_STEP 1e-5          /* a level ends early once every |x_i| of an update is below this */
#define TRK_MIN_PAIRS 64            /* a system with fewer pairs loses the frame */
#define TRK_MAX_RMS 0.02            /* metres: a final point-to-plane RMS above this loses the frame */
#define TRK_DAMP 0x1p-13            /* added to every diagonal entry per pair: a view of one plane leaves the unobservable
                                     * directions at the prediction instead of an undetermined system */

typedef struct {
  uint32_t width, height;           /* tracking / raycast resolution: depth resolution / 2^s */
  float dist_thresh;                /* s_projCorrDistThres */
  float normal_thresh;              /* s_projCorrNormalThres */
  float ray_increment_factor;       /* s_SDFRayIncrementFactor */
} oracle_track_params;

typedef struct {                    /* = scn_track_frame_t */
  float    cam2world[16];
  uint32_t iterations[TRK_LEVELS];
  uint32_t pairs;
  uint32_t valid_pixels;
  uint32_t lost;
  double   residual_ss;
  double   rms;
} oracle_track_frame_t;

typedef struct { float x, y, z, w; } f4;    /* w = 1 valid */

typedef struct {
  int W, H;                        /* level size */
  float fx, fy, cx, cy, ifx, ify;
  float* depth; f4* v; f4* n;      /* frame */
  float* mdepth; f4* mv; f4* mn;   /* model */
} trk_level;

typedef struct {
  oracle_track_params p;
  oracle_tsdf* vol;
  int s;                           /* depth resolution = tracking resolution * 2^s */
  trk_level L[TRK_LEVELS];
  float* full;                     /* range-tested full-resolution depth */
  float* half[16];                 /* intermediate reductions between full and level 0 */
  int have_model;
  float ref[16];
} oracle_track;

/* ---- pyramid ------------------------------------------------------------------------------------------------------------ */
/* 2x2 -> 1: the mean of the valid ones among the four, ((a + b) + (c + d)) / n with an invalid pixel counted as 0 and n the
 * number of valid ones; invalid (-inf) when none is */
static void reduce2(const float* in, int W, int H, float* out) {
  const int w = W / 2, h = H / 2;
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    const float q[4] = { in[(2 * y) * W + 2 * x], in[(2 * y) * W + 2 * x + 1], in[(2 * y + 1) * W + 2 * x], in[(2 * y + 1) * W + 2 * x + 1] };
    float z[4]; int n = 0;
    for (int k = 0; k < 4; ++k) { const int ok = q[k] != -INFINITY; z[k] = ok ? q[k] : 0.0f; n += ok; }
    out[y * w + x] = n ? ((z[0] + z[1]) + (z[2] + z[3])) / (float)n : -INFINITY;
  }
}

static f4 backproject(const trk_level* l, const float* D, int x, int y) {
  f4 v = { 0.f, 0.f, 0.f, 0.f };
  const float d = D[y * l->W + x];
  if (d == -INFINITY) return v;
  v.x = (((float)x - l->cx) * l->ifx) * d; v.y = (((float)y - l->cy) * l->ify) * d; v.z = d; v.w = 1.f;
  return v;
}

/* vertex and normal maps of one level from its depth; returns the pixels with a normal */
static uint32_t vertex_normal(const trk_level* l, const float* D, f4* V, f4* N) {
  const int W = l->W, H = l->H;
  uint32_t valid = 0;
  for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) {
    const f4 c = backproject(l, D, x, y);
    f4 n = { 0.f, 0.f, 0.f, 0.f };
    V[y * W + x] = c;
    if (c.w != 0.f && x > 0 && y > 0 && x + 1 < W && y + 1 < H) {
      const f4 r = backproject(l, D, x + 1, y), le = backproject(l, D, x - 1, y);
      const f4 dn = backproject(l, D, x, y + 1), up = backproject(l, D, x, y - 1);
      if (r.w != 0.f && le.w != 0.f && dn.w != 0.f && up.w != 0.f) {
        const float ux = r.x - le.x, uy = r.y - le.y, uz = r.z - le.z;       /* du */
        const float vx = dn.x - up.x, vy = dn.y - up.y, vz = dn.z - up.z;    /* dv */
        const float cx = vy * uz - vz * uy, cy = vz * ux - vx * uz, cz = vx * uy - vy * ux;   /* dv x du: towards the camera */
        const float len = sqrtf((cx * cx + cy * cy) + cz * cz);
        if (len > 0.f) { n.x = cx / len; n.y = cy / len; n.z = cz / len; n.w = 1.f; ++valid; }
      }
    }
    N[y * W + x] = n;
  }
  return valid;
}

/* ---- raycast ------------------------------------------------------------------------------------------------------------- */
static float lerpf(float p, float q, float a) { return p * (1.0f - a) + q * a; }

/* trilinear SDF at voxel coordinates g; 0 when a corner is missing or has weight 0 */
static int sample_sdf(const oracle_tsdf* o, const float g[3], float* f) {
  for (int i = 0; i < 3; ++i) if (!(fabsf(g[i]) < 8388608.0f)) return 0;
  const float fl[3] = { floorf(g[0]), floorf(g[1]), floorf(g[2]) };
  const int b[3] = { (int)fl[0], (int)fl[1], (int)fl[2] };
  const float a[3] = { g[0] - fl[0], g[1] - fl[1], g[2] - fl[2] };
  float c[8];
  for (int k = 0; k < 8; ++k) {
    const ovoxel* v = vox_at(o, b[0] + (k & 1), b[1] + ((k >> 1) & 1), b[2] + (k >> 2));
    if (!v || v->w == 0) return 0;
    c[k] = v->sdf;
  }
  const float e0 = lerpf(c[0], c[1], a[0]), e1 = lerpf(c[2], c[3], a[0]), e2 = lerpf(c[4], c[5], a[0]), e3 = lerpf(c[6], c[7], a[0]);
  *f = lerpf(lerpf(e0, e1, a[1]), lerpf(e2, e3, a[1]), a[2]);
  return 1;
}

static void raycast(oracle_track* t, const float* T) {
  const oracle_tsdf_params* vp = &t->vol->p;
  const trk_level* l = &t->L[0];
  const float step = t->p.ray_increment_factor * vp->trunc_base;
  const float t_end = fminf(vp->depth_max, vp->max_integration_distance);
  const float inv_vs = 1.0f / vp->voxel_size;
#pragma omp parallel for schedule(dynamic, 4) num_threads(t->vol->threads)
  for (int y = 0; y < l->H; ++y) for (int x = 0; x < l->W; ++x) {
    const float rx = ((float)x - l->cx) * l->ifx, ry = ((float)y - l->cy) * l->ify;
    float res = -INFINITY, tp = 0.f, fp = 0.f;
    int prev = 0;
    for (int i = 0;; ++i) {
      const float tc = vp->depth_min + (float)i * step;
      if (!(tc <= t_end)) break;
      const float pc[3] = { rx * tc, ry * tc, tc };
      float g[3], f;
      for (int k = 0; k < 3; ++k) g[k] = (((T[4 * k] * pc[0] + T[4 * k + 1] * pc[1]) + T[4 * k + 2] * pc[2]) + T[4 * k + 3]) * inv_vs;
      const int ok = sample_sdf(t->vol, g, &f);
      if (ok && prev && fp > 0.f && f < 0.f) { res = tp + (tc - tp) * (fp / (fp - f)); break; }
      prev = ok; tp = tc; fp = f;
    }
    l->mdepth[y * l->W + x] = res;
  }
}

static void model_maps(oracle_track* t) {
  for (int k = 1; k < TRK_LEVELS; ++k) reduce2(t->L[k - 1].mdepth, t->L[k - 1].W, t->L[k - 1].H, t->L[k].mdepth);
  for (int k = 0; k < TRK_LEVELS; ++k) vertex_normal(&t->L[k], t->L[k].mdepth, t->L[k].mv, t->L[k].mn);
}

/* ---- association and the fixed-tree reduction -------------------------------------------------------------------------- */
/* One pixel's 28 exact binary64 products: zeros when it has no pair.  Returns 1 when paired. */
static int pair_terms(const trk_level* l, const oracle_track_params* tp, const float* Df, int i, double* out) {
  for (int k = 0; k < TRK_NSUM; ++k) out[k] = 0.0;
  const f4 p = l->v[i], np = l->n[i];
  if (np.w == 0.f) return 0;
  const float tx = ((Df[0] * p.x + Df[1] * p.y) + Df[2] * p.z) + Df[3];
  const float ty = ((Df[4] * p.x + Df[5] * p.y) + Df[6] * p.z) + Df[7];
  const float tz = ((Df[8] * p.x + Df[9] * p.y) + Df[10] * p.z) + Df[11];
  if (!(tz > 0.f)) return 0;
  const float u = rintf((tx / tz) * l->fx + l->cx), v = rintf((ty / tz) * l->fy + l->cy);   /* round half to even */
  if (!(u >= 0.f && u <= (float)(l->W - 1) && v >= 0.f && v <= (float)(l->H - 1))) return 0;
  const int j = (int)v * l->W + (int)u;
  const f4 q = l->mv[j], nq = l->mn[j];
  if (nq.w == 0.f) return 0;
  const float dx = tx - q.x, dy = ty - q.y, dz = tz - q.z;
  if (!((dx * dx + dy * dy) + dz * dz <= tp->dist_thresh * tp->dist_thresh)) return 0;
  const float rnx = (Df[0] * np.x + Df[1] * np.y) + Df[2] * np.z;
  const float rny = (Df[4] * np.x + Df[5] * np.y) + Df[6] * np.z;
  const float rnz = (Df[8] * np.x + Df[9] * np.y) + Df[10] * np.z;
  if (!((rnx * nq.x + rny * nq.y) + rnz * nq.z >= tp->normal_thresh)) return 0;
  const float r = (dx * nq.x + dy * nq.y) + dz * nq.z;
  const float J[6] = { ty * nq.z - tz * nq.y, tz * nq.x - tx * nq.z, tx * nq.y - ty * nq.x, nq.x, nq.y, nq.z };   /* (Tp x n_q, n_q) */
  int k = 0;
  for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) out[k++] = (double)J[a] * (double)J[b];
  for (int a = 0; a < 6; ++a) out[k++] = (double)J[a] * (double)r;
  out[k] = (double)r * (double)r;
  return 1;
}

/* The system of one iteration: per-CTA partials (256 pixels: warps of 32 summed by a halving tree, then the 8 warp sums by a
 * halving tree), then the partials added in CTA order. */
static void build_system(const trk_level* l, const oracle_track_params* tp, const float* Df, double* sum, uint32_t* pairs) {
  const int npx = l->W * l->H, ncta = (npx + TRK_CTA - 1) / TRK_CTA;
  double* part = (double*)malloc((size_t)ncta * TRK_NSUM * sizeof(double));
  uint32_t* pc = (uint32_t*)calloc((size_t)ncta, 4);
  for (int c = 0; c < ncta; ++c) {
    double v[TRK_CTA][TRK_NSUM], w[8][TRK_NSUM];
    for (int t = 0; t < TRK_CTA; ++t) {
      const int i = c * TRK_CTA + t;
      if (i < npx) pc[c] += (uint32_t)pair_terms(l, tp, Df, i, v[t]);
      else for (int k = 0; k < TRK_NSUM; ++k) v[t][k] = 0.0;
    }
    for (int wp = 0; wp < 8; ++wp) {
      double* lane[32];
      for (int t = 0; t < 32; ++t) lane[t] = v[32 * wp + t];
      for (int s = 16; s > 0; s >>= 1) for (int t = 0; t < s; ++t) for (int k = 0; k < TRK_NSUM; ++k) lane[t][k] = lane[t][k] + lane[t + s][k];
      for (int k = 0; k < TRK_NSUM; ++k) w[wp][k] = lane[0][k];
    }
    for (int s = 4; s > 0; s >>= 1) for (int t = 0; t < s; ++t) for (int k = 0; k < TRK_NSUM; ++k) w[t][k] = w[t][k] + w[t + s][k];
    for (int k = 0; k < TRK_NSUM; ++k) part[(size_t)c * TRK_NSUM + k] = w[0][k];
  }
  *pairs = 0;
  for (int k = 0; k < TRK_NSUM; ++k) sum[k] = 0.0;
  for (int c = 0; c < ncta; ++c) {
    for (int k = 0; k < TRK_NSUM; ++k) sum[k] = sum[k] + part[(size_t)c * TRK_NSUM + k];
    *pairs += pc[c];
  }
  free(part); free(pc);
}

/* ---- solve and update ------------------------------------------------------------------------------------------------------ */
/* Cholesky of the damped 6x6 system (JtJ + TRK_DAMP * pairs * I) x = -Jtr; returns 0 when a pivot is not positive */
int oracle_track_solve(const double* sum, uint32_t pairs, double* x) {
  double A[6][6], L[6][6], y[6];
  const double lambda = TRK_DAMP * (double)pairs;
  int k = 0;
  for (int a = 0; a < 6; ++a) for (int b = a; b < 6; ++b) { A[a][b] = a == b ? sum[k] + lambda : sum[k]; A[b][a] = A[a][b]; ++k; }
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
    for (int m = 0; m < j; ++m) s = s - L[j][m] * L[j][m];
    if (!(s > 0.0)) return 0;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double q = A[i][j];
      for (int m = 0; m < j; ++m) q = q - L[i][m] * L[j][m];
      L[i][j] = q / L[j][j];
    }
  }
  for (int i = 0; i < 6; ++i) {
    double q = -sum[21 + i];
    for (int m = 0; m < i; ++m) q = q - L[i][m] * y[m];
    y[i] = q / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double q = y[i];
    for (int m = i + 1; m < 6; ++m) q = q - L[m][i] * x[m];
    x[i] = q / L[i][i];
  }
  return 1;
}

/* Cayley rotation of w: R = (I - [w/2]x)^-1 (I + [w/2]x) = ((1 - g.g) I + 2 g g^T + 2 [g]x) / (1 + g.g), g = w / 2 */
void oracle_track_cayley(const double* w, double* R) {
  const double g[3] = { w[0] * 0.5, w[1] * 0.5, w[2] * 0.5 };
  const double gg = (g[0] * g[0] + g[1] * g[1]) + g[2] * g[2];
  const double den = 1.0 + gg;
  const double S[9] = { 0.0, -g[2], g[1], g[2], 0.0, -g[0], -g[1], g[0], 0.0 };
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
    R[3 * i + j] = (((i == j) ? (1.0 - gg) : 0.0) + (2.0 * g[i]) * g[j] + 2.0 * S[3 * i + j]) / den;
}

/* D (3x4, binary64) <- [Cayley(x[0..2]) | x[3..5]] D */
static void apply_update(double* D, const double* x) {
  double R[9], N[12];
  oracle_track_cayley(x, R);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 4; ++j) N[4 * i + j] = (R[3 * i] * D[j] + R[3 * i + 1] * D[4 + j]) + R[3 * i + 2] * D[8 + j];
    N[4 * i + 3] = N[4 * i + 3] + x[3 + i];
  }
  memcpy(D, N, sizeof(N));
}

/* ---- handle ------------------------------------------------------------------------------------------------------------------ */
oracle_track* oracle_track_create(const oracle_tsdf_params* vp, const oracle_track_params* tp, int threads) {
  const int W = (int)vp->width, H = (int)vp->height;
  int s = 0;
  while (s < 16 && ((uint32_t)W >> s) > tp->width) ++s;
  if (!tp->width || !tp->height || ((uint32_t)W >> s) != tp->width || ((uint32_t)W % tp->width) || ((uint32_t)H % tp->height) ||
      (uint32_t)H / tp->height != (uint32_t)W / tp->width || (tp->width >> (TRK_LEVELS - 1)) < 3 || (tp->height >> (TRK_LEVELS - 1)) < 3)
    return NULL;
  oracle_track* t = (oracle_track*)calloc(1, sizeof(oracle_track));
  t->p = *tp; t->s = s;
  t->vol = oracle_tsdf_create(vp, threads);
  t->full = (float*)malloc((size_t)W * H * 4);
  for (int k = 0; k < s; ++k) t->half[k] = (float*)malloc((size_t)(W >> (k + 1)) * (H >> (k + 1)) * 4);
  for (int k = 0; k < TRK_LEVELS; ++k) {
    trk_level* l = &t->L[k];
    l->W = (int)tp->width >> k; l->H = (int)tp->height >> k;
    const size_t n = (size_t)l->W * l->H;
    l->depth = (float*)malloc(n * 4); l->mdepth = (float*)malloc(n * 4);
    for (size_t i = 0; i < n; ++i) l->mdepth[i] = -INFINITY;
    l->v = (f4*)malloc(n * 16); l->n = (f4*)malloc(n * 16); l->mv = (f4*)calloc(n, 16); l->mn = (f4*)calloc(n, 16);
  }
  return t;
}

void oracle_track_destroy(oracle_track* t) {
  if (!t) return;
  oracle_tsdf_destroy(t->vol); free(t->full);
  for (int k = 0; k < t->s; ++k) free(t->half[k]);
  for (int k = 0; k < TRK_LEVELS; ++k) { trk_level* l = &t->L[k]; free(l->depth); free(l->mdepth); free(l->v); free(l->n); free(l->mv); free(l->mn); }
  free(t);
}

oracle_tsdf* oracle_track_volume(oracle_track* t) { return t->vol; }

/* Level intrinsics from the depth intrinsic K; the frame's depth pyramid, vertices and normals.  Returns valid pixels of level 0. */
static uint32_t frame_maps(oracle_track* t, const float* metres, const float* K) {
  const oracle_tsdf_params* vp = &t->vol->p;
  const int W = (int)vp->width, H = (int)vp->height;
  for (int i = 0; i < W * H; ++i) { const float m = metres[i]; t->full[i] = (m >= vp->depth_min && m <= vp->depth_max) ? m : -INFINITY; }
  const float* src = t->full;
  for (int k = 0; k < t->s; ++k) { reduce2(src, W >> k, H >> k, t->half[k]); src = t->half[k]; }
  memcpy(t->L[0].depth, src, (size_t)t->L[0].W * t->L[0].H * 4);
  for (int k = 1; k < TRK_LEVELS; ++k) reduce2(t->L[k - 1].depth, t->L[k - 1].W, t->L[k - 1].H, t->L[k].depth);
  uint32_t valid0 = 0;
  for (int k = 0; k < TRK_LEVELS; ++k) {
    trk_level* l = &t->L[k];
    const float sc = 1.0f / (float)(1 << (t->s + k));
    l->fx = K[0] * sc; l->fy = K[5] * sc; l->cx = (K[2] + 0.5f) * sc - 0.5f; l->cy = (K[6] + 0.5f) * sc - 0.5f;
    l->ifx = 1.0f / l->fx; l->ify = 1.0f / l->fy;
    const uint32_t v = vertex_normal(l, l->depth, l->v, l->n);
    if (k == 0) valid0 = v;
  }
  return valid0;
}

/* One frame: metres = the (filtered) depth at the volume's resolution, -inf invalid; rgb registered to it or NULL; K the depth
 * intrinsic; first_pose is read for the first frame only.  Returns 0. */
int oracle_track_frame(oracle_track* t, const float* metres, const uint8_t* rgb, const float* K, const float* first_pose,
                       oracle_track_frame_t* out) {
  memset(out, 0, sizeof(*out));
  out->valid_pixels = frame_maps(t, metres, K);
  float T[16];
  if (!t->have_model) {
    /* the seed: the first frame with at least TRK_MIN_PAIRS valid pixels; a frame before it is lost */
    if (out->valid_pixels < TRK_MIN_PAIRS) {
      out->lost = 1;
      for (int i = 0; i < 16; ++i) out->cam2world[i] = -INFINITY;
      return 0;
    }
    int finite = 1;
    for (int i = 0; i < 16; ++i) finite &= isfinite(first_pose[i]) ? 1 : 0;
    for (int i = 0; i < 16; ++i) T[i] = finite ? first_pose[i] : (i % 5 == 0 ? 1.f : 0.f);
  } else {
    double D[12] = { 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0 }, sum[TRK_NSUM], x[6];
    int lost = 0;
    uint32_t pairs = 0;
    for (int k = TRK_LEVELS - 1; k >= 0 && !lost; --k) {
      for (int it = 0; it < trk_iters[k]; ++it) {
        float Df[12];
        for (int i = 0; i < 12; ++i) Df[i] = (float)D[i];
        build_system(&t->L[k], &t->p, Df, sum, &pairs);
        out->iterations[k]++;
        out->pairs = pairs; out->residual_ss = sum[27];
        if (pairs < TRK_MIN_PAIRS || !oracle_track_solve(sum, pairs, x)) { lost = 1; break; }
        apply_update(D, x);
        double mx = 0.0;
        for (int i = 0; i < 6; ++i) mx = fmax(mx, fabs(x[i]));
        if (mx < TRK_EXIT_STEP) break;
      }
    }
    out->rms = pairs ? sqrt(out->residual_ss / (double)pairs) : 0.0;
    if (!lost && ((uint64_t)pairs * 4 < out->valid_pixels || out->rms > TRK_MAX_RMS)) lost = 1;
    if (lost) {
      out->lost = 1;
      for (int i = 0; i < 16; ++i) out->cam2world[i] = -INFINITY;
      return 0;
    }
    for (int i = 0; i < 3; ++i) {
      const double r0 = t->ref[4 * i], r1 = t->ref[4 * i + 1], r2 = t->ref[4 * i + 2];
      for (int j = 0; j < 3; ++j) T[4 * i + j] = (float)((r0 * D[j] + r1 * D[4 + j]) + r2 * D[8 + j]);
      T[4 * i + 3] = (float)(((r0 * D[3] + r1 * D[7]) + r2 * D[11]) + (double)t->ref[4 * i + 3]);
    }
    T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
  }
  memcpy(out->cam2world, T, sizeof(T));
  oracle_tsdf_integrate_metres(t->vol, metres, rgb, T, K);
  raycast(t, T);
  model_maps(t);
  memcpy(t->ref, T, sizeof(T));
  t->have_model = 1;
  return 0;
}

/* Test hooks: the model depth of level 0 (the last raycast), and the system of one iteration for a given estimate D (3x4 float)
 * at level k against the current model and the frame of the last oracle_track_frame call (or oracle_track_set_frame). */
void oracle_track_model_depth(const oracle_track* t, float* out) {
  memcpy(out, t->L[0].mdepth, (size_t)t->L[0].W * t->L[0].H * 4);
}
uint32_t oracle_track_set_frame(oracle_track* t, const float* metres, const float* K) { return frame_maps(t, metres, K); }
void oracle_track_system(oracle_track* t, int k, const float* Df, double* sum, uint32_t* pairs) {
  build_system(&t->L[k], &t->p, Df, sum, pairs);
}
/* per-pixel products of the same call in pixel order (npx * 28) and the pair flags, for a restatement of the tree */
void oracle_track_terms(oracle_track* t, int k, const float* Df, double* terms, uint8_t* paired) {
  const trk_level* l = &t->L[k];
  for (int i = 0; i < l->W * l->H; ++i) paired[i] = (uint8_t)pair_terms(l, &t->p, Df, i, terms + (size_t)i * TRK_NSUM);
}
/* frame / model maps of level k (W*H*4 floats each; w = 1 valid) */
void oracle_track_maps(const oracle_track* t, int k, float* v, float* n, float* mv, float* mn) {
  const trk_level* l = &t->L[k];
  const size_t b = (size_t)l->W * l->H * 16;
  if (v) memcpy(v, l->v, b);
  if (n) memcpy(n, l->n, b);
  if (mv) memcpy(mv, l->mv, b);
  if (mn) memcpy(mn, l->mn, b);
}
