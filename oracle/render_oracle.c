/* TEST INFRASTRUCTURE — scalar C statement of "render spec v1" (DESIGN.md §6i), the preview render that stands in for
 * Server/mts_render.py.  Never linked into libscannet_b200.so.  Compiled with -ffp-contract=off: every binary32 + - * / sqrt
 * is one IEEE operation, round to nearest, as in csrc/render.cu under -fmad=false.
 *
 * It takes the binary32 cameras scn_render_camera makes and has two traversal modes: brute force over every face, and its own
 * host BVH (median split of the face centroids on the longest box axis, at most 4 faces per leaf) with the same monotone
 * sheared-box cull as the kernels.  The two trees differ from each other and from the kernels' Karras tree, so agreement of
 * all three is the evidence that no cull changes a result.  OpenMP over the rows of the requested pixel rectangle. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float origin[3], p00[3], du[3], dv[3], t_near, t_eps, ao_length; } Cam;

/* ---------------------------------------------------------------------------------------------- tables (binary64 host) */
static double srgb_decode(double x) { return x <= 0.04045 ? x / 12.92 : pow((x + 0.055) / 1.055, 2.4); }

void oracle_render_tables(float lin[256], float thr[255]) {
  for (int k = 0; k < 256; ++k) lin[k] = (float)srgb_decode(k / 255.0);
  for (int k = 0; k < 255; ++k) thr[k] = (float)srgb_decode((k + 0.5) / 255.0);
}

/* ---------------------------------------------------------------------------------------------- mesh */
typedef struct {
  const float* xyz; const uint8_t* rgb; const uint32_t* tri; uint32_t nf;
  uint8_t* degenerate;                       /* fl(|cross(v1 - v0, v2 - v0)|^2) is not > 0: never hit */
  /* BVH: nodes with box, children (or first face / count for leaves), faces permuted */
  int n_nodes; float (*box)[6]; int (*kid)[2]; int* first; int* count; uint32_t* perm;
} Mesh;

static float mnf(float a, float b) { return a < b ? a : b; }
static float mxf(float a, float b) { return a > b ? a : b; }

static uint32_t mix32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
static float unit(uint32_t h, uint32_t dim) { return (float)(mix32(h ^ dim) >> 8) * 5.9604644775390625e-8f; }

typedef struct { float o[3], d[3], S[3]; int kx, ky, kz; } Ray;

static void ray_prep(Ray* r) {
  const float ax = fabsf(r->d[0]), ay = fabsf(r->d[1]), az = fabsf(r->d[2]);
  r->kz = ax >= ay ? (ax >= az ? 0 : 2) : (ay >= az ? 1 : 2);
  r->kx = (r->kz + 1) % 3; r->ky = (r->kx + 1) % 3;
  r->S[0] = r->d[r->kx] / r->d[r->kz]; r->S[1] = r->d[r->ky] / r->d[r->kz]; r->S[2] = 1.0f / r->d[r->kz];
}

static const float* vtx(const Mesh* m, uint32_t f, int j) { return m->xyz + 3 * (size_t)m->tri[3 * (size_t)f + j]; }

/* watertight test (Woop, Benthin, Wald 2013) without the binary64 fallback, plus the bounding-box clause and the clamp of t
 * to [min, max] of the sheared depths of the vertices */
static int tri_test(const Ray* r, const float* v0, const float* v1, const float* v2, float* t, float* U, float* V, float* W, float* det) {
  const int kx = r->kx, ky = r->ky, kz = r->kz;
  const float Akx = v0[kx] - r->o[kx], Aky = v0[ky] - r->o[ky], Akz = v0[kz] - r->o[kz];
  const float Bkx = v1[kx] - r->o[kx], Bky = v1[ky] - r->o[ky], Bkz = v1[kz] - r->o[kz];
  const float Ckx = v2[kx] - r->o[kx], Cky = v2[ky] - r->o[ky], Ckz = v2[kz] - r->o[kz];
  const float Ax = Akx - r->S[0] * Akz, Ay = Aky - r->S[1] * Akz;
  const float Bx = Bkx - r->S[0] * Bkz, By = Bky - r->S[1] * Bkz;
  const float Cx = Ckx - r->S[0] * Ckz, Cy = Cky - r->S[1] * Ckz;
  if (mnf(mnf(Ax, Bx), Cx) > 0.f || mxf(mxf(Ax, Bx), Cx) < 0.f || mnf(mnf(Ay, By), Cy) > 0.f || mxf(mxf(Ay, By), Cy) < 0.f) return 0;
  *U = Cx * By - Cy * Bx;
  *V = Ax * Cy - Ay * Cx;
  *W = Bx * Ay - By * Ax;
  if ((*U < 0.f || *V < 0.f || *W < 0.f) && (*U > 0.f || *V > 0.f || *W > 0.f)) return 0;
  *det = (*U + *V) + *W;
  if (*det == 0.f) return 0;
  const float Az = r->S[2] * Akz, Bz = r->S[2] * Bkz, Cz = r->S[2] * Ckz;
  const float T = (*U * Az + *V * Bz) + *W * Cz;
  float tt = mxf(T / *det, mnf(mnf(Az, Bz), Cz));
  *t = mnf(tt, mxf(mxf(Az, Bz), Cz));
  return 1;
}

/* the sheared-box cull: monotone in every vertex coordinate, so the corners bound any vertex in the box */
static int box_test(const Ray* r, const float* b, float tmin, float best) {
  const int kx = r->kx, ky = r->ky, kz = r->kz;
  const float lkx = b[kx] - r->o[kx], hkx = b[3 + kx] - r->o[kx];
  const float lky = b[ky] - r->o[ky], hky = b[3 + ky] - r->o[ky];
  const float lkz = b[kz] - r->o[kz], hkz = b[3 + kz] - r->o[kz];
  const float gx0 = r->S[0] * lkz, gx1 = r->S[0] * hkz, gy0 = r->S[1] * lkz, gy1 = r->S[1] * hkz;
  if (lkx - mxf(gx0, gx1) > 0.f || hkx - mnf(gx0, gx1) < 0.f) return 0;
  if (lky - mxf(gy0, gy1) > 0.f || hky - mnf(gy0, gy1) < 0.f) return 0;
  const float z0 = r->S[2] * lkz, z1 = r->S[2] * hkz;
  return mnf(z0, z1) <= best && mxf(z0, z1) > tmin;
}

typedef struct { float t; uint32_t face; } Hit;

static void consider(const Mesh* m, const Ray* r, uint32_t f, float tmin, uint32_t skip, Hit* h) {
  if (f == skip || m->degenerate[f]) return;
  float t, U, V, W, det;
  if (tri_test(r, vtx(m, f, 0), vtx(m, f, 1), vtx(m, f, 2), &t, &U, &V, &W, &det) && t > tmin && (t < h->t || (t == h->t && f < h->face))) {
    h->t = t; h->face = f;
  }
}

/* closest hit with tmin < t <= tmax, smallest t then smallest face; face UINT32_MAX for none */
static Hit trace(const Mesh* m, const Ray* r, float tmin, float tmax, uint32_t skip, int bvh) {
  Hit h = {tmax, UINT32_MAX};
  if (!bvh) {
    for (uint32_t f = 0; f < m->nf; ++f) consider(m, r, f, tmin, skip, &h);
    return h;
  }
  int stack[128], sp = 0;
  stack[sp++] = 0;
  while (sp) {
    const int n = stack[--sp];
    if (!box_test(r, m->box[n], tmin, h.t)) continue;
    if (m->count[n]) { for (int i = 0; i < m->count[n]; ++i) consider(m, r, m->perm[m->first[n] + i], tmin, skip, &h); continue; }
    stack[sp++] = m->kid[n][1]; stack[sp++] = m->kid[n][0];
  }
  return h;
}

/* ---------------------------------------------------------------------------------------------- host BVH (median split) */
static const float* g_cent;
static int g_axis;
static int cmp_face(const void* a, const void* b) {
  const uint32_t fa = *(const uint32_t*)a, fb = *(const uint32_t*)b;
  const float ca = g_cent[3 * (size_t)fa + g_axis], cb = g_cent[3 * (size_t)fb + g_axis];
  return ca < cb ? -1 : ca > cb ? 1 : (fa < fb ? -1 : fa > fb);
}

static int build(Mesh* m, const float* cent, int first, int count) {
  const int n = m->n_nodes++;
  float* b = m->box[n];
  for (int i = 0; i < 3; ++i) { b[i] = INFINITY; b[3 + i] = -INFINITY; }
  for (int k = 0; k < count; ++k)
    for (int j = 0; j < 3; ++j) {
      const float* v = vtx(m, m->perm[first + k], j);
      for (int i = 0; i < 3; ++i) { b[i] = mnf(b[i], v[i]); b[3 + i] = mxf(b[3 + i], v[i]); }
    }
  m->first[n] = first;
  if (count <= 4) { m->count[n] = count; return n; }
  m->count[n] = 0;
  int axis = 0;
  for (int i = 1; i < 3; ++i) if (b[3 + i] - b[i] > b[3 + axis] - b[axis]) axis = i;
  g_cent = cent; g_axis = axis;
  qsort(m->perm + first, (size_t)count, 4, cmp_face);
  const int half = count / 2;
  const int l = build(m, cent, first, half);
  const int r = build(m, cent, first + half, count - half);
  m->kid[n][0] = l; m->kid[n][1] = r;
  return n;
}

static int mesh_init(Mesh* m, const float* xyz, const uint8_t* rgb, const uint32_t* tri, uint64_t nf, int bvh) {
  memset(m, 0, sizeof(*m));
  m->xyz = xyz; m->rgb = rgb; m->tri = tri; m->nf = (uint32_t)nf;
  m->degenerate = malloc(nf ? nf : 1);
  if (!m->degenerate) return -1;
  for (uint64_t f = 0; f < nf; ++f) {
    const float *v0 = vtx(m, f, 0), *v1 = vtx(m, f, 1), *v2 = vtx(m, f, 2);
    const float e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]}, e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
    const float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
    m->degenerate[f] = !((nx * nx + ny * ny) + nz * nz > 0.f);
  }
  if (!bvh) return 0;
  const size_t cap = 2 * (size_t)nf + 1;
  m->box = malloc(cap * sizeof(*m->box)); m->kid = malloc(cap * sizeof(*m->kid));
  m->first = malloc(cap * sizeof(int)); m->count = malloc(cap * sizeof(int)); m->perm = malloc(nf * 4);
  float* cent = malloc(nf * 12);
  if (!m->box || !m->kid || !m->first || !m->count || !m->perm || !cent) { free(cent); return -1; }
  for (uint64_t f = 0; f < nf; ++f) {
    m->perm[f] = (uint32_t)f;
    for (int i = 0; i < 3; ++i) cent[3 * f + i] = vtx(m, f, 0)[i] + vtx(m, f, 1)[i] + vtx(m, f, 2)[i];
  }
  build(m, cent, 0, (int)nf);
  free(cent);
  return 0;
}

static void mesh_free(Mesh* m) { free(m->degenerate); free(m->box); free(m->kid); free(m->first); free(m->count); free(m->perm); }

/* ---------------------------------------------------------------------------------------------- shading */
static void face_normal(const Mesh* m, uint32_t f, const float d[3], float n[3]) {
  const float *v0 = vtx(m, f, 0), *v1 = vtx(m, f, 1), *v2 = vtx(m, f, 2);
  const float e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]}, e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
  n[0] = e1[1] * e2[2] - e1[2] * e2[1];
  n[1] = e1[2] * e2[0] - e1[0] * e2[2];
  n[2] = e1[0] * e2[1] - e1[1] * e2[0];
  const float l = sqrtf((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  n[0] = n[0] / l; n[1] = n[1] / l; n[2] = n[2] / l;
  if ((n[0] * d[0] + n[1] * d[1]) + n[2] * d[2] > 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

static void cosine_dir(const float n[3], uint32_t h, float d[3]) {
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

static void reflectance(const Mesh* m, const float* lin, const Ray* r, uint32_t f, float rho[3]) {
  if (!m->rgb) { rho[0] = rho[1] = rho[2] = 0.5f; return; }
  float t, U, V, W, det;
  tri_test(r, vtx(m, f, 0), vtx(m, f, 1), vtx(m, f, 2), &t, &U, &V, &W, &det);
  const float b0 = U / det, b1 = V / det, b2 = W / det;
  for (int ch = 0; ch < 3; ++ch) {
    const float c0 = lin[m->rgb[3 * (size_t)m->tri[3 * (size_t)f] + ch]], c1 = lin[m->rgb[3 * (size_t)m->tri[3 * (size_t)f + 1] + ch]],
                c2 = lin[m->rgb[3 * (size_t)m->tri[3 * (size_t)f + 2] + ch]];
    rho[ch] = (b0 * c0 + b1 * c1) + b2 * c2;
  }
}

/* One sample: radiance L and whether the primary ray hit.  counters: primary, secondary, primary hits. */
static int sample(const Mesh* m, const float* lin, const Cam* cam, uint32_t pix, uint32_t x, uint32_t y, uint32_t s,
                  int integrator, uint32_t max_depth, int bvh, float L[3], uint64_t cnt[3]) {
  const uint32_t hs = mix32(mix32(pix ^ 0x9e3779b9u) ^ s);
  const uint32_t h0 = mix32(hs);
  const float fx = (float)x + unit(h0, 0), fy = (float)y + unit(h0, 1);
  Ray r;
  for (int i = 0; i < 3; ++i) { r.o[i] = cam->origin[i]; r.d[i] = (cam->p00[i] + fx * cam->du[i]) + fy * cam->dv[i]; }
  ray_prep(&r);
  Hit h = trace(m, &r, cam->t_near, INFINITY, UINT32_MAX, bvh);
  cnt[0]++;
  L[0] = L[1] = L[2] = 0.f;
  if (h.face == UINT32_MAX) { L[0] = L[1] = L[2] = 1.f; return 0; }
  cnt[2]++;
  float thr[3] = {1.f, 1.f, 1.f};
  for (uint32_t depth = 1;; ++depth) {
    if (integrator == 0) {
      float rho[3];
      reflectance(m, lin, &r, h.face, rho);
      thr[0] = thr[0] * rho[0]; thr[1] = thr[1] * rho[1]; thr[2] = thr[2] * rho[2];
      if (depth == max_depth) return 1;
    }
    float n[3];
    face_normal(m, h.face, r.d, n);
    Ray sr;
    for (int i = 0; i < 3; ++i) sr.o[i] = r.o[i] + h.t * r.d[i];
    cosine_dir(n, mix32(hs ^ depth), sr.d);
    ray_prep(&sr);
    const Hit h2 = trace(m, &sr, cam->t_eps, integrator == 1 ? cam->ao_length : INFINITY, h.face, bvh);
    cnt[1]++;
    if (h2.face == UINT32_MAX) { L[0] = thr[0]; L[1] = thr[1]; L[2] = thr[2]; return 1; }
    if (integrator == 1) return 1;
    r = sr; h = h2;
  }
}

/* Renders the pixels [x0, x0+w) x [y0, y0+h) of each view into rgba (n_views * h * w * 4).  mode 0: brute force, 1: BVH.
 * counters[3]: primary rays, secondary rays, primary hits.  Returns 0, or -1 when out of memory. */
int oracle_render(const float* xyz, const uint8_t* rgb, uint64_t nv, const uint32_t* tri, uint64_t nf, uint32_t W, uint32_t H,
                  uint32_t spp, int integrator, uint32_t max_depth, float exposure, const float* cams, uint32_t n_views,
                  uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, int mode, uint8_t* rgba, uint64_t counters[3]) {
  (void)nv;
  Mesh m;
  if (mesh_init(&m, xyz, rgb, tri, nf, mode)) { mesh_free(&m); return -1; }
  float lin[256], thr[255];
  oracle_render_tables(lin, thr);
  const float scale = (float)exp2((double)exposure);
  uint32_t P = 1; while (P < spp) P <<= 1;
  uint64_t c0 = 0, c1 = 0, c2 = 0;
  for (uint32_t v = 0; v < n_views; ++v) {
    const Cam* cam = (const Cam*)(cams + 15 * (size_t)v);
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : c0, c1, c2)
    for (uint32_t yy = 0; yy < h; ++yy) {
      float (*s)[4] = malloc(sizeof(float[4]) * P);
      for (uint32_t xx = 0; xx < w; ++xx) {
        const uint32_t x = x0 + xx, y = y0 + yy, pix = y * W + x;
        uint64_t cnt[3] = {0, 0, 0};
        for (uint32_t k = 0; k < P; ++k) {
          s[k][0] = s[k][1] = s[k][2] = s[k][3] = 0.f;
          if (k < spp) s[k][3] = (float)sample(&m, lin, cam, pix, x, y, k, integrator, max_depth, mode, s[k], cnt);
        }
        c0 += cnt[0]; c1 += cnt[1]; c2 += cnt[2];
        /* the fixed pairwise tree: for off = P/2 .. 1, s[i] += s[i + off] for i < off */
        for (uint32_t off = P >> 1; off; off >>= 1)
          for (uint32_t i = 0; i < off; ++i)
            for (int ch = 0; ch < 4; ++ch) s[i][ch] = s[i][ch] + s[i + off][ch];
        uint8_t* o = rgba + 4 * (((size_t)v * h + yy) * w + xx);
        for (int ch = 0; ch < 3; ++ch) {
          const float val = (s[0][ch] / (float)spp) * scale;
          int k = 0;
          while (k < 255 && thr[k] <= val) ++k;
          o[ch] = (uint8_t)k;
        }
        const uint32_t hits = (uint32_t)s[0][3];
        o[3] = (uint8_t)((510u * hits + spp) / (2u * spp));
      }
      free(s);
    }
  }
  counters[0] = c0; counters[1] = c1; counters[2] = c2;
  mesh_free(&m);
  return 0;
}

/* First hits of n rays (o, d: n*3) with tmin < t, no face skipped: face (UINT32_MAX for none) and t.  mode as above. */
int oracle_first_hits(const float* xyz, const uint32_t* tri, uint64_t nf, const float* o, const float* d, uint64_t n, float tmin,
                      int mode, uint32_t* face, float* t) {
  Mesh m;
  if (mesh_init(&m, xyz, NULL, tri, nf, mode)) { mesh_free(&m); return -1; }
#pragma omp parallel for schedule(dynamic, 64)
  for (uint64_t i = 0; i < n; ++i) {
    Ray r;
    for (int k = 0; k < 3; ++k) { r.o[k] = o[3 * i + k]; r.d[k] = d[3 * i + k]; }
    ray_prep(&r);
    const Hit h = trace(&m, &r, tmin, INFINITY, UINT32_MAX, mode);
    face[i] = h.face; t[i] = h.t;
  }
  mesh_free(&m);
  return 0;
}
