/* TEST INFRASTRUCTURE — not product code.
 *
 * Sequential CPU statement of the mesh-cleaning stage, DESIGN.md §6f: the mLib MeshData operators
 * (external/mLib/include/core-mesh/meshData.cpp) in the order of MeshLab's clean.mlx.
 *   merge   mergeCloseVertices(t, approx=false) :217-289, then removeDegeneratedFaces :293-318
 *   dedup   removeDuplicateFaces :40-104
 *   pieces  removeIsolatedPieces :407-454 (vertex count), a face-count threshold on the same pieces, then
 *           removeIsolatedVertices :324-360 (first-appearance renumbering)
 * All arithmetic is binary32 with contraction off (oracle/meshclean.mk: -ffp-contract=off).
 * The merge and dedup steps are pinned against the unmodified mLib code in the CPU suite (oracle/ref_shim_meshdata.cpp). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define CLEAN_SKIP_MERGE 1u
#define CLEAN_SKIP_DEDUP 2u
#define CLEAN_SKIP_PIECES 4u

/* counters[]: the integer fields of scn_mesh_clean_report_t after the four size fields, in order */
enum { C_MERGED, C_MERGE_COMPONENTS, C_LARGEST, C_DEGENERATE, C_DUPLICATE, C_PIECES, C_PIECES_REMOVED, C_FACES_REMOVED, C_N };

/* ---- open-addressing hash of 3-int keys -> value (cell -> list head, sorted triple -> seen) ---- */
typedef struct { int64_t k[3]; int64_t v; int used; } Slot;
typedef struct { Slot* s; uint64_t mask; } Hash;

static uint64_t hkey(const int64_t* k) {
  uint64_t h = (uint64_t)k[0] * 0x9E3779B97F4A7C15ull;
  h ^= (uint64_t)k[1] * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
  h ^= (uint64_t)k[2] * 0x165667B19E3779F9ull + (h << 6) + (h >> 2);
  return h ^ (h >> 29);
}
static int hash_init(Hash* h, uint64_t n) {
  uint64_t cap = 16; while (cap < 2 * n + 16) cap <<= 1;
  h->s = (Slot*)calloc(cap, sizeof(Slot)); h->mask = cap - 1;
  return h->s != NULL;
}
/* returns the slot for k; *found = whether it existed (a new slot is marked used with v = -1) */
static Slot* hash_get(Hash* h, const int64_t* k, int* found) {
  uint64_t i = hkey(k) & h->mask;
  for (;;) {
    Slot* s = &h->s[i];
    if (!s->used) { s->used = 1; memcpy(s->k, k, sizeof(s->k)); s->v = -1; *found = 0; return s; }
    if (s->k[0] == k[0] && s->k[1] == k[1] && s->k[2] == k[2]) { *found = 1; return s; }
    i = (i + 1) & h->mask;
  }
}
static Slot* hash_find(const Hash* h, const int64_t* k) {
  uint64_t i = hkey(k) & h->mask;
  for (;;) {
    Slot* s = &h->s[i];
    if (!s->used) return NULL;
    if (s->k[0] == k[0] && s->k[1] == k[1] && s->k[2] == k[2]) return s;
    i = (i + 1) & h->mask;
  }
}

static int64_t uf_find(int64_t* p, int64_t x) {
  while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; }
  return x;
}
static void uf_union(int64_t* p, int64_t a, int64_t b) {
  a = uf_find(p, a); b = uf_find(p, b);
  if (a == b) return;
  if (a < b) p[b] = a; else p[a] = b;
}

static float dist_sq(const float* a, const float* b) {              /* vec3::distSq, vec3.h:199-201 */
  const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return (dx * dx + dy * dy) + dz * dz;
}

/* toVirtualVoxelPos (meshData.h:946-948): (int)(v * (1/t) + 0.5f * sign(v)); returns 0 when the conversion is undefined */
static int cell_of(const float* v, float inv, int64_t* c) {
  for (int i = 0; i < 3; ++i) {
    const float s = v[i] * inv;
    if (!(fabsf(s) < 2147483648.0f)) return 0;
    const float sg = (float)((0.f < v[i]) - (v[i] < 0.f));
    c[i] = (int)(s + 0.5f * sg);
  }
  return 1;
}

/* Step 1. Writes the representatives to (xyz, rgb) in place, remaps and filters tri in place. */
static int merge(float* xyz, uint8_t* rgb, int64_t* nV, uint32_t* tri, int64_t* nF, float t, uint64_t* cnt) {
  const int64_t n = *nV;
  const float inv = 1.0f / t, tsq = t * t;
  int64_t* cell = (int64_t*)malloc((size_t)(n ? n : 1) * 3 * sizeof(int64_t));
  int64_t* next = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));     /* representative list of a cell, in insertion order */
  int64_t* tail = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));
  int64_t* lookup = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));   /* vertex -> representative (old index) */
  int64_t* newid = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));
  int64_t* par = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));
  int64_t* csize = (int64_t*)calloc((size_t)(n ? n : 1), sizeof(int64_t));
  Hash all = {0}, reps = {0};
  int rc = 0;
  if (!cell || !next || !tail || !lookup || !newid || !par || !csize || !hash_init(&all, (uint64_t)n) || !hash_init(&reps, (uint64_t)n)) { rc = -2; goto out; }
  for (int64_t v = 0; v < n; ++v) if (!cell_of(xyz + 3 * v, inv, cell + 3 * v)) { rc = -1; goto out; }
  /* the rule itself: representatives only, mLib's scan order (x offset outermost, then y, then z; a cell's list in insertion order) */
  int64_t cntv = 0;
  for (int64_t v = 0; v < n; ++v) {
    int64_t nn = -1;
    for (int i = -1; i <= 1 && nn < 0; ++i)
      for (int j = -1; j <= 1 && nn < 0; ++j)
        for (int k = -1; k <= 1 && nn < 0; ++k) {
          const int64_t c[3] = {cell[3 * v] + i, cell[3 * v + 1] + j, cell[3 * v + 2] + k};
          const Slot* s = hash_find(&reps, c);
          if (!s) continue;
          for (int64_t r = s->v; r >= 0; r = next[r])
            if (dist_sq(xyz + 3 * v, xyz + 3 * r) < tsq) { nn = r; break; }
        }
    if (nn < 0) {
      int found; Slot* s = hash_get(&reps, cell + 3 * v, &found);
      next[v] = -1;
      if (!found) s->v = v; else next[tail[s->v]] = v;
      tail[s->v] = v;
      lookup[v] = v; newid[v] = cntv++;
    } else lookup[v] = nn;
  }
  /* report: components of the proximity graph (pairs in neighbouring cells with d^2 < t^2), over ALL vertices */
  for (int64_t v = 0; v < n; ++v) par[v] = v;
  {
    for (int64_t v = 0; v < n; ++v) {
      int found; Slot* s = hash_get(&all, cell + 3 * v, &found);
      next[v] = -1;
      if (!found) s->v = v; else next[tail[s->v]] = v;
      tail[s->v] = v;
    }
    for (int64_t v = 0; v < n; ++v)
      for (int i = -1; i <= 1; ++i) for (int j = -1; j <= 1; ++j) for (int k = -1; k <= 1; ++k) {
        const int64_t c[3] = {cell[3 * v] + i, cell[3 * v + 1] + j, cell[3 * v + 2] + k};
        const Slot* s = hash_find(&all, c);
        if (!s) continue;
        for (int64_t u = s->v; u >= 0 && u < v; u = next[u])
          if (dist_sq(xyz + 3 * v, xyz + 3 * u) < tsq) uf_union(par, u, v);
      }
    uint64_t ncomp = 0, largest = 0;
    for (int64_t v = 0; v < n; ++v) csize[uf_find(par, v)]++;
    for (int64_t v = 0; v < n; ++v) if (par[v] == v) { if (csize[v] >= 2) ++ncomp; if ((uint64_t)csize[v] > largest) largest = (uint64_t)csize[v]; }
    cnt[C_MERGE_COMPONENTS] = ncomp; cnt[C_LARGEST] = largest;
  }
  cnt[C_MERGED] = (uint64_t)(n - cntv);
  for (int64_t v = 0; v < n; ++v) if (lookup[v] == v) {                 /* ascending: newid[v] <= v, so in place is safe */
    const int64_t d = newid[v];
    memmove(xyz + 3 * d, xyz + 3 * v, 12);
    if (rgb) memmove(rgb + 3 * d, rgb + 3 * v, 3);
  }
  int64_t f2 = 0;
  for (int64_t f = 0; f < *nF; ++f) {
    const uint32_t a = (uint32_t)newid[lookup[tri[3 * f]]], b = (uint32_t)newid[lookup[tri[3 * f + 1]]], c = (uint32_t)newid[lookup[tri[3 * f + 2]]];
    if (a == b || a == c || b == c) continue;                           /* removeDegeneratedFaces */
    tri[3 * f2] = a; tri[3 * f2 + 1] = b; tri[3 * f2 + 2] = c; ++f2;
  }
  cnt[C_DEGENERATE] = (uint64_t)(*nF - f2);
  *nV = cntv; *nF = f2;
out:
  free(cell); free(next); free(tail); free(lookup); free(newid); free(par); free(csize);
  if (all.s) free(all.s);
  if (reps.s) free(reps.s);
  return rc;
}

/* Step 2: the first face (current order) of every sorted index triple survives, corners untouched. */
static int dedup(uint32_t* tri, int64_t* nF, uint64_t* cnt) {
  Hash h;
  if (!hash_init(&h, (uint64_t)*nF)) return -2;
  int64_t f2 = 0;
  for (int64_t f = 0; f < *nF; ++f) {
    int64_t k[3] = {tri[3 * f], tri[3 * f + 1], tri[3 * f + 2]}, x;
    if (k[0] > k[1]) { x = k[0]; k[0] = k[1]; k[1] = x; }
    if (k[1] > k[2]) { x = k[1]; k[1] = k[2]; k[2] = x; }
    if (k[0] > k[1]) { x = k[0]; k[0] = k[1]; k[1] = x; }
    int found; hash_get(&h, k, &found);
    if (found) continue;
    memmove(tri + 3 * f2, tri + 3 * f, 12); ++f2;
  }
  free(h.s);
  cnt[C_DUPLICATE] = (uint64_t)(*nF - f2);
  *nF = f2;
  return 0;
}

/* Step 3: pieces = connected components of the vertex graph (a face links its corners); renumber by first appearance. */
static int pieces(float* xyz, uint8_t* rgb, int64_t* nV, uint32_t* tri, int64_t* nF, uint32_t min_v, uint32_t min_f, uint64_t* cnt) {
  const int64_t n = *nV;
  int64_t* par = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));
  int64_t* vc = (int64_t*)calloc((size_t)(n ? n : 1), sizeof(int64_t));
  int64_t* fc = (int64_t*)calloc((size_t)(n ? n : 1), sizeof(int64_t));
  int64_t* map = (int64_t*)malloc((size_t)(n ? n : 1) * sizeof(int64_t));
  float* nx = (float*)malloc((size_t)(n ? n : 1) * 12);
  uint8_t* nc = (uint8_t*)malloc((size_t)(n ? n : 1) * 3);
  int rc = 0;
  if (!par || !vc || !fc || !map || !nx || !nc) { rc = -2; goto out; }
  for (int64_t v = 0; v < n; ++v) par[v] = v;
  for (int64_t f = 0; f < *nF; ++f) { uf_union(par, tri[3 * f], tri[3 * f + 1]); uf_union(par, tri[3 * f], tri[3 * f + 2]); }
  for (int64_t v = 0; v < n; ++v) vc[uf_find(par, v)]++;
  for (int64_t f = 0; f < *nF; ++f) fc[uf_find(par, tri[3 * f])]++;
  for (int64_t v = 0; v < n; ++v) if (par[v] == v && fc[v] > 0) {
    cnt[C_PIECES]++;
    if (vc[v] < (int64_t)min_v || fc[v] < (int64_t)min_f) { cnt[C_PIECES_REMOVED]++; cnt[C_FACES_REMOVED] += (uint64_t)fc[v]; }
  }
  int64_t f2 = 0, v2 = 0;
  for (int64_t v = 0; v < n; ++v) map[v] = -1;
  for (int64_t f = 0; f < *nF; ++f) {
    const int64_t r = uf_find(par, tri[3 * f]);
    if (vc[r] < (int64_t)min_v || fc[r] < (int64_t)min_f) continue;
    for (int k = 0; k < 3; ++k) {
      const uint32_t v = tri[3 * f + k];
      if (map[v] < 0) { map[v] = v2; memcpy(nx + 3 * v2, xyz + 3 * v, 12); if (rgb) memcpy(nc + 3 * v2, rgb + 3 * v, 3); ++v2; }
      tri[3 * f2 + k] = (uint32_t)map[v];
    }
    ++f2;
  }
  memcpy(xyz, nx, (size_t)v2 * 12);
  if (rgb) memcpy(rgb, nc, (size_t)v2 * 3);
  *nV = v2; *nF = f2;
out:
  free(par); free(vc); free(fc); free(map); free(nx); free(nc);
  return rc;
}

/* The whole stage.  Outputs are caller-owned with room for nV vertices and nF faces (the stage never grows the mesh);
 * rgb / rgb_out may be NULL.  Returns 0, -1 for the inputs the library refuses with SCN_ERR_ARG, -2 out of memory. */
int oracle_mesh_clean(const float* xyz, const uint8_t* rgb, int64_t nV, const uint32_t* tri, int64_t nF, float t, uint32_t min_v,
                      uint32_t min_f, uint32_t flags, float* xyz_out, uint8_t* rgb_out, uint32_t* tri_out, int64_t* nV_out,
                      int64_t* nF_out, uint64_t* counters) {
  memset(counters, 0, C_N * sizeof(uint64_t));
  for (int64_t c = 0; c < 3 * nF; ++c) if ((int64_t)tri[c] >= nV) return -1;
  if (!(flags & CLEAN_SKIP_MERGE) && !(t > 0.f)) return -1;
  if (nV) memcpy(xyz_out, xyz, (size_t)nV * 12);
  if (nV && rgb && rgb_out) memcpy(rgb_out, rgb, (size_t)nV * 3);
  if (nF) memcpy(tri_out, tri, (size_t)nF * 12);
  uint8_t* c = rgb && rgb_out ? rgb_out : NULL;
  int rc = 0;
  if (!(flags & CLEAN_SKIP_MERGE)) rc = merge(xyz_out, c, &nV, tri_out, &nF, t, counters);
  if (!rc && !(flags & CLEAN_SKIP_DEDUP)) rc = dedup(tri_out, &nF, counters);
  if (!rc && !(flags & CLEAN_SKIP_PIECES)) rc = pieces(xyz_out, c, &nV, tri_out, &nF, min_v, min_f, counters);
  *nV_out = nV; *nF_out = nF;
  return rc;
}
