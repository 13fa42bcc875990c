/* TEST INFRASTRUCTURE — scalar CPU statement of the TSDF voxel-block integration.
 *
 * PARITY UNPINNED.  The reference tree contains NO TSDF source: reconstruction is done
 * by the external FriedLiver.exe (BundleFusion) / DepthSensing.exe (VoxelHashing)
 * binaries (/root/reference/Server/scan_processor.py:27-35,126,138), neither vendored
 * nor version-pinned (SURVEY.md §0 fact 2, §8c).  No golden vector, test or fixture in
 * the reference constrains any TSDF value.  This file is therefore the single source of
 * truth for the numerical spec written down in DESIGN.md §"TSDF spec v1"; the CUDA path
 * is compared against it (bit-exact where stated, since the spec is written in terms of
 * correctly-rounded IEEE binary32 operations and explicit fmaf()).
 *
 * In-tree statements this spec follows:
 *   parameters            Server/tools/recons/zParametersScanNet.txt:34-35,47-58
 *   back-projection       SensReader/c++/src/sensorData.h:1577-1578, filter.cu:87
 *   depth units / invalid sensorData.h:972-974 (value / depthShift, 0 = invalid)
 *   invalid pose          sensorData.h:382 (all -inf)
 *   block hash primes     external/mLib/include/core-util/sparseGrid3.h:14-17 (GPU side only)
 * Everything else (8^3 blocks, voxel {f32 sdf, rgb8, u8 weight}, ray-band allocation,
 * weighted running average) is the published VoxelHashing scheme (Niessner et al. 2013),
 * restated from the paper's description, not from source.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library.  Compile: -O2 -ffp-contract=off -mfma (fmaf must be fused).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct {
  float voxel_size, trunc_base, trunc_scale, depth_min, depth_max, max_integration_distance;
  uint32_t weight_sample, weight_max;
  uint32_t width, height;
  float depth_shift;
} oracle_tsdf_params;

typedef struct { float sdf; uint8_t r, g, b, w; } ovoxel;        /* 8 bytes */

typedef struct {
  oracle_tsdf_params p;
  /* open-addressing table: key -> block index */
  uint64_t cap; uint64_t* keys; int32_t* vals;
  /* block store */
  uint64_t n_blocks, blocks_cap; uint64_t* block_key; ovoxel* vox; uint32_t* touched_stamp;
  /* per-frame scratch */
  int32_t* touched; uint64_t n_touched, touched_cap; float* dm;
  uint32_t frame_no;
  /* counters */
  uint64_t last_updated, last_touched, total_updated, total_touched, frames_done, frames_skipped;
  int threads;
} oracle_tsdf;

#define EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
#define KEY_BIAS  (1 << 20)

static inline int key_ok(int x, int y, int z) {
  return x >= -KEY_BIAS && x < KEY_BIAS && y >= -KEY_BIAS && y < KEY_BIAS && z >= -KEY_BIAS && z < KEY_BIAS;
}
static inline uint64_t pack_key(int x, int y, int z) {
  return (uint64_t)(uint32_t)(x + KEY_BIAS) | ((uint64_t)(uint32_t)(y + KEY_BIAS) << 21) |
         ((uint64_t)(uint32_t)(z + KEY_BIAS) << 42);
}
static inline void unpack_key(uint64_t k, int32_t* xyz) {
  xyz[0] = (int32_t)(k & 0x1FFFFF) - KEY_BIAS;
  xyz[1] = (int32_t)((k >> 21) & 0x1FFFFF) - KEY_BIAS;
  xyz[2] = (int32_t)((k >> 42) & 0x1FFFFF) - KEY_BIAS;
}
static inline uint64_t mix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33; return k;
}

static void table_grow(oracle_tsdf* o) {
  uint64_t ncap = o->cap * 2;
  uint64_t* nk = (uint64_t*)malloc(ncap * 8); int32_t* nv = (int32_t*)malloc(ncap * 4);
  for (uint64_t i = 0; i < ncap; ++i) nk[i] = EMPTY_KEY;
  for (uint64_t i = 0; i < o->cap; ++i) if (o->keys[i] != EMPTY_KEY) {
    uint64_t s = mix64(o->keys[i]) & (ncap - 1);
    while (nk[s] != EMPTY_KEY) s = (s + 1) & (ncap - 1);
    nk[s] = o->keys[i]; nv[s] = o->vals[i];
  }
  free(o->keys); free(o->vals); o->keys = nk; o->vals = nv; o->cap = ncap;
}

/* find-or-create; marks the block touched for the current frame */
static void touch_block(oracle_tsdf* o, int bx, int by, int bz) {
  if (!key_ok(bx, by, bz)) return;
  const uint64_t key = pack_key(bx, by, bz);
  uint64_t s = mix64(key) & (o->cap - 1);
  while (o->keys[s] != EMPTY_KEY && o->keys[s] != key) s = (s + 1) & (o->cap - 1);
  int32_t idx;
  if (o->keys[s] == key) idx = o->vals[s];
  else {
    if (o->n_blocks == o->blocks_cap) {
      o->blocks_cap *= 2;
      o->block_key = (uint64_t*)realloc(o->block_key, o->blocks_cap * 8);
      o->vox = (ovoxel*)realloc(o->vox, o->blocks_cap * 512 * sizeof(ovoxel));
      o->touched_stamp = (uint32_t*)realloc(o->touched_stamp, o->blocks_cap * 4);
    }
    idx = (int32_t)o->n_blocks++;
    o->block_key[idx] = key;
    memset(o->vox + (size_t)idx * 512, 0, 512 * sizeof(ovoxel));
    o->touched_stamp[idx] = 0;
    o->keys[s] = key; o->vals[s] = idx;
    if (o->n_blocks * 2 > o->cap) table_grow(o);
  }
  if (o->touched_stamp[idx] != o->frame_no) {
    o->touched_stamp[idx] = o->frame_no;
    if (o->n_touched == o->touched_cap) {
      o->touched_cap *= 2; o->touched = (int32_t*)realloc(o->touched, o->touched_cap * 4);
    }
    o->touched[o->n_touched++] = idx;
  }
}

oracle_tsdf* oracle_tsdf_create(const oracle_tsdf_params* p, int threads) {
  oracle_tsdf* o = (oracle_tsdf*)calloc(1, sizeof(oracle_tsdf));
  o->p = *p;
  if (o->p.weight_max > 255) o->p.weight_max = 255;
  o->cap = 1 << 16; o->keys = (uint64_t*)malloc(o->cap * 8); o->vals = (int32_t*)malloc(o->cap * 4);
  for (uint64_t i = 0; i < o->cap; ++i) o->keys[i] = EMPTY_KEY;
  o->blocks_cap = 1 << 12;
  o->block_key = (uint64_t*)malloc(o->blocks_cap * 8);
  o->vox = (ovoxel*)malloc(o->blocks_cap * 512 * sizeof(ovoxel));
  o->touched_stamp = (uint32_t*)malloc(o->blocks_cap * 4);
  o->touched_cap = 1 << 12; o->touched = (int32_t*)malloc(o->touched_cap * 4);
  o->dm = (float*)malloc((size_t)p->width * p->height * 4);
  o->threads = threads > 0 ? threads : 1;
  return o;
}
void oracle_tsdf_destroy(oracle_tsdf* o) {
  if (!o) return;
  free(o->keys); free(o->vals); free(o->block_key); free(o->vox); free(o->touched_stamp);
  free(o->touched); free(o->dm); free(o);
}

/* Per-thread set of block keys seen by step B (the touched SET does not depend on order, so the pixel walks
 * may run on all host threads; the sets are merged into the table sequentially afterwards). */
typedef struct { uint64_t* slot; uint64_t cap; uint64_t* list; uint64_t n, list_cap; } keyset;
static void keyset_init(keyset* k) {
  k->cap = 1 << 12; k->slot = (uint64_t*)malloc(k->cap * 8);
  for (uint64_t i = 0; i < k->cap; ++i) k->slot[i] = EMPTY_KEY;
  k->list_cap = 1 << 11; k->list = (uint64_t*)malloc(k->list_cap * 8); k->n = 0;
}
static void keyset_free(keyset* k) { free(k->slot); free(k->list); }
static void keyset_add(keyset* k, int bx, int by, int bz) {
  if (!key_ok(bx, by, bz)) return;
  const uint64_t key = pack_key(bx, by, bz);
  uint64_t s = mix64(key) & (k->cap - 1);
  while (k->slot[s] != EMPTY_KEY) { if (k->slot[s] == key) return; s = (s + 1) & (k->cap - 1); }
  k->slot[s] = key;
  if (k->n == k->list_cap) { k->list_cap *= 2; k->list = (uint64_t*)realloc(k->list, k->list_cap * 8); }
  k->list[k->n++] = key;
  if (k->n * 2 > k->cap) {                                             /* grow + rehash */
    const uint64_t nc = k->cap * 2; uint64_t* ns = (uint64_t*)malloc(nc * 8);
    for (uint64_t i = 0; i < nc; ++i) ns[i] = EMPTY_KEY;
    for (uint64_t i = 0; i < k->n; ++i) { uint64_t q = mix64(k->list[i]) & (nc - 1); while (ns[q] != EMPTY_KEY) q = (q + 1) & (nc - 1); ns[q] = k->list[i]; }
    free(k->slot); k->slot = ns; k->cap = nc;
  }
}

/* ---- spec step B: ray-band block allocation for one pixel ---------------------------- */
static void alloc_pixel(const oracle_tsdf* o, keyset* ks, const float* T, float ifx, float ify, float cx, float cy,
                        float inv_bs, int x, int y, float d) {
  const oracle_tsdf_params* p = &o->p;
  if (!(d >= p->depth_min && d <= p->depth_max)) return;
  if (d >= p->max_integration_distance) return;
  const float tr = fmaf(p->trunc_scale, d, p->trunc_base);
  const float zmin = fminf(p->max_integration_distance, d - tr);
  const float zmax = fminf(p->max_integration_distance, d + tr);
  if (zmin >= zmax) return;
  const float rx = ((float)x - cx) * ifx, ry = ((float)y - cy) * ify;      /* ifx = 1/fx, ify = 1/fy */
  float A[3], Bp[3];
  for (int e = 0; e < 2; ++e) {
    const float Z = e ? zmax : zmin, X = rx * Z, Y = ry * Z;
    float* dst = e ? Bp : A;
    for (int i = 0; i < 3; ++i) {
      const float w = fmaf(T[4 * i + 2], Z, fmaf(T[4 * i + 1], Y, fmaf(T[4 * i + 0], X, T[4 * i + 3])));
      dst[i] = fmaf(w, inv_bs, 0.0625f);
    }
  }
  int cell[3], end[3], step[3]; float tmax[3], tdelta[3];
  for (int i = 0; i < 3; ++i) {
    cell[i] = (int)floorf(A[i]); end[i] = (int)floorf(Bp[i]);
    const float dir = Bp[i] - A[i];
    const float eps = 9.5367431640625e-07f;                        /* 2^-20: flatter than this = parallel to the axis */
    if (dir >= eps)       { const float inv = 1.0f / dir; step[i] = 1;  tmax[i] = ((float)(cell[i] + 1) - A[i]) * inv; tdelta[i] = inv; }
    else if (dir <= -eps) { const float inv = 1.0f / dir; step[i] = -1; tmax[i] = ((float)cell[i] - A[i]) * inv;       tdelta[i] = -inv; }
    else                  { step[i] = 0;  tmax[i] = INFINITY; tdelta[i] = INFINITY; }
  }
  for (int it = 0; it < 48; ++it) {
    keyset_add(ks, cell[0], cell[1], cell[2]);
    if (cell[0] == end[0] && cell[1] == end[1] && cell[2] == end[2]) return;
    int ax;
    if (tmax[0] <= tmax[1] && tmax[0] <= tmax[2]) ax = 0; else if (tmax[1] <= tmax[2]) ax = 1; else ax = 2;
    if (tmax[ax] > 1.0f) break;
    cell[ax] += step[ax];
    tmax[ax] += tdelta[ax];
  }
  keyset_add(ks, end[0], end[1], end[2]);
}

/* ---- spec step C: integrate one block ------------------------------------------------ */
static uint64_t integrate_block(oracle_tsdf* o, int32_t idx, const float* Rt, const float* tinv,
                                const float* Avs, float fx, float fy, float cx, float cy,
                                const uint8_t* rgb) {
  const oracle_tsdf_params* p = &o->p;
  const int W = (int)p->width, H = (int)p->height;
  int32_t b[3]; unpack_key(o->block_key[idx], b);
  float org[3], base[3];
  for (int i = 0; i < 3; ++i) org[i] = (float)(8 * b[i]) * p->voxel_size;
  for (int i = 0; i < 3; ++i)
    base[i] = fmaf(Rt[3 * i + 2], org[2], fmaf(Rt[3 * i + 1], org[1], fmaf(Rt[3 * i + 0], org[0], tinv[i])));
  const float inv_range = 1.0f / (p->depth_max - p->depth_min);
  const float ws15 = (float)p->weight_sample * 1.5f;
  ovoxel* vb = o->vox + (size_t)idx * 512;
  uint64_t n_upd = 0;
  for (int lz = 0; lz < 8; ++lz) for (int ly = 0; ly < 8; ++ly) for (int lx = 0; lx < 8; ++lx) {
    float pc[3];
    for (int i = 0; i < 3; ++i)
      pc[i] = fmaf((float)lz, Avs[3 * i + 2], fmaf((float)ly, Avs[3 * i + 1], fmaf((float)lx, Avs[3 * i + 0], base[i])));
    const float z = pc[2];
    if (!(z >= 0.015625f)) continue;                              /* 2^-6 m */
    const float rz = 1.0f / z;
    const float u = fmaf(pc[0] * rz, fx, cx), v = fmaf(pc[1] * rz, fy, cy);
    const long ix = lrintf(u), iy = lrintf(v);                 /* round-half-even */
    if (ix < 0 || ix >= W || iy < 0 || iy >= H) continue;
    const float d = o->dm[iy * W + ix];
    if (!(d >= p->depth_min && d <= p->depth_max)) continue;
    const float sdf = d - z;
    const float tr = fmaf(p->trunc_scale, d, p->trunc_base);
    if (!(sdf > -tr)) continue;
    const float s = fminf(sdf, tr);
    const float dz01 = (d - p->depth_min) * inv_range;
    const float wf = fmaxf(ws15 * (1.0f - dz01), 1.0f);
    const int w1 = (int)wf;
    ovoxel* vx = vb + (lz * 64 + ly * 8 + lx);
    const int w0 = vx->w, wsum = w0 + w1;
    const float inv = 1.0f / (float)wsum, w0f = (float)w0, w1f = (float)w1;
    vx->sdf = fmaf(vx->sdf, w0f, s * w1f) * inv;
    if (rgb) {
      const uint8_t* c1 = rgb + 3 * ((size_t)iy * W + ix);
      vx->r = (uint8_t)(int)(fmaf((float)vx->r, w0f, (float)c1[0] * w1f) * inv + 0.5f);
      vx->g = (uint8_t)(int)(fmaf((float)vx->g, w0f, (float)c1[1] * w1f) * inv + 0.5f);
      vx->b = (uint8_t)(int)(fmaf((float)vx->b, w0f, (float)c1[2] * w1f) * inv + 0.5f);
    }
    vx->w = (uint8_t)(wsum < (int)p->weight_max ? wsum : (int)p->weight_max);
    ++n_upd;
  }
  return n_upd;
}

/* One frame.  K is the 4x4 row-major depth intrinsic as stored in a .sens header
 * (sensorData.h:300-307): fx=K[0], cx=K[2], fy=K[5], cy=K[6].  Returns 1 if the frame was
 * skipped (invalid pose), 0 otherwise. */
static int integrate_dm(oracle_tsdf* o, const uint8_t* rgb, const float* T, const float* K);

int oracle_tsdf_integrate(oracle_tsdf* o, const uint16_t* depth, const uint8_t* rgb,
                          const float* T /*cam2world 16*/, const float* K /*16*/) {
  const oracle_tsdf_params* p = &o->p;
  const int W = (int)p->width, H = (int)p->height;
  o->last_updated = o->last_touched = 0;
  if (T[0] == -INFINITY) { o->frames_skipped++; return 1; }
  /* step A: depth in metres */
  for (int i = 0; i < W * H; ++i) o->dm[i] = depth[i] == 0 ? 0.0f : (float)depth[i] / p->depth_shift;
  return integrate_dm(o, rgb, T, K);
}

/* Same, from an already prepared metres image (-inf or 0 = invalid): the path taken when the depth map went through the
 * bilateral pre-filter first (the GPU-filtered image is handed in so that the comparison stays bit-exact). */
int oracle_tsdf_integrate_metres(oracle_tsdf* o, const float* metres, const uint8_t* rgb, const float* T, const float* K) {
  const int n = (int)o->p.width * (int)o->p.height;
  o->last_updated = o->last_touched = 0;
  if (T[0] == -INFINITY) { o->frames_skipped++; return 1; }
  for (int i = 0; i < n; ++i) o->dm[i] = metres[i] == -INFINITY ? 0.0f : metres[i];
  return integrate_dm(o, rgb, T, K);
}

static int integrate_dm(oracle_tsdf* o, const uint8_t* rgb, const float* T, const float* K) {
  const oracle_tsdf_params* p = &o->p;
  const int W = (int)p->width, H = (int)p->height;
  const float fx = K[0], cx = K[2], fy = K[5], cy = K[6];
  o->frame_no++;
  o->n_touched = 0;
  /* per-frame constants */
  float Rt[9], tinv[3], Avs[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[3 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; ++i)
    tinv[i] = -((Rt[3 * i + 0] * T[3] + Rt[3 * i + 1] * T[7]) + Rt[3 * i + 2] * T[11]);
  for (int i = 0; i < 9; ++i) Avs[i] = Rt[i] * p->voxel_size;
  const float inv_bs = 1.0f / (8.0f * p->voxel_size);
  const float ifx = 1.0f / fx, ify = 1.0f / fy;
  /* step B: pixel walks on all threads into per-thread key sets (the touched SET does not depend on order),
   * then one sequential merge into the table */
  {
    const int nth = o->threads;
    keyset* sets = (keyset*)malloc((size_t)nth * sizeof(keyset));
    for (int i = 0; i < nth; ++i) keyset_init(&sets[i]);
#pragma omp parallel num_threads(nth)
    {
#ifdef _OPENMP
      keyset* ks = &sets[omp_get_thread_num()];
#else
      keyset* ks = &sets[0];
#endif
#pragma omp for schedule(static)
      for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x)
        alloc_pixel(o, ks, T, ifx, ify, cx, cy, inv_bs, x, y, o->dm[y * W + x]);
    }
    for (int i = 0; i < nth; ++i) {
      for (uint64_t j = 0; j < sets[i].n; ++j) { int32_t b[3]; unpack_key(sets[i].list[j], b); touch_block(o, b[0], b[1], b[2]); }
      keyset_free(&sets[i]);
    }
    free(sets);
  }
  /* step C (blocks are independent) */
  uint64_t n_upd = 0;
  const int64_t nt = (int64_t)o->n_touched;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : n_upd) num_threads(o->threads)
  for (int64_t t = 0; t < nt; ++t)
    n_upd += integrate_block(o, o->touched[t], Rt, tinv, Avs, fx, fy, cx, cy, rgb);
  o->last_updated = n_upd; o->last_touched = o->n_touched;
  o->total_updated += n_upd; o->total_touched += o->n_touched; o->frames_done++;
  return 0;
}

uint64_t oracle_tsdf_num_blocks(const oracle_tsdf* o) { return o->n_blocks; }
void oracle_tsdf_counters(const oracle_tsdf* o, uint64_t* out /*6*/) {
  out[0] = o->last_updated; out[1] = o->last_touched; out[2] = o->total_updated;
  out[3] = o->total_touched; out[4] = o->frames_done; out[5] = o->frames_skipped;
}

static int cmp_u64idx(const void* a, const void* b) {
  const uint64_t x = ((const uint64_t*)a)[0], y = ((const uint64_t*)b)[0];
  return x < y ? -1 : (x > y ? 1 : 0);
}
/* Blocks sorted by packed key.  block_xyz: 3*n int32, voxels: n*512*8 bytes {f32 sdf, r,g,b,w}. */
void oracle_tsdf_export(const oracle_tsdf* o, int32_t* block_xyz, void* voxels) {
  const uint64_t n = o->n_blocks;
  uint64_t* ki = (uint64_t*)malloc((n ? n : 1) * 16);
  for (uint64_t i = 0; i < n; ++i) { ki[2 * i] = o->block_key[i]; ki[2 * i + 1] = i; }
  qsort(ki, n, 16, cmp_u64idx);
  for (uint64_t i = 0; i < n; ++i) {
    unpack_key(ki[2 * i], block_xyz + 3 * i);
    memcpy((char*)voxels + i * 4096, o->vox + ki[2 * i + 1] * 512, 4096);
  }
  free(ki);
}

/* The inverse of export: adds n blocks (layout as export) to the volume.  Returns -1 with the volume unchanged when a
 * coordinate is outside the key range or a block is given twice or already present, else 0. */
static int64_t find_block(const oracle_tsdf* o, uint64_t key) {
  uint64_t s = mix64(key) & (o->cap - 1);
  while (o->keys[s] != EMPTY_KEY && o->keys[s] != key) s = (s + 1) & (o->cap - 1);
  return o->keys[s] == key ? o->vals[s] : -1;
}
int oracle_tsdf_import(oracle_tsdf* o, const int32_t* block_xyz, const void* voxels, uint64_t n) {
  uint64_t* key = (uint64_t*)malloc((n ? n : 1) * 8);
  int bad = 0;
  for (uint64_t i = 0; i < n && !bad; ++i) {
    const int32_t* b = block_xyz + 3 * i;
    bad = !key_ok(b[0], b[1], b[2]);
    if (!bad) { key[i] = pack_key(b[0], b[1], b[2]); bad = find_block(o, key[i]) >= 0; }
  }
  if (!bad) {
    uint64_t* s = (uint64_t*)malloc((n ? n : 1) * 16);
    for (uint64_t i = 0; i < n; ++i) { s[2 * i] = key[i]; s[2 * i + 1] = i; }
    qsort(s, n, 16, cmp_u64idx);
    for (uint64_t i = 1; i < n && !bad; ++i) bad = s[2 * i] == s[2 * i - 2];
    free(s);
  }
  for (uint64_t i = 0; i < n && !bad; ++i) {
    const int32_t* b = block_xyz + 3 * i;
    touch_block(o, b[0], b[1], b[2]);                                  /* creates the block (zeroed) */
    memcpy(o->vox + (size_t)find_block(o, key[i]) * 512, (const char*)voxels + i * 4096, 4096);
  }
  o->n_touched = 0;                                                    /* the import is not a frame */
  free(key);
  return bad ? -1 : 0;
}

/* ------------------------------------------------------------------ marching cubes (DESIGN.md §6) -----
 * Own spec (the reference's meshing lives in the external binaries).  Independent statement of the rules
 * the product implements in csrc/mc.cu: usable voxels, valid cubes, lattice-edge vertices, a 256-case
 * table built by face-contour linking, deterministic ordering, dropped unreferenced vertices. */
static const ovoxel* vox_at(const oracle_tsdf* o, int gx, int gy, int gz) {
  const int bx = gx >> 3, by = gy >> 3, bz = gz >> 3;                 /* arithmetic shift = floor division by 8 */
  if (!key_ok(bx, by, bz)) return NULL;
  const uint64_t key = pack_key(bx, by, bz);
  uint64_t s = mix64(key) & (o->cap - 1);
  while (o->keys[s] != EMPTY_KEY && o->keys[s] != key) s = (s + 1) & (o->cap - 1);
  if (o->keys[s] != key) return NULL;
  return o->vox + (size_t)o->vals[s] * 512 + ((gx & 7) | ((gy & 7) << 3) | ((gz & 7) << 6));
}
static int vox_usable(const ovoxel* v, float thr) { return v && v->w > 0 && fabsf(v->sdf) <= thr; }

static int edge_of(int c0, int c1) {                                   /* edge id = axis*4 + (u | v<<1) */
  const int d = c0 ^ c1, a = d == 1 ? 0 : (d == 2 ? 1 : 2), lo = c0 & ~d;
  const int c[3] = { lo & 1, (lo >> 1) & 1, (lo >> 2) & 1 };
  const int u = c[a == 0 ? 1 : 0], v = c[a == 2 ? 1 : 2];
  return a * 4 + (u | (v << 1));
}
static void make_case(int cs, int* ntri, int tri[36]) {
  int next[12], seen[12], nt = 0;
  for (int i = 0; i < 12; ++i) { next[i] = -1; seen[i] = 0; }
  for (int a = 0; a < 3; ++a) for (int s = 0; s < 2; ++s) {
    const int b = (a + 1) % 3, c = (a + 2) % 3;
    int p[4];
    /* face corners counter-clockwise seen from outside the cube */
    const int vb[2][4] = { {0, 0, 1, 1}, {0, 1, 1, 0} }, vc[2][4] = { {0, 1, 1, 0}, {0, 0, 1, 1} };
    for (int k = 0; k < 4; ++k) { int off[3]; off[a] = s; off[b] = vb[s][k]; off[c] = vc[s][k]; p[k] = off[0] | (off[1] << 1) | (off[2] << 2); }
    for (int k = 0; k < 4; ++k) {
      const int prev = (k + 3) & 3;
      if (((cs >> p[prev]) & 1) || !((cs >> p[k]) & 1)) continue;       /* k starts a run of inside corners */
      int m = k;
      while ((cs >> p[(m + 1) & 3]) & 1) m = (m + 1) & 3;
      next[edge_of(p[prev], p[k])] = edge_of(p[m], p[(m + 1) & 3]);     /* entering edge -> leaving edge */
    }
  }
  for (int e0 = 0; e0 < 12; ++e0) {
    if (next[e0] < 0 || seen[e0]) continue;
    int loop[12], n = 0;
    for (int e = e0; !seen[e]; e = next[e]) { seen[e] = 1; loop[n++] = e; }
    for (int i = 1; i + 1 < n; ++i) { tri[3 * nt] = loop[0]; tri[3 * nt + 1] = loop[i]; tri[3 * nt + 2] = loop[i + 1]; ++nt; }
  }
  *ntri = nt;
}

void oracle_mc_table(uint8_t* ntri_out /*256*/, uint8_t* tri_out /*256*36*/) {
  for (int cs = 0; cs < 256; ++cs) {
    int nt, tri[36];
    make_case(cs, &nt, tri);
    ntri_out[cs] = (uint8_t)nt;
    for (int i = 0; i < 36; ++i) tri_out[cs * 36 + i] = (uint8_t)(i < 3 * nt ? tri[i] : 0);
  }
}

/* Returns malloc'ed arrays (free with oracle_free). */
void oracle_tsdf_extract_mesh(const oracle_tsdf* o, float thresh_factor, float** xyz_out, uint8_t** rgb_out,
                              uint32_t** tri_out, uint64_t* nv_out, uint64_t* nf_out) {
  const uint64_t n = o->n_blocks;
  const float vs = o->p.voxel_size;
  const float thr = thresh_factor * vs;
  uint64_t* ki = (uint64_t*)malloc((n ? n : 1) * 16);
  for (uint64_t i = 0; i < n; ++i) { ki[2 * i] = o->block_key[i]; ki[2 * i + 1] = i; }
  qsort(ki, n, 16, cmp_u64idx);
  /* rank of each heap index in key order */
  uint32_t* rank = (uint32_t*)malloc((n ? n : 1) * 4);
  for (uint64_t j = 0; j < n; ++j) rank[ki[2 * j + 1]] = (uint32_t)j;
  int64_t* vid = (int64_t*)malloc((n ? n : 1) * 512 * 3 * sizeof(int64_t));
  size_t capv = 1 << 16, nv = 0;
  float* pos = (float*)malloc(capv * 12); uint8_t* col = (uint8_t*)malloc(capv * 3);
  /* vertices */
  for (uint64_t j = 0; j < n; ++j) {
    int32_t b[3]; unpack_key(ki[2 * j], b);
    for (int l = 0; l < 512; ++l) {
      const int g[3] = { 8 * b[0] + (l & 7), 8 * b[1] + ((l >> 3) & 7), 8 * b[2] + (l >> 6) };
      const ovoxel* v0 = vox_at(o, g[0], g[1], g[2]);
      for (int a = 0; a < 3; ++a) {
        int64_t id = -1;
        const ovoxel* v1 = vox_at(o, g[0] + (a == 0), g[1] + (a == 1), g[2] + (a == 2));
        if (vox_usable(v0, thr) && vox_usable(v1, thr) && ((v0->sdf < 0.0f) != (v1->sdf < 0.0f))) {
          if (nv == capv) { capv *= 2; pos = (float*)realloc(pos, capv * 12); col = (uint8_t*)realloc(col, capv * 3); }
          const float t = v0->sdf / (v0->sdf - v1->sdf);
          for (int i = 0; i < 3; ++i) pos[3 * nv + i] = (i == a ? (float)g[i] + t : (float)g[i]) * vs;
          const uint8_t c0[3] = { v0->r, v0->g, v0->b }, c1[3] = { v1->r, v1->g, v1->b };
          for (int ch = 0; ch < 3; ++ch)
            col[3 * nv + ch] = (uint8_t)(int)(fmaf(t, (float)c1[ch] - (float)c0[ch], (float)c0[ch]) + 0.5f);
          id = (int64_t)nv++;
        }
        vid[(j * 512 + l) * 3 + a] = id;
      }
    }
  }
  /* triangles */
  size_t capt = 1 << 16, nt = 0;
  uint32_t* tri = (uint32_t*)malloc(capt * 12);
  uint8_t* used = (uint8_t*)calloc(nv ? nv : 1, 1);
  static uint8_t T_n[256], T_t[256 * 36]; oracle_mc_table(T_n, T_t);
  for (uint64_t j = 0; j < n; ++j) {
    int32_t b[3]; unpack_key(ki[2 * j], b);
    for (int l = 0; l < 512; ++l) {
      const int g[3] = { 8 * b[0] + (l & 7), 8 * b[1] + ((l >> 3) & 7), 8 * b[2] + (l >> 6) };
      int cs = 0, ok = 1;
      for (int c = 0; c < 8 && ok; ++c) {
        const ovoxel* v = vox_at(o, g[0] + (c & 1), g[1] + ((c >> 1) & 1), g[2] + (c >> 2));
        if (!vox_usable(v, thr)) ok = 0; else if (v->sdf < 0.0f) cs |= 1 << c;
      }
      if (!ok) continue;
      for (int k = 0; k < T_n[cs]; ++k) {
        if (nt == capt) { capt *= 2; tri = (uint32_t*)realloc(tri, capt * 12); }
        for (int q = 0; q < 3; ++q) {
          const int e = T_t[cs * 36 + 3 * k + q], a = e >> 2, u = e & 1, v = (e >> 1) & 1;
          int off[3];
          if (a == 0) { off[0] = 0; off[1] = u; off[2] = v; } else if (a == 1) { off[0] = u; off[1] = 0; off[2] = v; } else { off[0] = u; off[1] = v; off[2] = 0; }
          const int h[3] = { g[0] + off[0], g[1] + off[1], g[2] + off[2] };
          const uint64_t key = pack_key(h[0] >> 3, h[1] >> 3, h[2] >> 3);
          uint64_t s = mix64(key) & (o->cap - 1);
          while (o->keys[s] != key) s = (s + 1) & (o->cap - 1);
          const uint64_t jj = rank[o->vals[s]];
          const int64_t id = vid[(jj * 512 + ((h[0] & 7) | ((h[1] & 7) << 3) | ((h[2] & 7) << 6))) * 3 + a];
          tri[3 * nt + q] = (uint32_t)id; used[id] = 1;
        }
        ++nt;
      }
    }
  }
  /* drop unreferenced vertices, keep order */
  uint32_t* newid = (uint32_t*)malloc((nv ? nv : 1) * 4);
  size_t nv2 = 0;
  for (size_t i = 0; i < nv; ++i) if (used[i]) {
    newid[i] = (uint32_t)nv2;
    memmove(pos + 3 * nv2, pos + 3 * i, 12); memmove(col + 3 * nv2, col + 3 * i, 3); ++nv2;
  }
  for (size_t i = 0; i < 3 * nt; ++i) tri[i] = newid[tri[i]];
  free(newid); free(used); free(vid); free(rank); free(ki);
  *xyz_out = pos; *rgb_out = col; *tri_out = tri; *nv_out = nv2; *nf_out = nt;
}
void oracle_free(void* p) { free(p); }


/* ------------------------------------------------------------------ depth bilateral filter --------------------
 * Restatement of bilateralFilterFloatMapDevice, /root/reference/AnnotationTools/Filter2dAnnotations/filter.cu:210-247
 * (gaussD :201-204 in float, gaussR :191-194 in double), fed as Filter2dAnnotations.cpp:245-256 feeds it
 * (0 -> -inf, else raw / depthShift).  The reference is a CUDA kernel; exp/expf here are libm's, so the CUDA kernel in
 * scannet_b200/csrc/filter.cu is compared to a tolerance, not bit for bit. */
void oracle_bilateral_filter(const uint16_t* depth, int W, int H, float depth_shift, float sigmaD, float sigmaR, float* out) {
  float* in = (float*)malloc((size_t)W * H * 4);
  for (int i = 0; i < W * H; ++i) in[i] = depth[i] == 0 ? -INFINITY : (float)depth[i] / depth_shift;
  const int r = (int)ceil(2.0 * sigmaD);
  for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) {
    float res = -INFINITY, sum = 0.0f, sumw = 0.0f;
    const float c = in[y * W + x];
    if (c != -INFINITY) {
      for (int m = x - r; m <= x + r; ++m) for (int n = y - r; n <= y + r; ++n) {
        if (m < 0 || n < 0 || m >= W || n >= H) continue;
        const float cur = in[n * W + m];
        if (cur == -INFINITY) continue;
        const int dx = m - x, dy = n - y;
        const float gd = expf(-((float)(dx * dx + dy * dy) / (2.0f * sigmaD * sigmaD)));
        const float dd = cur - c;
        const float gr = (float)exp(-(dd * dd) / (2.0 * sigmaR * sigmaR));
        const float w = gd * gr;
        sumw += w;
        sum = fmaf(w, cur, sum);
      }
      if (sumw > 0.0f) res = sum / sumw;
    }
    out[y * W + x] = res;
  }
  free(in);
}
