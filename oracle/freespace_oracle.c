/* TEST INFRASTRUCTURE — scalar CPU statement of free-space spec v1 (DESIGN.md §6h): per-voxel counts of free and occupied
 * observations over a dense lattice box.
 *
 * PARITY UNPINNED.  The reference pipeline's `freespace` stage calls the external FreeSpace.exe
 * (/root/reference/Server/scan_processor.py:150-152, Server/config.py:20), whose source is not in the tree; no golden vector,
 * test or fixture constrains its output.  This file is the single source of truth for the spec; the CUDA path
 * (scannet_b200/csrc/freespace.cu) is compared against it bit for bit.  Every voxel of the box is tested against every frame
 * (no culling), one OpenMP thread per z slice.
 *
 * The projection is TSDF spec step C (oracle/tsdf_oracle.c:integrate_block), with the pixel rounded by rintf and the image test
 * made on the rounded value.  Compile: -O2 -ffp-contract=off -mfma (fmaf must be fused).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {                 /* same layout as scn_freespace_params */
  float voxel_size, band_base, band_scale, depth_min, depth_max, max_distance;
  uint64_t max_voxels;
} oracle_fs_params;

/* Adds the observations of n frames (depth n*W*H u16, poses n*16 row-major cam2world, K the 4x4 depth intrinsic) to
 * n_free / n_occ over the box lo .. lo+dims-1 (x fastest).  Frames with cam2world[0] == -inf are skipped.  Returns the number
 * of frames used. */
uint32_t oracle_freespace_integrate(const oracle_fs_params* p, uint32_t W, uint32_t H, float depth_shift, const int32_t* lo,
                                    const uint64_t* dims, uint32_t n, const uint16_t* depth, const float* poses, const float* K,
                                    uint32_t* n_free, uint32_t* n_occ, int threads) {
  const size_t px = (size_t)W * H;
  float* dm = (float*)malloc((px ? px : 1) * sizeof(float));
  const float fx = K[0], cx = K[2], fy = K[5], cy = K[6], vs = p->voxel_size;
  uint32_t used = 0;
  for (uint32_t f = 0; f < n; ++f) {
    const float* T = poses + 16 * (size_t)f;
    if (T[0] == -INFINITY) continue;                                 /* sensorData.h:382 */
    ++used;
    /* step A: metres, NaN for raw 0 and outside [depth_min, depth_max] */
    const uint16_t* D = depth + (size_t)f * px;
    for (size_t i = 0; i < px; ++i) {
      const float d = D[i] == 0 ? NAN : (float)D[i] / depth_shift;
      dm[i] = (d >= p->depth_min && d <= p->depth_max) ? d : NAN;
    }
    float Rt[9], tinv[3], Avs[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[3 * i + j] = T[4 * j + i];
    for (int i = 0; i < 3; ++i) tinv[i] = -((Rt[3 * i + 0] * T[3] + Rt[3 * i + 1] * T[7]) + Rt[3 * i + 2] * T[11]);
    for (int i = 0; i < 9; ++i) Avs[i] = Rt[i] * vs;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 0 ? threads : 1)
    for (int64_t ez = 0; ez < (int64_t)dims[2]; ++ez) {
      for (uint64_t ey = 0; ey < dims[1]; ++ey) for (uint64_t ex = 0; ex < dims[0]; ++ex) {
        const int32_t g[3] = { lo[0] + (int32_t)ex, lo[1] + (int32_t)ey, lo[2] + (int32_t)ez };
        float o[3], l[3], base[3], pc[3];
        for (int a = 0; a < 3; ++a) { const int32_t b = g[a] >> 3; o[a] = (float)(8 * b) * vs; l[a] = (float)(g[a] & 7); }
        for (int i = 0; i < 3; ++i) base[i] = fmaf(Rt[3 * i + 2], o[2], fmaf(Rt[3 * i + 1], o[1], fmaf(Rt[3 * i + 0], o[0], tinv[i])));
        for (int i = 0; i < 3; ++i) pc[i] = fmaf(l[2], Avs[3 * i + 2], fmaf(l[1], Avs[3 * i + 1], fmaf(l[0], Avs[3 * i + 0], base[i])));
        const float z = pc[2];
        if (!(z >= 0.015625f)) continue;                             /* 2^-6 m */
        const float rz = 1.0f / z;
        const float ur = rintf(fmaf(pc[0] * rz, fx, cx)), vr = rintf(fmaf(pc[1] * rz, fy, cy));   /* round half to even */
        if (!(ur >= 0.0f && ur < (float)W && vr >= 0.0f && vr < (float)H)) continue;
        const float d = dm[(size_t)vr * W + (size_t)ur];
        if (!(d == d)) continue;
        const float s = d - z, band = fmaf(p->band_scale, d, p->band_base);
        const size_t v = ((size_t)ez * dims[1] + ey) * dims[0] + ex;
        if (s > band) { if (z < p->max_distance) n_free[v]++; }     /* free: in front of the band, z < max_distance */
        else if (s > -band && d < p->max_distance) n_occ[v]++;       /* occupied: inside the band, d < max_distance */
      }
    }
  }
  free(dm);
  return used;
}
