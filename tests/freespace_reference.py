"""Free-space spec v1 (DESIGN.md §6h) stated independently in float64 numpy, for checking the C oracle.  Besides the counts it
marks every voxel for which some frame's deciding quantity lies within eps of a threshold (the binary32 oracle may decide those
differently): the near plane, a pixel rounding boundary (the image edges are such boundaries), the depth range, the band edges
and max_distance."""
from __future__ import annotations

import numpy as np


def counts_f64(params, lo, dims, width, height, depth, poses, K, depth_shift=1000.0, eps_m=1e-4, eps_px=2e-3):
    """(n_free, n_occ, ambiguous) over the box, arrays [z, y, x]"""
    vs = float(params.voxel_size)
    bb, bs = float(params.band_base), float(params.band_scale)
    dmin, dmax, md = float(params.depth_min), float(params.depth_max), float(params.max_distance)
    fx, cx, fy, cy = float(K[0, 0]), float(K[0, 2]), float(K[1, 1]), float(K[1, 2])
    nx, ny, nz = (int(x) for x in dims)
    gz, gy, gx = np.meshgrid(np.arange(nz) + lo[2], np.arange(ny) + lo[1], np.arange(nx) + lo[0], indexing="ij")
    world = np.stack([gx, gy, gz], -1).reshape(-1, 3).astype(np.float64) * vs
    n_free = np.zeros(len(world), np.uint32); n_occ = np.zeros(len(world), np.uint32); amb = np.zeros(len(world), bool)
    for f in range(len(poses)):
        T = np.asarray(poses[f], np.float64)
        if T[0, 0] == -np.inf:
            continue
        cam = (world - T[:3, 3]) @ T[:3, :3]                       # R^T (p - t)
        z = cam[:, 2]
        front = z >= 2.0 ** -6
        amb |= np.abs(z - 2.0 ** -6) < eps_m
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.where(front, cam[:, 0] / z * fx + cx, np.nan); v = np.where(front, cam[:, 1] / z * fy + cy, np.nan)
        iu, iv = np.rint(u), np.rint(v)
        near_half = (np.abs(np.abs(u - np.floor(u)) - 0.5) < eps_px) | (np.abs(np.abs(v - np.floor(v)) - 0.5) < eps_px)
        inside = front & (iu >= 0) & (iu < width) & (iv >= 0) & (iv < height)
        amb |= front & near_half & (u > -1) & (u < width) & (v > -1) & (v < height)
        raw = np.zeros(len(world), np.float64)
        raw[inside] = depth[f][iv[inside].astype(np.int64), iu[inside].astype(np.int64)]
        d = raw / depth_shift
        valid = inside & (raw > 0) & (d >= dmin) & (d <= dmax)
        amb |= inside & (raw > 0) & ((np.abs(d - dmin) < eps_m) | (np.abs(d - dmax) < eps_m))
        s = d - z; band = bs * d + bb
        free = valid & (s > band) & (z < md)
        occ = valid & (s > -band) & (s <= band) & (d < md)
        amb |= valid & ((np.abs(s - band) < eps_m) | (np.abs(s + band) < eps_m) | (np.abs(z - md) < eps_m) | (np.abs(d - md) < eps_m))
        n_free += free; n_occ += occ
    shape = (nz, ny, nx)
    return n_free.reshape(shape), n_occ.reshape(shape), amb.reshape(shape)
