"""TEST INFRASTRUCTURE: float64 statement of projective TSDF fusion and marching cubes, written from the geometry (DESIGN.md §3, §6)
rather than from oracle/tsdf_oracle.c's binary32 operation order.

The bit-exact tests pin the CUDA kernels to the oracle; this module pins both to the plain maths, so that a convention
mistake they share (half a pixel in the pixel centre, a transposed pose, a voxel corner taken for its centre, ...) fails.

Conventions stated here once:
  * voxel g (integer lattice coordinate) has its centre at world g * vs; block b holds the voxels 8b .. 8b + 7 per axis;
  * cam2world T maps camera to world, so a world point p is seen at pc = R^T (p - t); the camera looks along +z;
  * pixel (x, y) of a frame with intrinsics fx, fy, cx, cy sees the ray ((x - cx) / fx, (y - cy) / fy, 1); a camera point
    projects to u = fx * X / Z + cx, rounded half to even to the pixel index.

Where binary32 and float64 can legitimately disagree (a projection next to a rounding boundary, sdf next to -tr, z next to
the 2^-6 near plane, a per-sample weight next to an integer, depth next to the ends of its range) the voxel is reported as
ambiguous and left out of the comparison.  The margins scale with the magnitude of the world coordinates."""
from __future__ import annotations

import numpy as np

Z_NEAR = 2.0 ** -6
KEY_BIAS = 1 << 20


def _p(params, name):
    return float(np.float32(getattr(params, name)))


def world_scale(cam2world, block_xyz=None, vs=None):
    """Magnitude of the world coordinates involved (>= 1 m): sets every float32 error margin below."""
    s = 1.0
    s = max(s, float(np.abs(np.asarray(cam2world, np.float64)[:3, 3]).max()))
    if block_xyz is not None and len(block_xyz):
        s = max(s, float(np.abs(block_xyz).max() + 1) * 8.0 * vs)
    return s


def tolerances(scale):
    """(position error of a float32 camera-space point, sdf tolerance) in metres for world coordinates of magnitude `scale`."""
    e_pos = 8.0 * 2.0 ** -24 * scale           # a few ulp of the largest coordinate: pose inversion + block origin + voxel offset
    return e_pos, 3.0 * e_pos                  # ~1.1e-5 m at 8 m


def depth_metres(depth_raw, depth_shift):
    d = np.asarray(depth_raw, np.float64) / float(np.float32(depth_shift))
    d[np.asarray(depth_raw) == 0] = np.nan
    return d


def fuse_single_frame(params, depth_raw, rgb, cam2world, K, block_xyz):
    """One frame fused into a fresh volume, for every voxel of the given blocks ([n,3] block coordinates).

    Returns a dict of [n, 512] arrays (voxel l = lx + 8 ly + 64 lz): `upd` (the frame updates the voxel), `amb` (float32 and
    float64 may disagree: excluded from comparisons), `sdf` (float64), `w` (weight byte), `rgb` ([n, 512, 3] colour bytes)."""
    vs = _p(params, "voxel_size")
    W, H = int(params.width), int(params.height)
    dmin, dmax = _p(params, "depth_min"), _p(params, "depth_max")
    tb, ts = _p(params, "trunc_base"), _p(params, "trunc_scale")
    ws15 = 1.5 * float(params.weight_sample)
    T = np.asarray(cam2world, np.float64); R, t = T[:3, :3], T[:3, 3]
    Kd = np.asarray(K, np.float64); fx, fy, cx, cy = Kd[0, 0], Kd[1, 1], Kd[0, 2], Kd[1, 2]
    bx = np.asarray(block_xyz, np.int64).reshape(-1, 3)
    n = len(bx)
    e_pos, tol_sdf = tolerances(world_scale(T, bx, vs))

    l = np.arange(512)
    loc = np.stack([l & 7, (l >> 3) & 7, l >> 6], -1)                             # [512, 3]
    g = (8 * bx[:, None, :] + loc[None]).astype(np.float64)                       # [n, 512, 3] voxel lattice coordinates
    pc = (g * vs - t) @ R                                                         # R^T (p - t), row vectors
    X, Y, Z = pc[..., 0], pc[..., 1], pc[..., 2]
    amb = np.abs(Z - Z_NEAR) < e_pos
    front = Z >= Z_NEAR
    with np.errstate(divide="ignore", invalid="ignore"):
        u = fx * X / Z + cx
        v = fy * Y / Z + cy
        # a float32 projection may round to the other neighbour within this distance of a half-integer (exact float64
        # half-integers are exact in binary32 as well - the dyadic test scenes - and are rounded half to even)
        mu = 1e-4 + e_pos * (np.abs(fx) + np.abs(u - cx)) / np.abs(Z) * 4.0
        mv = 1e-4 + e_pos * (np.abs(fy) + np.abs(v - cy)) / np.abs(Z) * 4.0
        for q, m in ((u, mu), (v, mv)):
            off = np.abs(q - np.floor(q) - 0.5)
            amb |= front & (off < m) & (off != 0.0)
        ix, iy = np.rint(u), np.rint(v)                                           # round half to even
    inimg = front & (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    ixc = np.where(inimg, ix, 0).astype(np.int64); iyc = np.where(inimg, iy, 0).astype(np.int64)
    dm = depth_metres(depth_raw, params.depth_shift)
    d = np.where(inimg, dm[iyc, ixc], np.nan)
    e_d = 4e-7 * np.where(np.isnan(d), 1.0, d)
    amb |= inimg & ((np.abs(d - dmin) < e_d) | (np.abs(d - dmax) < e_d))
    valid = inimg & (d >= dmin) & (d <= dmax)
    sdf = d - Z
    tr = ts * d + tb
    amb |= valid & (np.abs(sdf + tr) < tol_sdf)
    upd = valid & (sdf > -tr)
    s = np.minimum(sdf, tr)
    wf = np.maximum(ws15 * (1.0 - (d - dmin) / (dmax - dmin)), 1.0)
    amb |= upd & (wf > 1.5) & (np.abs(wf - np.rint(wf)) < 1e-6 + 4e-7 * wf)
    w1 = np.floor(np.where(upd, wf, 0.0)).astype(np.int64)
    out_rgb = np.zeros((n, 512, 3), np.uint8)
    if rgb is not None:
        out_rgb = np.where(upd[..., None], np.asarray(rgb)[iyc, ixc], 0).astype(np.uint8)
    return dict(upd=upd, amb=amb, sdf=np.where(upd, s, 0.0), w=np.minimum(w1, int(params.weight_max)), rgb=out_rgb,
                tol_sdf=tol_sdf)


def check_single_frame(params, depth_raw, rgb, cam2world, K, block_xyz, vox, max_ambiguous=0.02):
    """Asserts that a fused volume ([n,3] blocks, [n,512] voxels after ONE frame into an empty volume) is the float64 statement
    of that frame, outside the ambiguous voxels.  Returns the reference dict."""
    ref = fuse_single_frame(params, depth_raw, rgb, cam2world, K, block_xyz)
    keep = ~ref["amb"]
    got_upd = vox["w"] > 0
    n_upd = int(ref["upd"].sum())
    assert n_upd > 0, "the case updates no voxel"
    assert ref["amb"].sum() <= max_ambiguous * max(n_upd, 1), f"{int(ref['amb'].sum())} ambiguous voxels of {n_upd} updated"
    bad = keep & (got_upd != ref["upd"])
    assert not bad.any(), f"{int(bad.sum())} voxels updated differently (first at {np.argwhere(bad)[:3].tolist()})"
    m = keep & ref["upd"]
    err = np.abs(vox["sdf"].astype(np.float64) - ref["sdf"])[m]
    assert err.max(initial=0.0) <= ref["tol_sdf"], f"max |sdf - float64| = {err.max():.3g} m > {ref['tol_sdf']:.3g}"
    assert (vox["w"][m] == ref["w"][m]).all(), "weights differ from float64"
    if rgb is not None:
        for i, ch in enumerate("rgb"):
            assert (vox[ch][m] == ref["rgb"][..., i][m]).all(), f"colour channel {ch} differs"
    return ref


# ---- block allocation ----------------------------------------------------------------------------------------------
def _segments(params, depth_raw, cam2world, K):
    """Float64 truncation segment of every pixel that allocates, in block units (block b covers [b, b + 1) per axis)."""
    vs = _p(params, "voxel_size")
    dmin, dmax, maxint = _p(params, "depth_min"), _p(params, "depth_max"), _p(params, "max_integration_distance")
    tb, ts = _p(params, "trunc_base"), _p(params, "trunc_scale")
    T = np.asarray(cam2world, np.float64)
    Kd = np.asarray(K, np.float64); fx, fy, cx, cy = Kd[0, 0], Kd[1, 1], Kd[0, 2], Kd[1, 2]
    d = depth_metres(depth_raw, params.depth_shift)
    H, W = d.shape
    y, x = np.mgrid[0:H, 0:W]
    d = d.ravel(); x = x.ravel(); y = y.ravel()
    tr = ts * d + tb
    zmin, zmax = np.minimum(maxint, d - tr), np.minimum(maxint, d + tr)
    ok = (d >= dmin) & (d <= dmax) & (d < maxint) & (zmin < zmax)
    ray = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones_like(d)], -1)[ok]
    # voxel centres at g*vs: the cell of voxel g is [g - 1/2, g + 1/2) vs, so block b spans [8b - 1/2, 8b + 15/2) vs
    to_blk = lambda Zc: ((ray * Zc[:, None]) @ T[:3, :3].T + T[:3, 3]) / (8.0 * vs) + 1.0 / 16.0
    return to_blk(zmin[ok]), to_blk(zmax[ok])


def _crossed(A, B, shrink):
    """Cells crossed by the segments A->B ([m,3] block units): returns packed keys of (cell, pixel) pairs, and the cells.
    With shrink > 0 the segment ends move inwards by `shrink` block units and pieces shorter than `shrink` (grazing a
    face or an edge) are dropped."""
    Dv = B - A
    L = np.linalg.norm(Dv, axis=1)
    if shrink > 0:
        f = np.minimum(shrink / np.maximum(L, 1e-300), 0.5)[:, None]
        A, B = A + f * Dv, B - f * Dv
        Dv = B - A
        L = np.linalg.norm(Dv, axis=1)
    ts = [np.zeros((len(A), 1)), np.ones((len(A), 1))]
    for i in range(3):
        lo, hi = np.minimum(A[:, i], B[:, i]), np.maximum(A[:, i], B[:, i])
        k0 = np.ceil(lo); nk = int(np.max(np.floor(hi) - k0 + 1, initial=0))
        for j in range(max(nk, 0)):
            k = k0 + j
            with np.errstate(divide="ignore", invalid="ignore"):
                tt = (k - A[:, i]) / Dv[:, i]
            ts.append(np.where((k <= hi) & np.isfinite(tt), tt, np.nan)[:, None])
    tt = np.sort(np.concatenate(ts, 1), axis=1)                                  # NaN sort last
    t0, t1 = tt[:, :-1], tt[:, 1:]
    keep = np.isfinite(t0) & np.isfinite(t1) & ((t1 - t0) * L[:, None] > shrink)
    mid = 0.5 * (t0 + t1)
    cells = np.floor(A[:, None, :] + mid[..., None] * Dv[:, None, :])
    return cells[keep].astype(np.int64)


def pack(c):
    c = np.asarray(c, np.int64) + KEY_BIAS
    return c[..., 0] | (c[..., 1] << 21) | (c[..., 2] << 42)


def check_allocation(params, depth_raw, cam2world, K, block_xyz, shrink=1e-3):
    """Every block crossed by the (slightly shrunk) float64 truncation segment of a valid pixel is allocated, and every
    allocated block lies within one block of some pixel's segment.  Pixels whose walk is longer than the 48-cell cap of the
    spec are left out of the first check."""
    A, B = _segments(params, depth_raw, cam2world, K)
    alloc = np.unique(pack(block_xyz))
    ok = key_range(A) & key_range(B)
    short = (np.abs(np.floor(B) - np.floor(A)).sum(1) + 1 + 2 < 48)
    need = np.unique(pack(_crossed(A[ok & short], B[ok & short], shrink)))
    missing = np.setdiff1d(need, alloc)
    assert len(missing) == 0, f"{len(missing)} blocks on the truncation band are not allocated"
    near = _crossed(A[ok], B[ok], 0.0)
    off = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3)
    reach = np.unique(pack((near[:, None, :] + off[None]).reshape(-1, 3)))
    stray = np.setdiff1d(alloc, reach)
    assert len(stray) == 0, f"{len(stray)} allocated blocks are more than one block away from every truncation segment"
    return len(need)


def key_range(P):
    return (np.abs(P) < KEY_BIAS - 2).all(1)


# ---- marching cubes ------------------------------------------------------------------------------------------------
def check_mesh(params, block_xyz, vox, xyz, tri, thresh_factor=10.0, ulps=2):
    """Every vertex lies on a lattice edge between two usable voxels (weight > 0, |sdf| <= thresh_factor * vs) of opposite
    sign (sdf < 0 inside), at the float64 zero crossing of the two stored sdf values to within `ulps` ulp of the edge's
    coordinate; the three vertices of every triangle lie on edges of one cube."""
    vs = _p(params, "voxel_size")
    thr = float(np.float32(np.float32(thresh_factor) * np.float32(vs)))
    keys = pack(block_xyz)
    order = np.argsort(keys); skeys = keys[order]
    sdf_all = vox["sdf"].astype(np.float64); w_all = vox["w"]

    def voxel(gc):                                                                # [m,3] lattice coords -> (sdf, usable)
        b = np.floor_divide(gc, 8); lc = gc - 8 * b
        k = pack(b); j = np.clip(np.searchsorted(skeys, k), 0, max(len(skeys) - 1, 0))
        found = (skeys[j] == k) if len(skeys) else np.zeros(len(k), bool)
        bi = order[j]; li = lc[:, 0] + 8 * lc[:, 1] + 64 * lc[:, 2]
        s = np.where(found, sdf_all[bi, li], 0.0); w = np.where(found, w_all[bi, li], 0)
        return s, found & (w > 0) & (np.abs(s) <= thr)

    P = np.asarray(xyz, np.float32).astype(np.float64)
    nv = len(P)
    G = P / vs
    Gr = np.rint(G)
    ulp_p = np.spacing(np.float32(np.abs(P) + vs)).astype(np.float64)
    on = np.abs(P - Gr * vs) <= 2 * ulp_p                                         # coordinates on a lattice plane
    assert (on.sum(1) >= 2).all(), "a vertex lies off every lattice edge"
    # candidate edges: (start voxel, axis); a vertex with three lattice coordinates sits on a voxel (stored sdf exactly 0)
    cand = []
    for a in range(3):
        use = on[:, [i for i in range(3) if i != a]].all(1)
        for back in (0, 1):                    # a vertex on a voxel ends the edge starting there (t = 0) or the one before (t = 1)
            st = Gr.copy()
            st[:, a] = np.where(on[:, a], Gr[:, a] - back, np.floor(G[:, a]))
            cand.append((st.astype(np.int64), a, use))
    ok_v = np.zeros(nv, bool)
    # origins of the cubes a vertex can belong to, per axis an interval: the edge's start on its own axis, start - 1 .. start
    # on the other two; a vertex on a voxel belongs to any of the 8 cubes around it
    c_lo = Gr.astype(np.int64) - 1; c_hi = Gr.astype(np.int64)
    for st, a, use in cand:
        g0 = st; g1 = st + np.eye(3, dtype=np.int64)[a]
        s0, u0 = voxel(g0); s1, u1 = voxel(g1)
        good = use & u0 & u1 & ((s0 < 0) != (s1 < 0))
        with np.errstate(divide="ignore", invalid="ignore"):
            tz = s0 / (s0 - s1)
        pa = (g0[:, a] + tz) * vs
        span = np.maximum(np.abs(g0[:, a]), np.abs(g1[:, a])).astype(np.float64) * vs
        ulp = np.spacing(np.float32(np.maximum(span, vs))).astype(np.float64)
        good &= np.abs(P[:, a] - pa) <= ulps * ulp
        others = [i for i in range(3) if i != a]
        good &= (np.abs(P[:, others] - g0[:, others] * vs) <= np.spacing(np.float32(np.abs(g0[:, others] * vs) + vs))).all(1)
        first = good & ~ok_v & ~on.all(1)
        c_lo[first, a] = g0[first, a]; c_hi[first, a] = g0[first, a]
        for o in others:
            c_lo[first, o] = g0[first, o] - 1; c_hi[first, o] = g0[first, o]
        ok_v |= good
    bad = np.nonzero(~ok_v)[0]
    assert len(bad) == 0, f"{len(bad)} of {nv} vertices are not at the float64 zero crossing of a usable sign-change edge " \
                          f"(first {P[bad[:3]].tolist()})"
    F = np.asarray(tri, np.int64).reshape(-1, 3)
    lo = c_lo[F].max(1); hi = c_hi[F].min(1)                                      # [nf, 3]: per-axis intersection
    split = np.nonzero((lo > hi).any(1))[0]
    assert len(split) == 0, f"{len(split)} triangles span more than one cube (first {F[split[:3]].tolist()})"
    return nv
