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
    """Depth in metres, NaN = invalid.  A float image is taken as metres already (the bilateral filter's output, -inf or 0 =
    invalid) and used exactly; a u16 image is raw sensor units (0 = invalid) divided by depth_shift."""
    a = np.asarray(depth_raw)
    if a.dtype.kind == "f":
        d = a.astype(np.float64)
        d[~np.isfinite(d) | (d == 0)] = np.nan
        return d
    d = a.astype(np.float64) / float(np.float32(depth_shift))
    d[a == 0] = np.nan
    return d


def fuse_single_frame(params, depth_raw, rgb, cam2world, K, block_xyz):
    """One frame fused into a fresh volume, for every voxel of the given blocks ([n,3] block coordinates).

    Returns a dict of [n, 512] arrays (voxel l = lx + 8 ly + 64 lz): `upd` (the frame updates the voxel), `amb` (float32 and
    float64 may disagree: excluded from comparisons), `sdf` (float64), `w` (weight byte), `rgb` ([n, 512, 3] colour bytes)."""
    f = _frame_samples(params, depth_raw, rgb, cam2world, K, block_xyz)
    return dict(upd=f["upd"], amb=f["amb"], sdf=f["sdf"], w=np.minimum(f["w1"], int(params.weight_max)), rgb=f["rgb"],
                tol_sdf=f["tol_sdf"])


def _frame_samples(params, depth_raw, rgb, cam2world, K, block_xyz, pixel_margin=4.0):
    """What one frame offers every voxel of the given blocks, before any averaging: `upd`, `amb`, the clamped sample `sdf`
    (float64), the per-sample weight `w1` (integer, not capped), the colour sample `rgb`, and `tol_sdf`.  A projection within
    1e-4 + pixel_margin * e_pos * (|f| + |u - c|) / z pixels of a half-integer is ambiguous; the float32 camera point is
    within about e_pos / 2 of the float64 one (a few roundings of coordinates of magnitude `scale`), so 4 is eight times
    that and 2 four times."""
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
    dm = depth_metres(depth_raw, params.depth_shift)
    rgb_img = None if rgb is None else np.asarray(rgb)

    def at(ix, iy, Z):
        """The update a voxel at depth Z gets from pixel (ix, iy), and its own doubts (range ends, band edge, w1 next to
        an integer)."""
        inimg = (Z >= Z_NEAR) & (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
        ixc = np.where(inimg, ix, 0).astype(np.int64); iyc = np.where(inimg, iy, 0).astype(np.int64)
        d = np.where(inimg, dm[iyc, ixc], np.nan)
        e_d = 4e-7 * np.where(np.isnan(d), 1.0, d)
        amb = inimg & ((np.abs(d - dmin) < e_d) | (np.abs(d - dmax) < e_d))
        valid = inimg & (d >= dmin) & (d <= dmax)
        sdf = d - Z
        tr = ts * d + tb
        amb |= valid & (np.abs(sdf + tr) < tol_sdf)
        upd = valid & (sdf > -tr)
        s = np.where(upd, np.minimum(sdf, tr), 0.0)
        wf = np.maximum(ws15 * (1.0 - (d - dmin) / (dmax - dmin)), 1.0)
        amb |= upd & (wf > 1.5) & (np.abs(wf - np.rint(wf)) < 1e-6 + 4e-7 * wf)
        w1 = np.floor(np.where(upd, wf, 0.0)).astype(np.int64)
        c = np.zeros(upd.shape + (3,), np.uint8)
        if rgb_img is not None:
            c = np.where(upd[..., None], rgb_img[iyc, ixc], 0).astype(np.uint8)
        return upd, s, w1, c, amb

    with np.errstate(divide="ignore", invalid="ignore"):
        u = fx * X / Z + cx
        v = fy * Y / Z + cy
        # a float32 projection may round to the other neighbour within this distance of a half-integer (exact float64
        # half-integers are exact in binary32 as well - the dyadic test scenes - and are rounded half to even)
        mu = 1e-4 + e_pos * (np.abs(fx) + np.abs(u - cx)) / np.abs(Z) * pixel_margin
        mv = 1e-4 + e_pos * (np.abs(fy) + np.abs(v - cy)) / np.abs(Z) * pixel_margin
        near = []
        for q, m in ((u, mu), (v, mv)):
            off = np.abs(q - np.floor(q) - 0.5)
            near.append(front & (off < m) & (off != 0.0))
        ix, iy = np.rint(u), np.rint(v)                                           # round half to even
        upd, s, w1, out_rgb, amb_d = at(ix, iy, Z)
        amb |= amb_d
        # next to a rounding boundary the voxel is ambiguous only if the neighbouring pixel would give another update
        j = np.nonzero(near[0] | near[1])
        if len(j[0]):
            alt_x = np.where(near[0][j], 2 * np.floor(u[j]) + 1 - ix[j], ix[j])
            alt_y = np.where(near[1][j], 2 * np.floor(v[j]) + 1 - iy[j], iy[j])
            for ax_, ay_ in ((alt_x, iy[j]), (ix[j], alt_y), (alt_x, alt_y)):
                ua, sa, wa, ca, aa = at(ax_, ay_, Z[j])
                differs = aa | (ua != upd[j]) | (sa != s[j]) | (wa != w1[j]) | (ca != out_rgb[j]).any(-1)
                amb[j] |= differs
    return dict(upd=upd, amb=amb, sdf=s, w1=w1, rgb=out_rgb, tol_sdf=tol_sdf)


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
    """Cells crossed by the segments A->B ([m,3] block units).  With shrink > 0 the segment ends move inwards by `shrink`
    block units and pieces shorter than `shrink` (grazing a face or an edge) are dropped."""
    return _pieces(A, B, shrink)[0]


def _pieces(A, B, shrink):
    """The pieces of the segments A->B ([m,3] block units) inside the cells they cross: (cells [q,3], segment index [q],
    piece parameters t0, t1 [q] along the (shrunk) segment).  `shrink` is a scalar or one value per segment (see _crossed)."""
    Dv = B - A
    L = np.linalg.norm(Dv, axis=1)
    shrink = np.broadcast_to(np.asarray(shrink, np.float64), (len(A),))
    if (shrink > 0).any():
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
    keep = np.isfinite(t0) & np.isfinite(t1) & ((t1 - t0) * L[:, None] > shrink[:, None])
    mid = 0.5 * (t0 + t1)
    cells = np.floor(A[:, None, :] + mid[..., None] * Dv[:, None, :])
    seg = np.nonzero(keep)[0]
    return cells[keep].astype(np.int64), seg, t0[keep], t1[keep]


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


# ---- several frames -------------------------------------------------------------------------------------------------
WALK_CAP = 48                  # cells a pixel's walk visits at most (spec step B)
COLOUR_HALF = 1e-4             # a colour average closer than this to k + 1/2 may round either way in binary32


def touched_blocks(params, depth, cam2world, K, region=None):
    """Packed keys of the blocks one frame's walks must touch (`certain`) and may touch (`possible`).

    The float32 walk follows the segment between its float32 ends, which lie within eps (block units) of the float64 ends;
    every point of it is then within eps of the float64 segment, and a crossing-parameter tie decided the other way by
    the walk's float32 accumulation moves it by less than WALK_CAP ulp of t along a segment of length L.  So with
    eps = 4 e_pos / (8 vs) + WALK_CAP 2^-23 L (e_pos as in tolerances()):
      * certain  = cells crossed by the float64 segment shrunk by eps, pieces shorter than eps dropped, of pixels whose
                   depth is more than its rounding error inside [depth_min, depth_max] and below max_integration_distance;
      * possible = cells within eps (max norm) of the float64 segment of any pixel that may be in range.  A cell within
                   eps of a segment is a neighbour of a crossed cell whose piece comes within eps of the shared face,
                   edge or corner, per axis; the per-axis test on the piece's bounding box can only add cells.
    Asserts that no walk comes near the WALK_CAP cell cap, beyond which the spec stops following the segment.
    `region` ([r, 2, 3] inclusive block bounds lo, hi) keeps only the pixels whose segment comes within two blocks of one of
    the boxes: both sets are then complete inside the boxes."""
    vs = _p(params, "voxel_size")
    dmin, dmax, maxint = _p(params, "depth_min"), _p(params, "depth_max"), _p(params, "max_integration_distance")
    tb, ts = _p(params, "trunc_base"), _p(params, "trunc_scale")
    T = np.asarray(cam2world, np.float64)
    Kd = np.asarray(K, np.float64); fx, fy, cx, cy = Kd[0, 0], Kd[1, 1], Kd[0, 2], Kd[1, 2]
    d = depth_metres(depth, params.depth_shift)
    H, W = d.shape
    y, x = np.mgrid[0:H, 0:W]
    d = d.ravel(); x = x.ravel(); y = y.ravel()
    e_d = 4e-7 * np.where(np.isnan(d), 1.0, d)
    loose = (d >= dmin - e_d) & (d <= dmax + e_d) & (d < maxint + e_d)
    sure = (d >= dmin + e_d) & (d <= dmax - e_d) & (d < maxint - e_d)
    tr = ts * d + tb
    zmin, zmax = np.minimum(maxint, d - tr), np.minimum(maxint, d + tr)
    loose &= zmin < zmax
    sure &= zmin < zmax
    ray = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones_like(d)], -1)[loose]
    to_blk = lambda Zc: ((ray * Zc[:, None]) @ T[:3, :3].T + T[:3, 3]) / (8.0 * vs) + 1.0 / 16.0
    A, B = to_blk(zmin[loose]), to_blk(zmax[loose])
    sure = sure[loose]
    inkey = key_range(A) & key_range(B)
    A, B, sure = A[inkey], B[inkey], sure[inkey]
    if region is not None:
        lo, hi = np.floor(np.minimum(A, B)), np.floor(np.maximum(A, B))
        near = np.zeros(len(A), bool)
        for r_lo, r_hi in np.asarray(region):
            near |= ((lo - 2 <= r_hi) & (hi + 2 >= r_lo)).all(1)
        A, B, sure = A[near], B[near], sure[near]
    empty = np.zeros(0, np.int64)
    if not len(A):
        return empty, empty
    steps = np.abs(np.floor(B) - np.floor(A)).sum(1)
    assert steps.max() + 1 + 3 <= WALK_CAP, \
        f"a walk crosses {int(steps.max()) + 1} cells, too close to the {WALK_CAP}-cell cap for the float64 statement"
    scale = max(world_scale(T), float(np.abs(np.concatenate([A, B])).max() + 1) * 8.0 * vs)
    L = np.linalg.norm(B - A, axis=1)
    eps = 4.0 * tolerances(scale)[0] / (8.0 * vs) + WALK_CAP * 2.0 ** -23 * L
    cells, seg, t0, t1 = _pieces(A, B, 0.0)
    L, e = L[seg], eps[seg]
    # the pieces of the segment shrunk by eps are these pieces clipped to [eps / L, 1 - eps / L]
    f = np.minimum(e / np.maximum(L, 1e-300), 0.5)
    sure_piece = sure[seg] & ((np.minimum(t1, 1 - f) - np.maximum(t0, f)) * L > e)
    certain = np.unique(pack(cells[sure_piece]))
    D = (B - A)[seg]
    P0, P1 = A[seg] + t0[:, None] * D, A[seg] + t1[:, None] * D
    near_hi = np.maximum(P0, P1) >= cells + 1 - e[:, None]                      # per axis: the piece's bounding box
    near_lo = np.minimum(P0, P1) <= cells + e[:, None]
    out = [cells]
    for o in np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3):
        if not o.any():
            continue
        ax = np.nonzero(o)[0]
        cand = np.ones(len(cells), bool)
        for i in ax:
            cand &= near_hi[:, i] if o[i] > 0 else near_lo[:, i]
        j = np.nonzero(cand)[0]
        if len(ax) > 1 and len(j):
            # an edge or corner: the piece P0 + t (P1 - P0), t in [0, 1], needs a point with p_i >= cell_i + 1 - eps
            # (o_i = 1) or p_i <= cell_i + eps (o_i = -1) on those axes at once - intersect the per-axis parameter ranges
            p0, dp, ej = P0[j], P1[j] - P0[j], e[j]
            t_lo, t_hi = np.zeros(len(j)), np.ones(len(j))
            for i in ax:
                c = cells[j, i] + (1 - ej if o[i] > 0 else ej)
                with np.errstate(divide="ignore", invalid="ignore"):
                    tc = (c - p0[:, i]) / dp[:, i]
                up = dp[:, i] * o[i] > 0                                          # moving towards the neighbour
                flat = dp[:, i] == 0
                ok_flat = (p0[:, i] - c) * o[i] >= 0
                t_lo = np.where(flat, np.where(ok_flat, t_lo, 2.0), np.where(up, np.maximum(t_lo, tc), t_lo))
                t_hi = np.where(flat | up, t_hi, np.minimum(t_hi, tc))
            j = j[t_lo <= t_hi]
        out.append(cells[j] + o)
    possible = np.unique(pack(np.concatenate(out)))
    return certain, possible


def _round_half_up(num, den, side):
    """Byte of binary32 floor(num/den + 1/2) for integer num, den > 0: the lower (side 0) or upper (side 1) of the values it
    may take; both neighbours when num/den lies within COLOUR_HALF of k + 1/2 - except an exact k + 1/2 over a power-of-two
    den, which every step computes exactly (1/den, the product and the + 1/2), so it rounds up."""
    k = num // den
    r2 = 2 * (num - k * den) - den                                                # 2 den (frac(q) - 1/2), in [-den, den)
    near = (np.abs(r2) < 2.0 * COLOUR_HALF * den) & ~((r2 == 0) & ((den & (den - 1)) == 0))
    nearest = k + (r2 >= 0)
    return np.where(near, k + side, nearest)


def frame_updates(params, frames, block_xyz, region=None):
    """Per valid frame of `frames` ((depth, rgb or None, cam2world, K); depth u16 raw or float metres), in order: the
    _frame_samples dict of the given blocks plus `in_certain` / `in_possible` ([n, 1]: the frame's walk must / may touch
    the block) and the frame's `certain` / `possible` key sets.  Frames with an invalid pose are skipped."""
    bx = np.asarray(block_xyz, np.int64).reshape(-1, 3)
    keys = pack(bx)
    for depth, rgb, T, K in frames:
        if np.asarray(T, np.float32)[0, 0] == -np.inf:
            continue
        fr = _frame_samples(params, depth, rgb, T, K, bx, pixel_margin=2.0)
        certain, possible = touched_blocks(params, depth, T, K, region)
        fr.update(in_certain=np.isin(keys, certain)[:, None], in_possible=np.isin(keys, possible)[:, None],
                  certain=certain, possible=possible, has_rgb=rgb is not None)
        yield fr


def fuse_sequence(params, frames, block_xyz, region=None):
    """Frames fused in order into a fresh volume, in float64, for every voxel of the given blocks ([n,3]).

    Per voxel: `sdf` is the exact weighted mean (sdf0 w0 + s w1) / (w0 + w1); `w` the exact integer weight, stored as
    min(w0 + w1, weight_max), and that capped value is the next update's w0; the colour is an interval [`lo`, `hi`] per
    channel ([n,512,3]) holding every byte binary32 may produce: the average of an interval is taken at both ends, and
    rounding it to a byte may go either way within COLOUR_HALF of k + 1/2.  A frame without colour leaves the colour as
    it is and still adds its weight.  A frame updates a voxel only if its walk touched the voxel's block.

    `amb` ([n,512]) marks voxels where float32 and float64 may have parted at some frame and stays set: whatever
    _frame_samples flags (with half its single-frame pixel margin: the flags of every frame add up), and an update of a block that the frame's walk may but need not touch.

    `err` ([n,512]) bounds |sdf_binary32 - sdf| for voxels never ambiguous.  A new sample s is within tol_sdf of its
    float64 value (single-frame bound); binary32 evaluates fl(fl(fma(sdf0, w0, fl(s w1))) * fl(1 / (w0 + w1))), four
    roundings of magnitude at most tr_max = trunc_scale depth_max + trunc_base (the weights are exact integers), so
        err' = (w0 err0 + w1 tol_sdf) / (w0 + w1) + 4 * 2^-24 tr_max:
    the mean shrinks the inherited error by w0 / (w0 + w1), and the bound never exceeds tol_sdf + 4 n 2^-24 tr_max after
    n updates.

    Also returns `seen` (a frame updated or may have updated the voxel), `coloured` (a frame with colour did), the unions
    `certain` / `possible` of the frames' block sets, and `frames` (valid frames fused)."""
    bx = np.asarray(block_xyz, np.int64).reshape(-1, 3)
    n = len(bx)
    wmax = int(params.weight_max)
    tr_max = _p(params, "trunc_scale") * _p(params, "depth_max") + _p(params, "trunc_base")
    rnd = 4.0 * 2.0 ** -24 * tr_max
    w = np.zeros((n, 512), np.int64)
    sdf = np.zeros((n, 512)); err = np.zeros((n, 512))
    lo = np.zeros((n, 512, 3), np.int64); hi = np.zeros((n, 512, 3), np.int64)
    amb = np.zeros((n, 512), bool); seen = np.zeros((n, 512), bool); coloured = np.zeros((n, 512), bool)
    certain, possible, done = [], [], 0
    for fr in frame_updates(params, frames, bx, region):
        done += 1
        certain.append(fr["certain"]); possible.append(fr["possible"])
        amb |= fr["amb"] | (fr["upd"] & fr["in_possible"] & ~fr["in_certain"])
        u = fr["upd"] & fr["in_possible"]
        seen |= u | (fr["amb"] & fr["in_possible"])
        w0, w1 = w, fr["w1"]
        ws = np.where(u, w0 + w1, 1)
        sdf = np.where(u, (sdf * w0 + fr["sdf"] * w1) / ws, sdf)
        err = np.where(u, (w0 * err + w1 * fr["tol_sdf"]) / ws + rnd, err)
        if fr["has_rgb"]:
            c1 = fr["rgb"].astype(np.int64) * w1[..., None]
            den = ws[..., None]
            lo = np.where(u[..., None], _round_half_up(lo * w0[..., None] + c1, den, 0), lo)
            hi = np.where(u[..., None], _round_half_up(hi * w0[..., None] + c1, den, 1), hi)
            coloured |= u
        w = np.where(u, np.minimum(w0 + w1, wmax), w)
    cat = lambda s: np.unique(np.concatenate(s)) if s else np.zeros(0, np.int64)
    return dict(w=w, sdf=sdf, err=err, lo=lo, hi=hi, amb=amb, seen=seen, coloured=coloured,
                certain=cat(certain), possible=cat(possible), frames=done)


def check_sequence(params, frames, block_xyz, vox, max_ambiguous=0.05, min_exact_colour=0.8, sample=None, seed=0):
    """Asserts that a volume ([n,3] blocks, [n,512] voxels) fused from `frames` into an empty volume is the float64
    fusion of fuse_sequence outside its ambiguous voxels: weights exact, sdf within the derived bound, colour bytes inside
    their intervals; and that certain blocks of every frame ⊆ allocated blocks ⊆ possible blocks of some frame.

    Also asserts coverage, so that the check is never vacuous: at most `max_ambiguous` of the voxels a frame updated are
    ambiguous, and at least `min_exact_colour` of the coloured voxels' channels have a single admissible byte (lo == hi).

    `sample` = k checks about k blocks: the allocated blocks nearest (max norm) to 8 allocated blocks drawn with `seed`, k / 8
    around each; only the pixels whose segments come near those 8 clusters are walked, and the block-set check is made
    inside the clusters' bounding boxes.  Returns the reference dict with the fractions `ambiguous` and `exact_colour`."""
    all_bx = np.asarray(block_xyz, np.int64).reshape(-1, 3)
    bx, region = all_bx, None
    if sample is not None and sample < len(all_bx):
        rng = np.random.default_rng(seed)
        pick, region = [], []
        for c in all_bx[rng.choice(len(all_bx), 8, replace=False)]:
            near = np.argsort(np.abs(all_bx - c).max(1), kind="stable")[:sample // 8]
            pick.append(near)
            region.append([all_bx[near].min(0), all_bx[near].max(0)])
        pick = np.unique(np.concatenate(pick))
        bx, vox, region = all_bx[pick], vox[pick], np.asarray(region)
    ref = fuse_sequence(params, frames, bx, region)
    n_seen = int(ref["seen"].sum())
    assert n_seen > 0, "the sequence updates no voxel"
    n_amb = int((ref["amb"] & ref["seen"]).sum())
    ref["ambiguous"] = n_amb / n_seen
    assert n_amb <= max_ambiguous * n_seen, f"{n_amb} ambiguous voxels of {n_seen} updated (limit {max_ambiguous:.0%})"
    keep = ~ref["amb"]
    gw = vox["w"].astype(np.int64)
    bad = keep & (gw != ref["w"])
    assert not bad.any(), (f"{int(bad.sum())} voxel weights differ from the float64 fusion (first: got "
                           f"{gw[bad][:5].tolist()}, expected {ref['w'][bad][:5].tolist()})")
    m = keep & (ref["w"] > 0)
    e = np.abs(vox["sdf"].astype(np.float64) - ref["sdf"])
    over = m & (e > ref["err"])
    assert not over.any(), (f"{int(over.sum())} voxel sdf values differ from the float64 fusion by more than the bound "
                            f"(worst {(e - ref['err'])[over].max():.3g} m over it, max |dsdf| {e[m].max():.3g} m)")
    mc = m & ref["coloured"]
    got = np.stack([vox["r"], vox["g"], vox["b"]], -1).astype(np.int64)
    out = mc[..., None] & ((got < ref["lo"]) | (got > ref["hi"]))
    if out.any():
        i = np.argwhere(out)[0]
        raise AssertionError(f"{int(out.any(-1).sum())} voxel colours lie outside their float64 intervals (first: channel "
                             f"{'rgb'[i[2]]} = {got[tuple(i)]}, interval [{ref['lo'][tuple(i)]}, {ref['hi'][tuple(i)]}])")
    n_col = int(mc.sum())
    ref["exact_colour"] = float((ref["lo"] == ref["hi"])[mc].mean()) if n_col else 1.0
    assert ref["exact_colour"] >= min_exact_colour, \
        f"only {ref['exact_colour']:.1%} of the coloured voxels' channels have a single admissible byte"
    def inside(keys_or_xyz):
        if region is None:
            return keys_or_xyz
        c = keys_or_xyz if keys_or_xyz.ndim == 2 else np.stack([(keys_or_xyz >> (21 * i)) & 0x1FFFFF for i in range(3)], -1) - KEY_BIAS
        m = np.zeros(len(c), bool)
        for r_lo, r_hi in region:
            m |= ((c >= r_lo) & (c <= r_hi)).all(1)
        return keys_or_xyz[m]
    alloc = np.unique(pack(inside(all_bx)))
    ref["certain"], ref["possible"] = inside(ref["certain"]), inside(ref["possible"])
    missing = np.setdiff1d(ref["certain"], alloc)
    assert len(missing) == 0, f"{len(missing)} blocks every walk must touch are not allocated"
    stray = np.setdiff1d(alloc, ref["possible"])
    assert len(stray) == 0, f"{len(stray)} allocated blocks are not within reach of any frame's truncation segments"
    return ref


# ---- depth bilateral filter ----------------------------------------------------------------------------------------
def bilateral_f64(depth_raw, depth_shift, sigma_d, sigma_r):
    """Float64 statement of the depth pre-filter: radius r = ceil(2 sigma_d); every tap (dx, dy) within r per axis that is
    inside the image and valid weighs exp(-(dx^2 + dy^2) / (2 sigma_d^2)) * exp(-(d - d_centre)^2 / (2 sigma_r^2)); the
    output is the weighted mean, -inf where the centre is invalid (0).  Returns (metres [H,W], taps per pixel)."""
    a = np.asarray(depth_raw)
    sd, sr = float(np.float32(sigma_d)), float(np.float32(sigma_r))
    d = np.where(a == 0, np.nan, a.astype(np.float64) / float(np.float32(depth_shift)))
    H, W = d.shape
    r = int(np.ceil(2.0 * sd))
    pad = np.full((H + 2 * r, W + 2 * r), np.nan)
    pad[r:r + H, r:r + W] = d
    num = np.zeros((H, W)); den = np.zeros((H, W))
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            cur = pad[r + dy:r + dy + H, r + dx:r + dx + W]
            wt = np.exp(-(dx * dx + dy * dy) / (2.0 * sd * sd)) * np.exp(-(cur - d) ** 2 / (2.0 * sr * sr))
            ok = ~np.isnan(cur)
            num += np.where(ok, wt * cur, 0.0); den += np.where(ok, wt, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(np.isnan(d), -np.inf, num / den)
    return out, (2 * r + 1) ** 2


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
