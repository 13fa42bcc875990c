"""TEST INFRASTRUCTURE — float64 statement of the marching-cubes spec written in the header comment of
scannet_b200/csrc/mc.cu, restated from that text (it does not use the oracle's table or its construction).

Voxel v is usable iff weight > 0 and |sdf| <= thr.  Cube at voxel g has corners g + (c&1, (c>>1)&1, (c>>2)&1), c = 0..7; it is
valid iff all 8 corners are usable; corner c is inside iff sdf < 0, and the case index has bit c set for an inside corner.
Lattice edge (g, a) carries a vertex iff both ends are usable and exactly one is inside, at t = s0 / (s0 - s1).

The twelve edges of a cube are numbered 4*a + u + 2*v, where a is the edge's axis and (u, v) are the cube-local offsets of
the edge along the two other axes in increasing axis order (x, y for a = 2; x, z for a = 1; y, z for a = 0): this is the
numbering "lowest edge id" refers to.  The triangulation of a case is derived geometrically here: each face's corners are
sorted by angle counter-clockwise as seen from outside; every maximal run of inside corners gives a segment from the edge
entering the run to the edge leaving it; the segments chain into loops, taken in the order of their lowest edge id and
started there, each fanned (v0, vi, vi+1).

Output order: blocks by packed key, voxels by lx + 8 ly + 64 lz, edges by axis, triangles by cube in the same order and by
table order within a cube; vertices no triangle references are dropped, order preserved."""
from __future__ import annotations

import math

import numpy as np

KEY_BIAS = 1 << 20


def pack(xyz) -> np.ndarray:
    b = np.asarray(xyz, np.int64).reshape(-1, 3) + KEY_BIAS
    return b[:, 0] | (b[:, 1] << 21) | (b[:, 2] << 42)


def corner(c: int) -> np.ndarray:
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.int64)


def edge_id(c0: int, c1: int) -> int:
    d = corner(c0) ^ corner(c1)
    assert d.sum() == 1, (c0, c1)
    a = int(np.argmax(d)); lo = np.minimum(corner(c0), corner(c1))
    o = [i for i in range(3) if i != a]
    return 4 * a + int(lo[o[0]]) + 2 * int(lo[o[1]])


def edge_owner(e: int):
    """(axis, cube-local offset of the edge's start corner) of edge id e"""
    a, u, v = e >> 2, e & 1, (e >> 1) & 1
    off = [0, 0, 0]; o = [i for i in range(3) if i != a]
    off[o[0]] = u; off[o[1]] = v
    return a, tuple(off)


def face_cycles():
    """The six faces, each as its four corner ids counter-clockwise seen from outside the cube."""
    out = []
    for a in range(3):
        for s in (0, 1):
            n = np.zeros(3); n[a] = 1.0 if s else -1.0
            cs = [c for c in range(8) if corner(c)[a] == s]
            ctr = np.mean([corner(c) for c in cs], 0)
            e1 = np.zeros(3); e1[(a + 1) % 3] = 1.0
            e2 = np.cross(n, e1)                                         # (e1, e2, n) right-handed
            ang = [math.atan2(float((corner(c) - ctr) @ e2), float((corner(c) - ctr) @ e1)) for c in cs]
            out.append([cs[i] for i in np.argsort(ang)])
    return out


def triangulate(cs: int):
    """[(e0, e1, e2), ...] for case cs"""
    nxt = {}
    for cyc in face_cycles():
        ins = [(cs >> c) & 1 for c in cyc]
        if all(ins) or not any(ins):
            continue
        for k in range(4):
            if ins[k] and not ins[k - 1]:
                m = k
                while ins[(m + 1) % 4]:
                    m = (m + 1) % 4
                enter, leave = edge_id(cyc[k - 1], cyc[k]), edge_id(cyc[m], cyc[(m + 1) % 4])
                assert enter not in nxt
                nxt[enter] = leave
    assert sorted(nxt) == sorted(nxt.values())                          # every edge enters once and leaves once
    tris, seen = [], set()
    for e0 in sorted(nxt):
        if e0 in seen:
            continue
        loop, e = [], e0
        while e not in seen:
            seen.add(e); loop.append(e); e = nxt[e]
        assert e == e0
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
    return tris


def table():
    """(ntri uint8 [256], tri uint8 [256, 12, 3]) of the spec's triangulation"""
    nt = np.zeros(256, np.uint8); tt = np.zeros((256, 12, 3), np.uint8)
    for cs in range(256):
        t = triangulate(cs)
        nt[cs] = len(t)
        if t:
            tt[cs, : len(t)] = t
    return nt, tt


_TABLE = None


def _table():
    global _TABLE
    if _TABLE is None:
        _TABLE = table()
    return _TABLE


def extract(block_xyz, vox, thr, vs):
    """The spec's mesh of a volume in float64.  block_xyz int [n,3], vox VOXEL_DTYPE [n,512]; thr, vs: the float32 values
    the implementation uses.  Returns a dict:
      edge [V,4] int64        (gx, gy, gz, axis) of each output vertex's lattice edge, in output order
      t, pos                  float64 [V], [V,3]: the crossing
      rgb_lo, rgb_hi [V,3]    the admissible colour bytes: u8(c0 + t (c1 - c0) + 0.5) with t exact, widened at a tie
      tri [F,3]               vertex ids (output order), tri_edge [F,3,4] the same as lattice edges
      cube [F,3] int64        origin g of the cube that emitted each triangle
      valid_g [C,3], valid_case [C]   every valid cube (all 8 corners usable), in output order, and its case"""
    thr = np.float32(thr); vs64 = float(np.float32(vs))
    NT, TT = _table()
    xyz = np.asarray(block_xyz, np.int64).reshape(-1, 3)
    n = len(xyz)
    keys = pack(xyz)
    order = np.argsort(keys, kind="stable")
    xyz, skeys = xyz[order], keys[order]
    assert n == 0 or (np.diff(skeys) > 0).all(), "a block is given twice"
    vox = np.asarray(vox).reshape(n, 512)[order]
    nb = np.full((n, 8), -1, np.int64)                                   # sorted index of block + (d&1, d>>1&1, d>>2), or -1
    for d in range(8):
        q = xyz + corner(d)
        ok = ((q >= -KEY_BIAS) & (q < KEY_BIAS)).all(1)
        k = pack(np.where(ok[:, None], q, 0))
        j = np.minimum(np.searchsorted(skeys, k), max(n - 1, 0))
        nb[:, d] = np.where(ok & (skeys[j] == k) if n else ok, j, -1)
    # 9^3 halo per block: the block and the first layer of its +x, +y, +z neighbours; index [block, z, y, x]
    S = np.zeros((n, 9, 9, 9), np.float32); W = np.zeros((n, 9, 9, 9), np.uint8); Cc = np.zeros((n, 9, 9, 9, 3), np.uint8)
    sdf = vox["sdf"].reshape(n, 8, 8, 8); w = vox["w"].reshape(n, 8, 8, 8)
    col = np.stack([vox["r"], vox["g"], vox["b"]], -1).reshape(n, 8, 8, 8, 3)
    for d in range(8):
        dx, dy, dz = corner(d)
        dst = tuple(slice(0, 8) if o == 0 else slice(8, 9) for o in (dz, dy, dx))
        src = tuple(slice(0, 8) if o == 0 else slice(0, 1) for o in (dz, dy, dx))
        has = np.nonzero(nb[:, d] >= 0)[0]
        s = nb[has, d]
        S[(has,) + dst] = sdf[(s,) + src]; W[(has,) + dst] = w[(s,) + src]; Cc[(has,) + dst] = col[(s,) + src]
    U = (W > 0) & (np.abs(S) <= thr)
    I = S < 0
    own = (slice(None), slice(0, 8), slice(0, 8), slice(0, 8))

    def shifted(a, off=1):                                               # the voxel `off` further along axis a (x = last)
        sl = [slice(None), slice(0, 8), slice(0, 8), slice(0, 8)]
        sl[3 - a] = slice(off, off + 8)
        return tuple(sl)

    flags = np.stack([U[own] & U[shifted(a)] & (I[own] != I[shifted(a)]) for a in range(3)], -1)    # [n,z,y,x,3]
    fl = flags.ravel()
    vid0 = np.cumsum(fl) - 1                                             # pre-drop vertex id of flat (block, l, axis)
    fi = np.nonzero(fl)[0]
    j, l, a = fi // 1536, (fi // 3) % 512, fi % 3
    lc = np.stack([l & 7, (l >> 3) & 7, l >> 6], 1)
    g = 8 * xyz[j] + lc
    hz, hy, hx = lc[:, 2], lc[:, 1], lc[:, 0]
    s0 = S[j, hz, hy, hx].astype(np.float64)
    step = np.eye(3, dtype=np.int64)[a]
    s1 = S[j, hz + step[:, 2], hy + step[:, 1], hx + step[:, 0]].astype(np.float64)
    t = s0 / (s0 - s1)
    pos = g.astype(np.float64) * vs64
    pos[np.arange(len(fi)), a] = (g[np.arange(len(fi)), a] + t) * vs64
    c0 = Cc[j, hz, hy, hx].astype(np.float64)
    c1 = Cc[j, hz + step[:, 2], hy + step[:, 1], hx + step[:, 0]].astype(np.float64)
    cv = c0 + t[:, None] * (c1 - c0) + 0.5
    eps = 2.0 ** -10                                                     # far above the binary32 evaluation's error
    rgb_lo = np.clip(np.floor(cv - eps), 0, 255).astype(np.uint8)
    rgb_hi = np.clip(np.floor(cv + eps), 0, 255).astype(np.uint8)
    # cubes
    valid = np.ones((n, 8, 8, 8), bool); cs = np.zeros((n, 8, 8, 8), np.int64)
    for c in range(8):
        cx, cy, cz = corner(c)
        sl = (slice(None), slice(cz, cz + 8), slice(cy, cy + 8), slice(cx, cx + 8))
        valid &= U[sl]; cs |= I[sl].astype(np.int64) << c
    vflat = np.nonzero(valid.ravel())[0]
    vcase = cs.ravel()[vflat]
    vj, vl = vflat // 512, vflat % 512
    vlc = np.stack([vl & 7, (vl >> 3) & 7, vl >> 6], 1)
    valid_g = 8 * xyz[vj] + vlc
    cnt = NT[vcase].astype(np.int64)
    rep = np.repeat(np.arange(len(vflat)), cnt)
    k = np.arange(len(rep)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    E = TT[vcase[rep], k].astype(np.int64)                               # [F,3] edge ids
    tri0 = np.zeros(E.shape, np.int64); tri_edge = np.zeros(E.shape + (4,), np.int64)
    owner = [edge_owner(e) for e in range(12)]
    ea = np.array([o[0] for o in owner]); eoff = np.array([o[1] for o in owner])
    for q in range(3):
        e = E[:, q]
        X = vlc[rep] + eoff[e]                                           # owner voxel, block-local, 0..8
        d = (X[:, 0] >> 3) | ((X[:, 1] >> 3) << 1) | ((X[:, 2] >> 3) << 2)
        jj = nb[vj[rep], d]
        assert (jj >= 0).all()
        ll = (X[:, 0] & 7) + 8 * (X[:, 1] & 7) + 64 * (X[:, 2] & 7)
        f = (jj * 512 + ll) * 3 + ea[e]
        assert fl[f].all(), "a triangle uses an edge without a vertex"
        tri0[:, q] = vid0[f]
        tri_edge[:, q, :3] = valid_g[rep] + eoff[e]; tri_edge[:, q, 3] = ea[e]
    used = np.zeros(len(fi), bool); used[tri0.ravel()] = True
    newid = np.cumsum(used) - 1
    edge = np.concatenate([g, a[:, None]], 1)
    return dict(edge=edge[used], t=t[used], pos=pos[used], rgb_lo=rgb_lo[used], rgb_hi=rgb_hi[used],
                tri=newid[tri0], tri_edge=tri_edge, cube=valid_g[rep], valid_g=valid_g, valid_case=vcase,
                n_edges=len(fi))


def check(ref, xyz, rgb, tri, vs, ulps=2):
    """A mesh (xyz float32 [V,3], rgb uint8 [V,3], tri [F,3]) against extract()'s statement: the same triangles as lattice
    edges in the same order, every coordinate within `ulps` ulp of the float64 crossing (ulp of the binary32 coordinate
    span of its edge), every colour byte inside its interval."""
    vs64 = float(np.float32(vs))
    tri = np.asarray(tri, np.int64).reshape(-1, 3)
    assert len(xyz) == len(ref["edge"]), f"{len(xyz)} vertices, the spec has {len(ref['edge'])}"
    assert len(tri) == len(ref["tri"]), f"{len(tri)} triangles, the spec has {len(ref['tri'])}"
    if len(tri):
        te = ref["edge"][tri]
        bad = np.nonzero((te != ref["tri_edge"]).any((1, 2)))[0]
        assert len(bad) == 0, f"{len(bad)} triangles differ as lattice edges (first #{bad[0]}: {te[bad[0]].tolist()} " \
                              f"vs {ref['tri_edge'][bad[0]].tolist()}, case cube {ref['cube'][bad[0]].tolist()})"
    P = np.asarray(xyz, np.float32).astype(np.float64)
    g = ref["edge"][:, :3].astype(np.float64)
    span = np.maximum(np.maximum(np.abs(g), np.abs(g + 1)) * vs64, vs64)
    ulp = np.spacing(span.astype(np.float32)).astype(np.float64)
    err = np.abs(P - ref["pos"]) / ulp
    assert len(err) == 0 or err.max() <= ulps, f"vertex {int(np.argmax(err.max(1)))} is {err.max():.2f} ulp off its crossing"
    rgb = np.asarray(rgb, np.uint8)
    out = (rgb < ref["rgb_lo"]) | (rgb > ref["rgb_hi"])
    assert not out.any(), f"{int(out.any(1).sum())} vertex colours outside their interval (first vertex {int(np.argmax(out.any(1)))})"
