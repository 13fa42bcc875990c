"""TEST INFRASTRUCTURE — TSDF volumes built voxel by voxel for the marching-cubes tests (tests/test_mc_reference_cpu.py,
tests/test_mc_designed_gpu.py): every cube case at every block-seam position, boundary values, key-range edges, closed
analytic surfaces and degenerate volumes.  Each builder returns (block_xyz int32 [n,3], voxels VOXEL_DTYPE [n,512]) in an
arbitrary block order."""
from __future__ import annotations

import numpy as np

from oracle_bindings import VOXEL_DTYPE

VS = np.float32(0.004)                      # voxel size of scn_tsdf_default_params
THR = np.float32(np.float32(10.0) * VS)     # mc_thresh_factor * voxel_size, as binary32
THR_UP = np.nextafter(THR, np.float32(np.inf))
KEY_LO, KEY_HI = -(1 << 20), (1 << 20) - 1  # block coordinate range

# cube origin inside a case block for each of the 8 position kinds: bit a set = the cube straddles the block's +a seam
POSITIONS = [tuple(7 if (p >> a) & 1 else 4 for a in range(3)) for p in range(8)]
POSITION_NAMES = ["interior", "x", "y", "xy", "z", "xz", "yz", "xyz"]


def corner(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.int64)


class Volume:
    """Blocks keyed by coordinate.  A new block is background: every voxel unusable, either weight 0 (random sdf of either
    sign) or weight > 0 with |sdf| > THR."""

    def __init__(self, seed=0):
        self.rng = np.random.default_rng(seed)
        self.blocks = {}

    def block(self, b):
        b = tuple(int(v) for v in b)
        if not all(KEY_LO <= v <= KEY_HI for v in b):
            return None
        if b not in self.blocks:
            r = self.rng
            v = np.zeros(512, VOXEL_DTYPE)
            zero_w = r.random(512) < 0.7
            mag = np.where(zero_w, r.uniform(0, 3, 512) * THR, THR * (1 + r.uniform(0, 2, 512)))
            mag = np.where(r.random(512) < 0.1, THR_UP, mag).astype(np.float32)
            v["sdf"] = np.where(r.random(512) < 0.5, -mag, mag)
            v["w"] = np.where(zero_w, 0, r.integers(1, 256, 512))
            for ch in "rgb":
                v[ch] = r.integers(0, 256, 512)
            self.blocks[b] = v
        return self.blocks[b]

    def set(self, g, sdf, w, rgb):
        """voxel g of an existing block (a voxel of a missing block is dropped)"""
        g = np.asarray(g, np.int64)
        blk = self.blocks.get(tuple(int(v) for v in g >> 3))
        if blk is None:
            return
        l = int((g[0] & 7) + 8 * (g[1] & 7) + 64 * (g[2] & 7))
        blk[l]["sdf"] = np.float32(sdf); blk[l]["w"] = w
        blk[l]["r"], blk[l]["g"], blk[l]["b"] = (int(c) for c in rgb)

    def cube(self, g0, sdf, w=None, rgb=None):
        """the 8 corners of the cube at voxel g0 (corner c at g0 + (c&1, c>>1&1, c>>2))"""
        w = self.rng.integers(1, 256, 8) if w is None else w
        rgb = self.rng.integers(0, 256, (8, 3)) if rgb is None else rgb
        for c in range(8):
            self.set(np.asarray(g0, np.int64) + corner(c), sdf[c], w[c], rgb[c])

    def random_corners(self, cs):
        """usable sdf values with the signs of case cs, |sdf| random in (0, THR], sometimes exactly THR"""
        mag = (THR * (1.0 - self.rng.random(8))).astype(np.float32)
        mag = np.where(self.rng.random(8) < 0.1, THR, np.maximum(mag, np.float32(1e-30)))
        return np.where([(cs >> c) & 1 for c in range(8)], -mag, mag).astype(np.float32)

    def case_block(self, b, cubes, neighbours=True):
        """up to 8 isolated cubes in block b, cube p at POSITIONS[p]; cubes[p] = (sdf[8], w[8] or None, rgb[8,3] or None).
        The +1 neighbours the seam cubes reach into are created unless `neighbours` is False or they are outside the key
        range; corners in a missing block are dropped."""
        b = np.asarray(b, np.int64)
        self.block(b)
        if neighbours:
            for d in range(1, 8):
                self.block(b + corner(d))
        for p, cube in enumerate(cubes):
            if cube is not None:
                self.cube(8 * b + np.array(POSITIONS[p]), *cube)

    def arrays(self, shuffle=True):
        keys = list(self.blocks)
        if shuffle:
            self.rng.shuffle(keys)
        xyz = np.array(keys, np.int32).reshape(-1, 3)
        vox = np.stack([self.blocks[k] for k in keys]) if keys else np.zeros((0, 512), VOXEL_DTYPE)
        return xyz, vox


def atlas(seed=0, origin=(0, 0, 0)):
    """Every one of the 256 cases once at each of the 8 position kinds (2048 isolated cubes): case block k of an 8x8x4 grid
    holds case (k + 32 p) % 256 at position p."""
    v = Volume(seed)
    for k in range(256):
        b = np.asarray(origin) + np.array([k % 8, (k // 8) % 8, k // 64])
        v.case_block(b, [(v.random_corners((k + 32 * p) % 256), None, None) for p in range(8)])
    return v.arrays()


def boundary_values(seed=1):
    """Corners at the ends of the usable range and colours at the ends of the byte range."""
    v = Volume(seed)
    r = v.rng
    up = THR_UP
    specs = []

    def usable(cs):
        return v.random_corners(cs)

    # +0 and -0 are both outside; exactly +-THR is usable
    for c0 in (np.float32(0.0), np.float32(-0.0)):
        for other in (-THR, THR, np.float32(-0.001)):
            s = usable(0b10010110); s[0] = c0; s[1] = other
            specs.append((s, None, None))
    s = np.array([THR, -THR, -THR, THR, -THR, THR, THR, -THR], np.float32); specs.append((s, None, None))
    s = np.full(8, -THR, np.float32); s[7] = THR; specs.append((s, None, None))
    s = np.full(8, np.float32(0.0)); s[3] = -THR; specs.append((s, None, None))                # t = 0 at six edges
    s = np.full(8, np.float32(-0.0)); s[5] = -THR; s[6] = np.float32(-1e-45); specs.append((s, None, None))
    s = np.array([1e-45, -1e-45, -1e-45, 1e-45, -1e-45, 1e-45, 1e-45, -1e-45], np.float32); specs.append((s, None, None))
    # the next float past THR is unusable: no cube, and no vertex on any edge that ends there
    for c in (0, 3, 7):
        for sign in (1, -1):
            s = usable(0b01101001); s[c] = sign * up; specs.append((s, None, None))
    # weight 0 with a negative sdf: unusable
    for c in (0, 6):
        s = usable(0b00111100); s[c] = -THR / 2; w = r.integers(1, 256, 8); w[c] = 0; specs.append((s, w, None))
    # colours: channels at 0 and 255, c1 < c0, and t placing c + 0.5 exactly on an integer
    ties = [(1.0, -1.0, 0, 1), (1.0, -3.0, 10, 20), (3.0, -1.0, 20, 10), (1.0, -1.0, 255, 0), (1.0, -1.0, 0, 255),
            (1.0, -1.0, 3, 4), (0.5, -1.5, 200, 0), (1.0, -254.0, 0, 255), (254.0, -1.0, 0, 255)]
    for s0, s1, c0, c1 in ties:
        s = usable(0b00000010); s[0] = np.float32(s0 * float(THR) / 256); s[1] = np.float32(s1 * float(THR) / 256)
        rgb = r.integers(0, 256, (8, 3)); rgb[0] = c0; rgb[1] = c1
        specs.append((s, None, rgb))
    for k in range(40):
        cs = int(r.integers(1, 255))
        s = usable(cs)
        s[r.random(8) < 0.3] = np.float32(0.0)
        s[r.random(8) < 0.2] = np.float32(-0.0)
        s = np.where(r.random(8) < 0.2, np.where(s < 0, -THR, THR), s).astype(np.float32)
        rgb = r.choice(np.array([0, 1, 254, 255], np.uint8), (8, 3))
        specs.append((s, None, rgb))
    for i in range(0, len(specs), 8):
        k = i // 8
        v.case_block((k % 4, k // 4, 0), specs[i:i + 8])
    return v.arrays()


def seams_and_keys(seed=2):
    """Seam cubes next to a missing neighbour block, all-negative block coordinates, and blocks at both ends of the key
    range, including one whose +x neighbour would alias to an existing block if the key were packed without a range check."""
    v = Volume(seed)
    cases = lambda k: [(v.random_corners((k * 67 + 29 * p + 1) % 254 + 1), None, None) for p in range(8)]  # noqa: E731
    # a missing neighbour: the cubes that straddle into it are not valid (their own-block edges still carry vertices)
    v.case_block((0, 0, 0), cases(0), neighbours=False)
    v.case_block((3, 0, 0), cases(1)); del v.blocks[(4, 0, 0)]
    v.case_block((6, 0, 0), cases(2)); del v.blocks[(6, 1, 1)]; del v.blocks[(7, 1, 1)]
    # all-negative coordinates, neighbours included
    for k, b in enumerate([(-3, -3, -3), (-2, -3, -3), (-3, -2, -2), (-9, -1, -5)]):
        v.case_block(b, cases(3 + k))
    # the ends of the key range: a +1 neighbour outside the range does not exist
    for k, b in enumerate([(KEY_LO, KEY_LO, KEY_LO), (KEY_HI, KEY_HI, KEY_HI), (KEY_HI, 0, 0), (KEY_HI - 1, KEY_LO, 5),
                           (0, KEY_HI, -1), (KEY_LO, KEY_HI, KEY_LO)]):
        v.case_block(b, cases(8 + k))
    # (KEY_HI + 1, 0, 0) packed without a range check is (KEY_LO, 1, 0): make that block fully usable
    bait = v.block((KEY_LO, 1, 0))
    bait["w"] = 7
    bait["sdf"] = np.where(v.rng.random(512) < 0.5, -THR / 3, THR / 3).astype(np.float32)
    return v.arrays()


def _dense(blocks_lo, blocks_hi, sdf_of, keep=None, seed=0):
    """All blocks in [blocks_lo, blocks_hi] (inclusive) with sdf_of(voxel coords [m,3]) -> metres; weights and colours
    vary smoothly.  keep(block sdf [512]) decides which blocks are allocated (default: any voxel within THR)."""
    lo, hi = np.asarray(blocks_lo), np.asarray(blocks_hi)
    gx, gy, gz = np.meshgrid(*[np.arange(lo[a], hi[a] + 1) for a in range(3)], indexing="ij")
    B = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], 1).astype(np.int64)
    l = np.arange(512)
    lc = np.stack([l & 7, (l >> 3) & 7, l >> 6], 1)
    G = (8 * B[:, None, :] + lc[None]).reshape(-1, 3)
    s = np.asarray(sdf_of(G.astype(np.float64)), np.float64).astype(np.float32).reshape(len(B), 512)
    sel = (np.abs(s) <= THR).any(1) if keep is None else keep(s)
    B, s, G = B[sel], s[sel], G.reshape(len(sel), 512, 3)[sel]
    vox = np.zeros((len(B), 512), VOXEL_DTYPE)
    vox["sdf"] = s
    vox["w"] = 1 + (G[..., 0] * 3 + G[..., 1] * 5 + G[..., 2] * 7) % 255
    vox["r"] = (G[..., 0] * 11) % 256; vox["g"] = (G[..., 1] * 13) % 256; vox["b"] = (G[..., 2] * 17 + 100) % 256
    o = np.random.default_rng(seed).permutation(len(B))
    return B[o].astype(np.int32), vox[o]


SPHERE_C, SPHERE_R = np.array([0.31, -0.27, 0.113]), 21.3            # voxels


def sphere_sdf(G):
    return (np.linalg.norm(G - SPHERE_C, axis=-1) - SPHERE_R) * float(VS)


def sphere_grad(G):
    d = G - SPHERE_C
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def sphere():
    r = int(np.ceil((SPHERE_R + 12) / 8)) + 1
    return _dense((-r, -r, -r), (r, r, r), sphere_sdf)


GYROID_K, GYROID_R, GYROID_A = 2 * np.pi / 15.7, 23.0, 0.05         # period 15.7 voxels inside a ball of radius ~23
GYROID_O = np.array([0.37, -0.21, 0.13])                              # keeps the field's exact zeros off the lattice


def gyroid_field(G):
    G = G + GYROID_O
    x, y, z = (G[..., a] * GYROID_K for a in range(3))
    g = np.sin(x) * np.cos(y) + np.sin(y) * np.cos(z) + np.sin(z) * np.cos(x)
    rr = np.maximum(np.linalg.norm(G, axis=-1) - GYROID_R, 0.0)
    return g + GYROID_A * rr * rr


def gyroid_sdf(G):
    return gyroid_field(G) * float(VS) / GYROID_K


def gyroid_grad(G):
    G = G + GYROID_O
    x, y, z = (G[..., a] * GYROID_K for a in range(3))
    gr = GYROID_K * np.stack([np.cos(x) * np.cos(y) - np.sin(z) * np.sin(x),
                              -np.sin(x) * np.sin(y) + np.cos(y) * np.cos(z),
                              -np.sin(y) * np.sin(z) + np.cos(z) * np.cos(x)], -1)
    n = np.linalg.norm(G, axis=-1, keepdims=True)
    rr = np.maximum(n - GYROID_R, 0.0)
    return gr + 2 * GYROID_A * rr * G / n


def gyroid():
    r = int(np.ceil((GYROID_R + 14) / 8)) + 1
    return _dense((-r, -r, -r), (r, r, r), gyroid_sdf)


def no_crossing(seed=3):
    """usable voxels, all outside (+0 included): no cube has a sign change"""
    r = np.random.default_rng(seed)
    xyz = np.array([(x, y, z) for x in range(3) for y in range(3) for z in range(2)], np.int32)
    vox = np.zeros((len(xyz), 512), VOXEL_DTYPE)
    vox["sdf"] = np.where(r.random(vox.shape) < 0.2, np.float32(0.0), THR * r.random(vox.shape)).astype(np.float32)
    vox["w"] = r.integers(1, 256, vox.shape)
    return xyz, vox


def all_unusable(seed=4):
    """every voxel unusable (weight 0, or |sdf| above THR) although the signs change everywhere"""
    v = Volume(seed)
    for b in [(x, y, z) for x in range(3) for y in range(2) for z in range(2)]:
        v.block(b)
    return v.arrays()


LATTICE_P, LATTICE_R = 32.0, 3.7                                      # small spheres on a 32-voxel lattice


def lattice_sdf(G):
    c = LATTICE_P * np.round((G - 5.5) / LATTICE_P) + 5.5
    return (np.linalg.norm(G - c, axis=-1) - LATTICE_R) * float(VS)


def large(nx=28, ny=28, nz=26):
    """a dense nx*ny*nz grid of blocks (20384 by default: the vertex and triangle scans over N*512 counts need three levels)
    holding small spheres spread through the key order"""
    return _dense((-nx // 2, -ny // 2, -nz // 2), (nx - nx // 2 - 1, ny - ny // 2 - 1, nz - nz // 2 - 1), lattice_sdf,
                  keep=lambda s: np.ones(len(s), bool))
