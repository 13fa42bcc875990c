"""Seeded synthetic inputs for the ScanNet hot path (SURVEY.md §8d).

* meshes in the VCGLIB / ScanNet ``_vh_clean_2.ply`` layout (binary little endian,
  ``float x,y,z; uchar red,green,blue,alpha; list uchar int vertex_indices``) — the
  layout Segmentator reads through tinyply
  (/root/reference/Segmentator/segmentator.cpp:130-140);
* RGB-D streams: analytic depth renders of a closed box room with spheres, a smooth
  camera loop, written as ``.sens`` v4 (/root/reference/SensReader/c++/src/sensorData.h:1058-1109).

Pure numpy; no GPU.  Everything is a deterministic function of its arguments.
"""
from __future__ import annotations

import struct
import zlib

import numpy as np

# ScannerApp sample intrinsics (/root/reference/ScannerApp/README.md:28-31)
FX = FY = 571.623718
CX, CY = 319.5, 239.5


# --------------------------------------------------------------------------- meshes
def make_grid_mesh(nx: int = 250, ny: int = 200, seed: int = 0, spacing: float = 0.02,
                   shuffle_faces: bool = True, flat_third: bool = True, noise: float = 0.0005):
    """Height-field mesh: ramp + sine + noise, with an exactly flat patch to force ties.

    Returns (xyz float32 [V,3], tri uint32 [F,3]).  nx=250, ny=200 gives V=50,000,
    F=99,102 (SURVEY.md §8d C1); nx=1600, ny=1250 gives the 2M-vertex C5 mesh.
    """
    rng = np.random.default_rng(seed)
    xs = np.arange(nx, dtype=np.float64) * spacing
    ys = np.arange(ny, dtype=np.float64) * spacing
    X, Y = np.meshgrid(xs, ys, indexing="xy")          # [ny, nx]
    mid = xs[nx // 2]
    Z = np.where(X > mid, (X - mid) * 0.5, 0.0) + 0.05 * np.sin(0.05 * Y / spacing)
    Z = Z + rng.normal(0.0, noise, size=Z.shape)
    if flat_third:
        Z[:, : nx // 3] = 0.0                           # exactly flat: exact-tie weights
    xyz = np.stack([X, Y, Z], axis=-1).reshape(-1, 3).astype(np.float32)
    vid = np.arange(nx * ny, dtype=np.uint32).reshape(ny, nx)
    a = vid[:-1, :-1].ravel(); b = vid[:-1, 1:].ravel()
    c = vid[1:, :-1].ravel(); d = vid[1:, 1:].ravel()
    tri = np.concatenate([np.stack([a, b, c], 1), np.stack([b, d, c], 1)], axis=0).astype(np.uint32)
    if shuffle_faces:
        tri = tri[rng.permutation(len(tri))]
    return xyz, np.ascontiguousarray(tri)


def make_feature_mesh(nx: int = 250, ny: int = 200, seed: int = 0, spacing: float = 0.02, noise: float = 0.0005):
    """Height field with plateaus, hemispherical bumps, a ramp and a quantised (exactly flat, exact-tie)
    third — gives tens to hundreds of segments at kThresh 0.01.  Same vertex/face layout as make_grid_mesh."""
    rng = np.random.default_rng(seed)
    xyz, tri = make_grid_mesh(nx, ny, seed=seed, spacing=spacing, shuffle_faces=True, flat_third=False, noise=0.0)
    X = xyz[:, 0].astype(np.float64).reshape(ny, nx); Y = xyz[:, 1].astype(np.float64).reshape(ny, nx)
    xs = np.arange(nx) * spacing; ys = np.arange(ny) * spacing
    Z = np.where(X > xs[nx // 2], (X - xs[nx // 2]) * 0.5, 0.0) + 0.05 * np.sin(0.05 * Y / spacing)
    for _ in range(min(200, max(4, (nx * ny) // 2500))):
        cx, cy = rng.uniform(0, xs[-1]), rng.uniform(0, ys[-1]); r = rng.uniform(4, 14) * spacing
        if rng.random() < 0.5:
            h = rng.uniform(0.05, 0.3)
            msk = (np.abs(X - cx) < r) & (np.abs(Y - cy) < r * rng.uniform(0.5, 1.5))
            Z = np.where(msk, Z + h, Z)
        else:
            Z = Z + np.sqrt(np.maximum(r * r - ((X - cx) ** 2 + (Y - cy) ** 2), 0.0))
    Z = Z + rng.normal(0.0, noise, Z.shape)
    Z[:, : nx // 3] = np.round(Z[:, : nx // 3] / 0.25) * 0.25
    xyz = xyz.copy(); xyz[:, 2] = Z.reshape(-1).astype(np.float32)
    return xyz, tri


def make_adversarial_mesh(seed: int = 0):
    """Small mesh exercising the reference's edge cases (SURVEY.md §8a S1-S3, §8d):
    a face repeating a vertex index, duplicated vertex positions (zero-length edge),
    an unreferenced vertex, exactly coplanar fans (±0 and equal weights)."""
    xyz, tri = make_grid_mesh(24, 20, seed=seed, shuffle_faces=True)
    xyz = xyz.copy(); tri = tri.copy()
    xyz = np.concatenate([xyz, np.array([[9.0, 9.0, 9.0]], np.float32)])   # unreferenced
    xyz[101] = xyz[100]                                                      # duplicate position
    rep = np.array([[7, 7, 8], [30, 31, 30]], np.uint32)                     # repeated index
    tri = np.concatenate([tri[:50], rep, tri[50:]])
    return xyz, np.ascontiguousarray(tri)


def write_ply(path, xyz: np.ndarray, tri: np.ndarray, rgba: np.ndarray | None = None,
              with_normals: bool = False):
    """Binary-LE PLY in the ScanNet/VCGLIB layout."""
    xyz = np.asarray(xyz, np.float32); tri = np.asarray(tri, np.int32)
    V, F = len(xyz), len(tri)
    if rgba is None:
        rgba = np.full((V, 4), 255, np.uint8)
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    hdr = ["ply", "format binary_little_endian 1.0", "comment VCGLIB generated",
           f"element vertex {V}", "property float x", "property float y", "property float z"]
    if with_normals:
        props += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        hdr += ["property float nx", "property float ny", "property float nz"]
    props += [("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1")]
    hdr += ["property uchar red", "property uchar green", "property uchar blue", "property uchar alpha",
            f"element face {F}", "property list uchar int vertex_indices", "end_header"]
    v = np.zeros(V, dtype=props)
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"], v["green"], v["blue"], v["alpha"] = rgba[:, 0], rgba[:, 1], rgba[:, 2], rgba[:, 3]
    f = np.zeros(F, dtype=[("n", "u1"), ("i", "<i4", (3,))])
    f["n"] = 3; f["i"] = tri
    with open(path, "wb") as fh:
        fh.write(("\n".join(hdr) + "\n").encode("ascii"))
        fh.write(v.tobytes()); fh.write(f.tobytes())


def read_ply(path):
    """Minimal binary-LE / ASCII PLY reader for tests: returns (xyz float32, tri uint32)."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header") + len(b"end_header")
    while data[end:end + 1] != b"\n":
        end += 1
    end += 1
    lines = data[:end].decode("ascii", "replace").split("\n")
    fmt = "ascii"; elems = []
    for ln in lines:
        t = ln.split()
        if not t:
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elems.append([t[1], int(t[2]), []])
        elif t[0] == "property":
            elems[-1][2].append(t[1:])
    tmap = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
            "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
            "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}
    xyz = tri = None
    if fmt == "ascii":
        toks = data[end:].split()
        pos = 0
        for name, n, props in elems:
            if name == "vertex":
                k = len(props)
                arr = np.array(toks[pos:pos + n * k], dtype=np.float64).reshape(n, k); pos += n * k
                names = [p[-1] for p in props]
                xyz = arr[:, [names.index("x"), names.index("y"), names.index("z")]].astype(np.float32)
            elif name == "face":
                out = np.zeros((n, 3), np.uint32)
                for i in range(n):
                    c = int(toks[pos]); out[i] = [int(x) for x in toks[pos + 1:pos + 4]]; pos += 1 + c
                tri = out
        return xyz, tri
    bo = "<" if fmt == "binary_little_endian" else ">"
    off = end
    for name, n, props in elems:
        if all(p[0] != "list" for p in props):
            dt = np.dtype([(p[-1], bo + tmap[p[0]]) for p in props])
            arr = np.frombuffer(data, dt, n, off); off += n * dt.itemsize
            if name == "vertex":
                xyz = np.stack([arr["x"], arr["y"], arr["z"]], 1).astype(np.float32)
        else:
            assert len(props) == 1 and name == "face"
            dt = np.dtype([("n", bo + tmap[props[0][1]]), ("i", bo + tmap[props[0][2]], (3,))])
            arr = np.frombuffer(data, dt, n, off); off += n * dt.itemsize
            assert (arr["n"] == 3).all()
            tri = arr["i"].astype(np.uint32)
    return xyz, tri


# --------------------------------------------------------------------------- RGB-D scenes
class BoxRoomScene:
    """Closed axis-aligned box room [0,sx]x[0,sy]x[0,sz] (z up) with spheres inside.

    ``render(cam2world)`` returns analytic depth (uint16 millimetres, 0 = invalid) and an
    RGB8 image for a pinhole camera looking along +z_cam with +x right, +y down
    (sensorData.h:1577-1578 back-projection convention)."""

    def __init__(self, size=(6.0, 5.0, 3.0), n_spheres: int = 4, seed: int = 0,
                 width: int = 640, height: int = 480, fx: float = FX, fy: float = FY,
                 cx: float = CX, cy: float = CY):
        rng = np.random.default_rng(seed)
        self.size = np.asarray(size, np.float64)
        self.W, self.H, self.fx, self.fy, self.cx, self.cy = width, height, fx, fy, cx, cy
        c = rng.uniform([1.0, 1.0, 0.3], self.size - [1.0, 1.0, 1.5], size=(n_spheres, 3))
        r = rng.uniform(0.2, 0.45, size=n_spheres)
        self.spheres = [(c[i], float(r[i])) for i in range(n_spheres)]
        u = (np.arange(width, dtype=np.float64) - cx) / fx
        v = (np.arange(height, dtype=np.float64) - cy) / fy
        U, V = np.meshgrid(u, v, indexing="xy")
        self.rays_cam = np.stack([U, V, np.ones_like(U)], -1)      # z_cam = 1 → t equals depth
        self.seed = seed

    def intrinsics(self) -> np.ndarray:
        K = np.eye(4, dtype=np.float32)
        K[0, 0], K[1, 1], K[0, 2], K[1, 2] = self.fx, self.fy, self.cx, self.cy
        return K

    def camera_pose(self, i: int, n: int) -> np.ndarray:
        """Smooth loop at ~1.5 m height looking outward/down slightly; ≤2 cm / ≤1° per frame for n≥1000."""
        t = 2.0 * np.pi * (i / max(n, 1))
        ctr = self.size / 2.0
        pos = np.array([ctr[0] + 0.8 * np.cos(t), ctr[1] + 0.6 * np.sin(t), 1.5 + 0.1 * np.sin(2 * t)])
        yaw = t + 0.5 * np.sin(t)
        fwd = np.array([np.cos(yaw), np.sin(yaw), -0.25]); fwd /= np.linalg.norm(fwd)
        up = np.array([0.0, 0.0, 1.0])
        right = np.cross(fwd, up); right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        T = np.eye(4)
        T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, fwd, pos
        return T.astype(np.float32)

    def orbit_pose(self, i: int, n: int, radius: float = 1.6, height: float = 1.6, target_z: float = 0.7) -> np.ndarray:
        """Frame i of n on a circle of `radius` around the room's vertical axis, looking at the axis at height target_z: every view
        holds spheres, floor and walls at several orientations, so all six degrees of freedom of a camera pose are observable
        from depth alone (camera_pose's outward views often see one wall only)."""
        t = 2.0 * np.pi * (i / max(n, 1))
        ctr = self.size / 2.0
        pos = np.array([ctr[0] + radius * np.cos(t), ctr[1] + radius * np.sin(t), height])
        fwd = np.array([ctr[0], ctr[1], target_z]) - pos; fwd /= np.linalg.norm(fwd)
        right = np.cross(fwd, [0.0, 0.0, 1.0]); right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        T = np.eye(4)
        T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, fwd, pos
        return T.astype(np.float32)

    def render(self, cam2world: np.ndarray, noise_mm: float = 0.0, drop: float = 0.0, frame_seed: int = 0):
        T = cam2world.astype(np.float64)
        R, o = T[:3, :3], T[:3, 3]
        d = self.rays_cam @ R.T                               # [H,W,3] world dirs, t = depth
        with np.errstate(divide="ignore", invalid="ignore"):
            t_best = np.full(d.shape[:2], np.inf)
            col = np.zeros(d.shape[:2] + (3,), np.float64)
            for ax in range(3):
                for wall, base in ((0.0, 0), (self.size[ax], 1)):
                    t = (wall - o[ax]) / d[..., ax]
                    hit = (t > 1e-6) & (t < t_best)
                    t_best = np.where(hit, t, t_best)
                    shade = np.array([0.35 + 0.2 * ax + 0.1 * base, 0.55 - 0.1 * ax, 0.4 + 0.15 * base])
                    col = np.where(hit[..., None], shade, col)
            for k, (c, r) in enumerate(self.spheres):
                oc = o - c
                a = (d * d).sum(-1); b = 2.0 * (d @ oc); cc = oc @ oc - r * r
                disc = b * b - 4 * a * cc
                t = (-b - np.sqrt(np.maximum(disc, 0.0))) / (2 * a)
                hit = (disc > 0) & (t > 1e-6) & (t < t_best)
                t_best = np.where(hit, t, t_best)
                shade = np.array([0.9 - 0.15 * k, 0.3 + 0.15 * k, 0.25 + 0.1 * k])
                col = np.where(hit[..., None], shade, col)
        mm = t_best * 1000.0
        rng = np.random.default_rng((self.seed << 20) ^ (frame_seed + 1))
        if noise_mm > 0:
            mm = mm + rng.normal(0.0, noise_mm, mm.shape)
        depth = np.clip(np.rint(mm), 0, 65535).astype(np.uint16)
        depth[~np.isfinite(t_best)] = 0
        if drop > 0:
            depth[rng.random(depth.shape) < drop] = 0
        rgb = np.clip(col * 255.0, 0, 255).astype(np.uint8)
        return depth, rgb


def make_frames(n_frames: int, seed: int = 0, size=(6.0, 5.0, 3.0), noise_mm: float = 0.0,
                drop: float = 0.0, invalid_pose_every: int = 0, width: int = 640, height: int = 480,
                loop_frames: int | None = None, with_color: bool = True):
    """Returns (depth u16 [N,H,W], rgb u8 [N,H,W,3] or None, poses f32 [N,4,4], K f32 [4,4])."""
    sc = BoxRoomScene(size=size, seed=seed, width=width, height=height,
                      fx=FX * width / 640.0, fy=FY * height / 480.0,
                      cx=(width - 1) / 2.0, cy=(height - 1) / 2.0)
    loop = loop_frames or max(n_frames, 1)
    D = np.zeros((n_frames, height, width), np.uint16)
    C = np.zeros((n_frames, height, width, 3), np.uint8) if with_color else None
    P = np.zeros((n_frames, 4, 4), np.float32)
    for i in range(n_frames):
        T = sc.camera_pose(i, loop)
        d, c = sc.render(T, noise_mm=noise_mm, drop=drop, frame_seed=i)
        D[i] = d
        if with_color:
            C[i] = c
        if invalid_pose_every and i % invalid_pose_every == invalid_pose_every - 1:
            T = np.full((4, 4), -np.inf, np.float32)          # sensorData.h:382 invalid pose
        P[i] = T
    return D, C, P, sc.intrinsics()


def write_sens(path, depth: np.ndarray, rgb: np.ndarray | None, poses: np.ndarray, K_depth: np.ndarray,
               K_color: np.ndarray | None = None, depth_shift: float = 1000.0, depth_comp: int = 1,
               color_comp: int = 0, sensor_name: str = "synthetic", jpeg_encoder=None):
    """Write a .sens v4 container (layout: sensorData.h:1058-1109, RGBDFrame :733-741).

    depth_comp 0 = raw u16, 1 = zlib.  color_comp 0 = raw RGB8, 2 = JPEG (needs
    ``jpeg_encoder(rgb)->bytes``, e.g. cv2.imencode)."""
    N, H, W = depth.shape
    if rgb is None:
        rgb = np.zeros((N, 1, 1, 3), np.uint8)
    CH, CW = rgb.shape[1:3]
    K_color = K_depth if K_color is None else K_color
    eye = np.eye(4, dtype=np.float32)
    with open(path, "wb") as f:
        f.write(struct.pack("<I", 4))
        nm = sensor_name.encode("ascii")
        f.write(struct.pack("<Q", len(nm))); f.write(nm)
        for m in (K_color, eye, K_depth, eye):
            f.write(np.asarray(m, "<f4").tobytes())
        f.write(struct.pack("<ii", color_comp, depth_comp))
        f.write(struct.pack("<IIII", CW, CH, W, H))
        f.write(struct.pack("<f", depth_shift))
        f.write(struct.pack("<Q", N))
        for i in range(N):
            if color_comp == 0:
                cb = rgb[i].tobytes()
            elif color_comp in (1, 2):                      # PNG / JPEG payload produced by the supplied encoder
                cb = bytes(jpeg_encoder(rgb[i]))
            else:
                raise ValueError("color_comp")
            db = depth[i].astype("<u2").tobytes()
            if depth_comp == 1:
                db = zlib.compress(db, 6)
            f.write(np.asarray(poses[i], "<f4").tobytes())
            f.write(struct.pack("<QQQQ", i * 33333, i * 33333, len(cb), len(db)))
            f.write(cb); f.write(db)
        f.write(struct.pack("<Q", 0))


class SensWriter:
    """Streaming .sens v4 writer for pre-compressed payloads (same layout as write_sens): the frame count goes into the header up
    front, frames are appended one by one, so a several-GB synthetic scan never sits in memory."""

    def __init__(self, path, n_frames: int, depth_wh, color_wh, K_depth, K_color=None, depth_shift: float = 1000.0,
                 depth_comp: int = 1, color_comp: int = 2, sensor_name: str = "synthetic"):
        self.f = open(path, "wb"); self.n = n_frames; self.i = 0
        f = self.f
        f.write(struct.pack("<I", 4))
        nm = sensor_name.encode("ascii")
        f.write(struct.pack("<Q", len(nm))); f.write(nm)
        eye = np.eye(4, dtype=np.float32)
        for m in (K_depth if K_color is None else K_color, eye, K_depth, eye):
            f.write(np.asarray(m, "<f4").tobytes())
        f.write(struct.pack("<ii", color_comp, depth_comp))
        f.write(struct.pack("<IIII", color_wh[0], color_wh[1], depth_wh[0], depth_wh[1]))
        f.write(struct.pack("<f", depth_shift))
        f.write(struct.pack("<Q", n_frames))

    def add(self, color_payload: bytes, depth_payload: bytes, pose):
        f = self.f
        f.write(np.asarray(pose, "<f4").tobytes())
        f.write(struct.pack("<QQQQ", self.i * 33333, self.i * 33333, len(color_payload), len(depth_payload)))
        f.write(color_payload); f.write(depth_payload)
        self.i += 1

    def close(self):
        assert self.i == self.n, (self.i, self.n)
        self.f.write(struct.pack("<Q", 0)); self.f.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        if a[0] is None:
            self.close()
        else:
            self.f.close()
