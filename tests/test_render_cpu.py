"""CPU checks of the render stage (DESIGN.md §6i): the camera against a binary64 restatement of mts_render.py's Transform
algebra, the oracle's first hits against a binary64 ray caster, the oracle's brute-force and BVH modes against each other,
the tables, the turntable names, argv refusals, the report size and the no-GPU failure."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import render_bindings as rb
from scannet_b200 import ScnError, render
from scannet_b200._lib import lib

ROOT = rb.ROOT
BIN = os.path.join(ROOT, "scannet_b200", "bin", "render")


# ------------------------------------------------------------------ mts_render.py's Transform algebra, 4x4 in binary64
def _translate(v):
    m = np.eye(4); m[:3, 3] = v
    return m


def _rotate(axis, deg):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    s, c = math.sin(math.radians(deg)), math.cos(math.radians(deg))
    m = np.eye(4)
    m[:3, :3] = [[a[0] * a[0] + (1 - a[0] * a[0]) * c, a[0] * a[1] * (1 - c) - a[2] * s, a[0] * a[2] * (1 - c) + a[1] * s],
                 [a[0] * a[1] * (1 - c) + a[2] * s, a[1] * a[1] + (1 - a[1] * a[1]) * c, a[1] * a[2] * (1 - c) - a[0] * s],
                 [a[0] * a[2] * (1 - c) - a[1] * s, a[1] * a[2] * (1 - c) + a[0] * s, a[2] * a[2] + (1 - a[2] * a[2]) * c]]
    return m


def _look_at(p, t, up):
    d = (t - p) / np.linalg.norm(t - p)
    left = np.cross(up, d); left /= np.linalg.norm(left)
    m = np.eye(4); m[:3, 0] = left; m[:3, 1] = np.cross(d, left); m[:3, 2] = d; m[:3, 3] = p
    return m


def _point(m, p):
    return (m @ np.append(p, 1.0))[:3]


def _vector(m, v):
    return m[:3, :3] @ v


def reference_camera(xyz, W, H, theta=0.0, turntable=False, world_up=(0, 0, 1), camera_up=(0, 1, 0), camera_offset=(0, 0, 0), mult=2.5):
    """mts_render.py:69-106 and Mitsuba's perspective sensor (fov 45 along x): origin, and the film corner and pixel steps."""
    x = np.asarray(xyz, np.float64)
    lo, hi = x.min(0), x.max(0)
    c = (lo + hi) * 0.5
    r = np.linalg.norm(hi - c)
    up = np.asarray(world_up, float)
    off = np.asarray(camera_offset, float) + up
    origin = c + mult * r * off / np.linalg.norm(off)
    cam_up = np.asarray(camera_up, float)
    if turntable:
        R = _translate(c) @ _rotate(up, theta) @ _translate(-c)
    else:
        R = _rotate(up, theta)
    T = _look_at(_point(R, origin), c, _vector(R, cam_up))
    # camera space: x = left, y = up, z = forward; the film's x runs along -x, its y (down) along -y
    th = math.tan(math.radians(22.5))
    step = 2 * th / W
    du = _vector(T, np.array([-step, 0, 0]))
    dv = _vector(T, np.array([0, -step, 0]))
    p00 = _vector(T, np.array([th, th * H / W, 1.0]))
    return T[:3, 3], p00, du, dv, r


def _mesh(seed=0, n=40, scale=1.0, shift=(0, 0, 0)):
    rng = np.random.default_rng(seed)
    xyz = (rng.uniform(-1, 1, (3 * n, 3)) * scale + shift).astype(np.float32)
    tri = np.arange(3 * n, dtype=np.uint32).reshape(-1, 3)
    return xyz, tri


CAMERA_CASES = [
    dict(),
    dict(theta=37.5),
    dict(theta=120, turntable=True),
    dict(theta=-15, world_up=(0, 1, 0), camera_up=(0, 0, 1)),
    dict(theta=200, turntable=True, camera_offset=tuple(np.array([1, 2, 0.5]) / np.linalg.norm([1, 2, 0.5])), mult=1.7),
    dict(world_up=(1, 0, 0), camera_up=(0, 1, 0), camera_offset=(0, 0.6, 0.8), mult=0.5),
]


@pytest.mark.parametrize("case", range(len(CAMERA_CASES)))
@pytest.mark.parametrize("film", [(640, 480), (33, 17)])
def test_camera_matches_the_transform_algebra(built, case, film):
    kw = dict(CAMERA_CASES[case])
    xyz, _ = _mesh(case, scale=2.0, shift=(10, -3, 1.5))
    W, H = film
    p = render.default_params(width=W, height=H, world_up=kw.get("world_up", (0, 0, 1)), camera_up=kw.get("camera_up", (0, 1, 0)),
                              camera_offset=kw.get("camera_offset", (0, 0, 0)), bsphere_mult=kw.get("mult", 2.5))
    cam = render.camera(xyz, p, kw.get("theta", 0.0), kw.get("turntable", False))
    o, p00, du, dv, r = reference_camera(xyz, W, H, **kw)
    s = np.linalg.norm(o) + 1
    np.testing.assert_allclose(np.array(cam.origin), o, rtol=0, atol=2e-7 * s)
    np.testing.assert_allclose(np.array(cam.p00), p00, rtol=0, atol=2e-7)
    np.testing.assert_allclose(np.array(cam.du), du, rtol=0, atol=2e-7 / W)
    np.testing.assert_allclose(np.array(cam.dv), dv, rtol=0, atol=2e-7 / W)
    assert cam.t_near == np.float32(0.01) and cam.ao_length == np.float32(r) and cam.t_eps == np.float32(r * 2.0 ** -16)


def test_default_camera_looks_straight_down_unmirrored(built):
    xyz, _ = _mesh(3)
    cam = render.camera(xyz)
    c = (xyz.astype(np.float64).min(0) + xyz.astype(np.float64).max(0)) / 2
    assert np.allclose(np.array(cam.origin)[:2], c[:2], atol=1e-6) and cam.origin[2] > c[2]
    # image right = +x, image down = -y seen from above (x right, y up): not mirrored
    assert cam.du[0] > 0 and abs(cam.du[1]) < 1e-9 and cam.dv[1] < 0 and abs(cam.dv[0]) < 1e-9
    assert cam.p00[2] == -1.0


def test_single_view_rotates_about_the_world_origin_and_turntable_about_the_centre(built):
    xyz, _ = _mesh(4, shift=(5, 0, 0))
    a = render.camera(xyz, theta=90)
    b = render.camera(xyz, theta=90, turntable=True)
    c = (xyz.astype(np.float64).min(0) + xyz.astype(np.float64).max(0)) / 2
    assert np.allclose(np.array(a.origin)[:2], (-c[1], c[0]), atol=1e-5)      # (cx, cy) swung to (-cy, cx)
    assert np.allclose(np.array(b.origin)[:2], c[:2], atol=1e-5)              # stays above the centre
    t0 = render.camera(xyz, turntable=True)
    assert bytes(t0) == bytes(render.camera(xyz))


@pytest.mark.parametrize("kw, msg", [(dict(camera_up=(0, 0, 1)), "parallel"), (dict(world_up=(0, 0, 0)), "non-zero"),
                                     (dict(world_up=(0, 0, 1), camera_offset=(0, 0, -1)), "non-zero"),
                                     (dict(bsphere_mult=0.0), "target")])
def test_camera_refusals(built, kw, msg):
    xyz, _ = _mesh(5)
    with pytest.raises(ScnError) as e:
        render.camera(xyz, render.default_params(**kw))
    assert e.value.code == -1 and msg in str(e.value)
    bad = xyz.copy(); bad[3, 1] = np.nan
    with pytest.raises(ScnError) as e:
        render.camera(bad)
    assert e.value.code == -1


# ------------------------------------------------------------------ first hits against binary64
def _ref_hits(xyz, tri, o, d, tmin, eps):
    """binary64 closest hits: (face or NO_HIT, t, ambiguous) — ambiguous within eps of an edge, or of a tie in t"""
    V = xyz.astype(np.float64)[tri.astype(np.int64)]            # F, 3, 3
    o = o.astype(np.float64); d = d.astype(np.float64)
    e1, e2 = V[:, 1] - V[:, 0], V[:, 2] - V[:, 0]
    faces = np.full(len(o), rb.NO_HIT, np.uint32); ts = np.full(len(o), np.inf); amb = np.zeros(len(o), bool)
    for i in range(len(o)):
        p = np.cross(d[i], e2); det = np.einsum("ij,ij->i", e1, p)
        ok = np.abs(det) > 1e-300
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        s = o[i] - V[:, 0]
        u = np.einsum("ij,ij->i", s, p) * inv
        q = np.cross(s, e1)
        v = (q @ d[i]) * inv
        t = np.einsum("ij,ij->i", q, e2) * inv
        w = 1 - u - v
        bmin = np.minimum(np.minimum(u, v), w)
        hit = ok & (bmin >= 0) & (t > tmin)
        tt = np.where(hit, t, np.inf)
        f = int(np.argmin(tt))
        best = tt[f]
        # an edge within eps of the ray in front of (or at) the closest hit could flip the answer under rounding
        if (ok & (np.abs(bmin) < eps) & (t > tmin) & (t <= best + eps * max(1.0, abs(best) if np.isfinite(best) else 1.0))).any():
            amb[i] = True
        if hit.any():
            ts[i] = best; faces[i] = f
            second = np.sort(tt)[1] if hit.sum() > 1 else np.inf
            if second - best <= eps * max(1.0, abs(best)) or abs(best - tmin) < eps:
                amb[i] = True
    return faces, ts, amb


def _rays(rng, n, axis_parallel=False):
    o = rng.uniform(-1 if axis_parallel else -3, 1 if axis_parallel else 3, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    if axis_parallel:
        k = rng.integers(0, 3, n)
        d = np.zeros((n, 3), np.float32); d[np.arange(n), k] = rng.choice([-1.0, 1.0], n)
        d[: n // 2] *= 0.37
    o -= d * 4.0
    return o, d


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("axis_parallel", [False, True])
def test_first_hits_match_binary64(built, seed, axis_parallel):
    rng = np.random.default_rng(seed)
    xyz, tri = _mesh(seed, n=60)
    o, d = _rays(rng, 3000, axis_parallel)
    eps = 1e-5
    want_f, want_t, amb = _ref_hits(xyz, tri, o, d, 0.0, eps)
    for mode in (0, 1):
        f, t = rb.first_hits(xyz, tri, o, d, 0.0, mode)
        keep = ~amb
        assert (f[keep] == want_f[keep]).all()
        h = keep & (want_f != rb.NO_HIT)
        np.testing.assert_allclose(t[h], want_t[h], rtol=2e-5, atol=1e-6)
    assert amb.mean() < 0.05, amb.mean()          # the excluded share, quoted in DESIGN.md §6i
    assert (want_f[~amb] != rb.NO_HIT).sum() > 300


def _room_mesh():
    """axis-aligned floor and walls made of grid quads, with duplicate and zero-area faces mixed in"""
    quads = []
    n = 6
    for i in range(n):
        for j in range(n):
            a, b = i / n, (i + 1) / n
            c, e = j / n, (j + 1) / n
            quads.append([(a, c, 0), (b, c, 0), (b, e, 0), (a, e, 0)])          # floor z = 0
            quads.append([(0, a, c), (0, b, c), (0, b, e), (0, a, e)])          # wall x = 0
            quads.append([(a, 1, c), (b, 1, c), (b, 1, e), (a, 1, e)])          # wall y = 1
    xyz, tri = [], []
    for q in quads:
        k = len(xyz); xyz += q; tri += [(k, k + 1, k + 2), (k, k + 2, k + 3)]
    tri += tri[:10]                                                              # coplanar duplicates (face-index ties)
    tri += [(0, 0, 1), (2, 2, 2)]                                                # zero-area faces
    return np.array(xyz, np.float32), np.array(tri, np.uint32)


def test_brute_force_and_bvh_agree_on_axis_parallel_rays(built):
    xyz, tri = _room_mesh()
    g = np.linspace(-0.1, 1.1, 97, dtype=np.float32)
    X, Y = np.meshgrid(g, g)
    o = np.stack([X.ravel(), Y.ravel(), np.full(X.size, 2.0, np.float32)], 1)
    d = np.tile(np.float32([0, 0, -1]), (len(o), 1))
    o2 = np.stack([np.full(X.size, 2.0, np.float32), X.ravel(), Y.ravel()], 1)
    d2 = np.tile(np.float32([-1, 0, 0]), (len(o), 1))
    O, D = np.concatenate([o, o2]), np.concatenate([d, d2])
    f0, t0 = rb.first_hits(xyz, tri, O, D, 0.0, 0)
    f1, t1 = rb.first_hits(xyz, tri, O, D, 0.0, 1)
    assert (f0 == f1).all() and t0.tobytes() == t1.tobytes()
    assert (f0 != rb.NO_HIT).sum() > 0.6 * len(O)
    dup = len(tri) - 12
    assert not np.isin(f0, np.arange(dup, len(tri))).any()          # duplicates lose the tie, zero-area faces are never hit


@pytest.mark.parametrize("integrator, spp, depth", [(0, 1, 1), (0, 4, 3), (1, 3, 5), (0, 16, 5)])
def test_oracle_render_modes_agree(built, integrator, spp, depth):
    xyz, tri = _room_mesh()
    rgb = np.random.default_rng(1).integers(0, 256, (len(xyz), 3), dtype=np.uint8)
    p = render.RenderParams()
    p.width, p.height, p.samples, p.integrator, p.max_depth, p.exposure = 24, 17, spp, integrator, depth, 1.0
    p.world_up[:] = (0, 0, 1); p.camera_up[:] = (0, 1, 0); p.bsphere_mult = 2.5
    # the camera in numpy (no library call: the CPU suite may run where the CUDA library is absent only in name)
    o, p00, du, dv, r = reference_camera(xyz, 24, 17, theta=30, turntable=True)
    cam = render.RenderCamera()
    cam.origin[:], cam.p00[:], cam.du[:], cam.dv[:] = o, p00, du, dv
    cam.t_near, cam.t_eps, cam.ao_length = 0.01, r * 2.0 ** -16, r
    a, ca = rb.oracle_render(xyz, rgb, tri, p, [cam], mode=0)
    b, cb = rb.oracle_render(xyz, rgb, tri, p, [cam], mode=1)
    assert a.tobytes() == b.tobytes() and ca == cb
    assert ca["primary_rays"] == 24 * 17 * spp and 0 < ca["primary_hits"] < ca["primary_rays"]
    sub, cs = rb.oracle_render(xyz, rgb, tri, p, [cam], mode=1, rect=(5, 3, 7, 9))
    assert sub.tobytes() == a[:, 3:12, 5:12].tobytes()


# ------------------------------------------------------------------ tables, names, argv, ABI
def test_tables_are_the_binary64_srgb_curve(built):
    lin, thr = rb.tables()
    dec = lambda x: np.where(x <= 0.04045, x / 12.92, ((x + 0.055) / 1.055) ** 2.4)    # noqa: E731
    assert lin.tobytes() == dec(np.arange(256) / 255.0).astype(np.float32).tobytes()
    assert thr.tobytes() == dec((np.arange(255) + 0.5) / 255.0).astype(np.float32).tobytes()
    assert (np.diff(thr) > 0).all() and lin[0] == 0 and lin[255] == 1
    # counting thresholds is sRGB encoding rounded to the nearest byte (away from the exact midpoints)
    v = np.random.default_rng(0).uniform(0, 1.2, 20000).astype(np.float32)
    enc = np.where(v <= 0.0031308, 12.92 * v.astype(np.float64), 1.055 * v.astype(np.float64) ** (1 / 2.4) - 0.055)
    want = np.clip(np.floor(enc * 255 + 0.5), 0, 255)
    got = np.searchsorted(thr, v, side="right")
    assert (got == want).mean() > 0.999


@pytest.mark.parametrize("D, n", [(5, 72), (7, 51), (360, 1), (1, 360)])
def test_turntable_frames(D, n):
    names = render.turntable_names("/x/scene_vh_clean_2.ply", D)
    assert len(names) == n == len(render.turntable_angles(D))
    assert names[0] == "/x/scene_vh_clean_2.ply_000.png" and render.turntable_angles(D)[-1] == (n - 1) * D


@pytest.mark.parametrize("args, code, msg", [
    (["--cameras", "c.txt", "m.ply"], 1, "--cameras"),
    (["--integrator", "mlt", "m.ply"], 1, "'mlt' is not supported"),
    (["--integrator=vpl", "m.ply"], 1, "'vpl' is not supported"),
    (["--integrator", "direct", "m.ply"], 2, "invalid integrator"),
    (["--samples", "x", "m.ply"], 2, "invalid argument --samples"),
    (["--world_up", "1,2", "m.ply"], 2, "invalid argument --world_up"),
    (["--frames_per_degree", "0", "m.ply"], 2, "invalid argument"),
    (["--render_turntable"], 2, "mesh argument is required"),
    (["a.ply", "b.ply"], 2, "unrecognised argument"),
    (["--bogus", "1", "m.ply"], 2, "invalid argument --bogus"),
    (["--width"], 2, "missing value"),
])
def test_argv_refusals(built, args, code, msg):
    r = subprocess.run([BIN] + args, capture_output=True, text=True)
    assert r.returncode == code and msg in r.stderr, r.stderr


def test_missing_mesh_is_an_io_error(built, tmp_path):
    r = subprocess.run([BIN, str(tmp_path / "none.ply")], capture_output=True, text=True)
    assert r.returncode == 1 and not list(tmp_path.iterdir())


def test_report_binding_matches_the_library_struct(built):
    assert render.report_sizeof() == C.sizeof(render.RenderReport)


def test_render_refusals(built):
    xyz, tri = _mesh(6)
    cam = render.camera(xyz)
    for bad_tri in (np.zeros((0, 3), np.uint32), np.array([[0, 1, len(xyz)]], np.uint32)):
        with pytest.raises(ScnError) as e:
            render.render(xyz, None, bad_tri, cams=cam)
        assert e.value.code == -1
    bad = xyz.copy(); bad[0, 0] = np.inf
    with pytest.raises(ScnError) as e:
        render.render(bad, None, tri, cams=cam)
    assert e.value.code == -1
    for k, v in (("samples", 0), ("samples", 257), ("max_depth", 0), ("integrator", 2), ("width", 0)):
        with pytest.raises(ScnError) as e:
            render.render(xyz, None, tri, render.default_params(**{k: v}), cams=cam)
        assert e.value.code == -1, (k, v)


def test_no_gpu_means_loud_failure(built, tmp_path):
    if lib().scn_device_count() > 0:
        return                      # on the GPU machine this test has nothing to show
    xyz, tri = _mesh(7)
    with pytest.raises(ScnError) as e:
        render.render(xyz, None, tri)
    assert e.value.code == -2
    from scannet_b200 import meshclean
    ply = tmp_path / "m.ply"
    _save_ply(ply, xyz, tri)
    assert meshclean.load_rgb(str(ply))[0].shape == xyz.shape
    r = subprocess.run([BIN, str(ply)], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stderr and not (tmp_path / "m.png").exists()


def _save_ply(path, xyz, tri):
    head = f"ply\nformat binary_little_endian 1.0\nelement vertex {len(xyz)}\nproperty float x\nproperty float y\nproperty float z\n" \
           f"element face {len(tri)}\nproperty list uchar int vertex_indices\nend_header\n"
    body = np.ascontiguousarray(xyz, "<f4").tobytes()
    f = np.zeros(len(tri), dtype=[("n", "u1"), ("i", "<i4", 3)]); f["n"] = 3; f["i"] = tri
    with open(path, "wb") as fh:
        fh.write(head.encode() + body + f.tobytes())
