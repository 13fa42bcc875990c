"""GPU parity: the render kernels (scannet_b200/csrc/render.cu through the C ABI) vs the CPU oracle (oracle/render_oracle.c),
bit for bit: RGBA bytes, the ray and hit counters, and the PNG files of the CLI."""
import io
import os
import subprocess

import numpy as np
import pytest

import render_bindings as rb
from scannet_b200 import meshclean, meshsimplify, render, synth, tsdf

pytestmark = pytest.mark.gpu
ROOT = rb.ROOT
BIN = os.path.join(ROOT, "scannet_b200", "bin")
GOLDEN = os.path.join(ROOT, "tests", "golden")


def check(xyz, rgb, tri, cams=None, mode=1, **kw):
    p = render.default_params(**kw)
    if cams is None:
        cams = [render.camera(xyz, p)]
    g, rep = render.render(xyz, rgb, tri, p, cams)
    o, cnt = rb.oracle_render(xyz, rgb, tri, p, cams, mode=mode)
    assert g.tobytes() == o.tobytes(), f"RGBA differs at {np.argwhere(g != o)[:5].tolist()}"
    assert {k: rep[k] for k in render.COUNTERS} == cnt
    assert rep["primary_rays"] == len(cams) * p.width * p.height * p.samples
    return g, rep


def _room(n=8, with_rgb=True, seed=0):
    """axis-aligned floor and two walls of grid quads (the default camera looks straight down: axis-parallel rays in its
    centre row and column), a box on the floor, coplanar duplicate faces and zero-area faces"""
    xyz, tri = [], []

    def quad(q):
        k = len(xyz); xyz.extend(q); tri.extend([(k, k + 1, k + 2), (k, k + 2, k + 3)])
    for i in range(n):
        for j in range(n):
            a, b, c, e = i / n, (i + 1) / n, j / n, (j + 1) / n
            quad([(a, c, 0), (b, c, 0), (b, e, 0), (a, e, 0)])
            quad([(0, a, c), (0, b, c), (0, b, e), (0, a, e)])
            quad([(a, 1, c), (b, 1, c), (b, 1, e), (a, 1, e)])
    quad([(0.5, 0.25, 0.25), (0.75, 0.25, 0.25), (0.75, 0.5, 0.25), (0.5, 0.5, 0.25)])
    tri.extend(tri[: 3 * n])
    tri.extend([(0, 0, 1), (5, 5, 5), (1, 2, 1)])
    x = np.array(xyz, np.float32); t = np.array(tri, np.uint32)
    c = np.random.default_rng(seed).integers(0, 256, (len(x), 3), dtype=np.uint8) if with_rgb else None
    return x, c, t


@pytest.fixture(scope="module")
def gates():
    return meshclean.load_rgb(os.path.join(GOLDEN, "gates381.ply"))


@pytest.fixture(scope="module")
def decimated():
    """a fused synthetic room at 4 mm, cleaned (clean.mlx) and decimated twice (simplify.mlx): a `_vh_clean_2` mesh"""
    p = tsdf.default_params(width=160, height=120, voxel_size=0.004, max_blocks=1 << 16, hash_slots=1 << 18, batch_frames=4)
    D, Cc, P, K = synth.make_frames(8, seed=11, width=160, height=120, loop_frames=300, noise_mm=1.0)
    vol = tsdf.TsdfVolume(p, device=0)
    vol.integrate_batch(D, Cc, P, K)
    vol.sync()
    xyz, rgb, tri = vol.extract_mesh()
    x, c, t, _ = meshclean.clean(xyz, tri, rgb)
    sp, sa = meshsimplify.default_params()
    for _ in range(2):
        x, c, t, _ = meshsimplify.simplify(x, t, c, sp, sa)
    assert len(t) > 1000
    return x, c, t


@pytest.mark.parametrize("kw", [dict(width=64, height=48), dict(width=37, height=23, samples=3, integrator="ao"),
                                dict(width=1, height=1, samples=16), dict(width=50, height=31, samples=1, max_depth=1)])
def test_gates381(built, gates, kw):
    xyz, rgb, tri = gates
    g, rep = check(xyz, rgb, tri, **kw)
    assert rep["primary_hits"] > 0 or kw["width"] == 1


@pytest.mark.parametrize("kw", [dict(width=80, height=60, samples=4), dict(width=41, height=29, samples=16, max_depth=8),
                                dict(width=33, height=25, samples=5, integrator="ao")])
def test_decimated_room(built, decimated, kw):
    xyz, rgb, tri = decimated
    _, rep = check(xyz, rgb, tri, **kw)
    assert rep["primary_hits"] > 0 and rep["secondary_rays"] > 0


def test_decimated_room_brute_force(built, decimated):
    xyz, rgb, tri = decimated
    check(xyz, rgb, tri, mode=0, width=24, height=18, samples=2)


def test_single_triangle(built):
    xyz = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.2]], np.float32)
    rgb = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255]], np.uint8)
    tri = np.array([[0, 1, 2]], np.uint32)
    for kw in (dict(width=40, height=30, samples=4), dict(width=7, height=5, samples=2, integrator="ao")):
        g, rep = check(xyz, rgb, tri, **kw)
        assert 0 < rep["primary_hits"] < rep["primary_rays"]


@pytest.mark.parametrize("with_rgb", [True, False])
@pytest.mark.parametrize("kw", [dict(width=64, height=64, samples=4, max_depth=3), dict(width=65, height=47, samples=7, integrator="ao"),
                                dict(width=31, height=31, samples=1, max_depth=2)])
def test_axis_aligned_room_duplicates_and_zero_area_faces(built, with_rgb, kw):
    xyz, rgb, tri = _room(with_rgb=with_rgb)
    check(xyz, rgb, tri, **kw)
    check(xyz, rgb, tri, mode=0, **kw)


def test_duplicate_faces_lose_the_tie(built):
    """the same triangle twice, the copy with the smaller index is the one hit: swapping colours shows which"""
    xyz = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 0, 0], [1, 0, 0], [1, 1, 0]], np.float32)
    rgb = np.array([[255, 255, 255]] * 3 + [[0, 0, 0]] * 3, np.uint8)
    a, _ = check(xyz, rgb, np.array([[0, 1, 2], [3, 4, 5]], np.uint32), width=20, height=20, samples=2, max_depth=2)
    b, _ = check(xyz, rgb, np.array([[3, 4, 5], [0, 1, 2]], np.uint32), width=20, height=20, samples=2, max_depth=2)
    assert a[..., :3].sum() > b[..., :3].sum()


def test_camera_inside_the_bounding_sphere(built, decimated):
    xyz, rgb, tri = decimated
    for mult in (0.3, 0.9):
        p = render.default_params(width=48, height=36, samples=2, bsphere_mult=mult)
        check(xyz, rgb, tri, cams=[render.camera(xyz, p, theta=25.0)], width=48, height=36, samples=2, bsphere_mult=mult)


def test_turntable_equals_views_one_at_a_time(built, gates):
    xyz, rgb, tri = gates
    p = render.default_params(width=40, height=30, samples=3)
    cams = [render.camera(xyz, p, a, turntable=True) for a in render.turntable_angles(45)]
    g, rep = check(xyz, rgb, tri, cams=cams, width=40, height=30, samples=3)
    for i, c in enumerate(cams):
        one, _ = render.render(xyz, rgb, tri, p, [c])
        assert one.tobytes() == g[i:i + 1].tobytes(), i
    assert rep["views"] == 8


def test_asymmetric_mesh_pins_the_orientation(built):
    """an L on the floor: its long arm along +x, the short one along +y, seen from above, image right = +x, image up = +y"""
    xyz = np.array([[0, 0, 0], [3, 0, 0], [3, 0.5, 0], [0, 0.5, 0], [0, 0.5, 0], [0.5, 0.5, 0], [0.5, 1.5, 0], [0, 1.5, 0]], np.float32)
    tri = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]], np.uint32)
    g, _ = check(xyz, None, tri, width=64, height=48, samples=1)
    cov = g[0, ..., 3] > 0
    ys, xs = np.nonzero(cov)
    # the long arm spans far more columns than rows, and the short arm sits on the left, above the long one
    assert xs.max() - xs.min() > 1.5 * (ys.max() - ys.min())
    left = cov[:, : xs.min() + (xs.max() - xs.min()) // 6]
    lys = np.nonzero(left)[0]
    assert lys.min() < ys.min() + (ys.max() - ys.min()) // 3
    rys = np.nonzero(cov[:, xs.max() - (xs.max() - xs.min()) // 6:])[0]
    assert rys.min() > ys.min() + (ys.max() - ys.min()) // 2


def test_cli_single_view_and_turntable(built, gates, tmp_path):
    from PIL import Image
    xyz, rgb, tri = gates
    src = os.path.join(GOLDEN, "gates381.ply")
    mesh = tmp_path / "scene_vh_clean_2.ply"
    mesh.write_bytes(open(src, "rb").read())
    r = subprocess.run([os.path.join(BIN, "render"), "--width", "48", "--height", "36", "--samples", "2", str(mesh)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    png = tmp_path / "scene_vh_clean_2.png"
    img = np.array(Image.open(io.BytesIO(png.read_bytes())))
    p = render.default_params(width=48, height=36, samples=2)
    o, _ = rb.oracle_render(xyz, rgb, tri, p, [render.camera(xyz, p)])
    assert img.shape == (36, 48, 4) and img.tobytes() == o[0].tobytes()
    # same render through -o and the in-process entry point: the same PNG bytes
    assert render.main(["--width=48", "--height=36", "--samples=2", "-o", str(tmp_path / "b.png"), str(mesh)]) == 0
    assert (tmp_path / "b.png").read_bytes() == png.read_bytes()
    r = subprocess.run([os.path.join(BIN, "render"), "--width", "16", "--height", "12", "--samples", "1", "--integrator", "ao",
                        "--render_turntable", "--frames_per_degree", "40", str(mesh)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    names = render.turntable_names(str(mesh), 40)
    assert len(names) == 9 and all(os.path.exists(n) for n in names)
    p = render.default_params(width=16, height=12, samples=1, integrator="ao")
    cams = [render.camera(xyz, p, a, turntable=True) for a in render.turntable_angles(40)]
    o, _ = rb.oracle_render(xyz, rgb, tri, p, cams)
    for i, n in enumerate(names):
        assert np.array(Image.open(n)).tobytes() == o[i].tobytes(), n
