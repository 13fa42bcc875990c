"""GPU parity: mesh decimation (scannet_b200/csrc/meshsimplify.cu through the C ABI) vs the CPU oracle
(oracle/meshsimplify_oracle.c, then oracle/meshclean_oracle.c for the clean filters), bit for bit: vertex bytes, colours,
indices and every counter of the report."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import meshclean_bindings as mb
import meshsimplify_bindings as sb
import oracle_bindings as ob
from meshsimplify_cases import fan, grid, soup, strip
from scannet_b200 import ScnError, meshclean, meshsimplify, synth, tsdf

pytestmark = pytest.mark.gpu
ROOT = mb.ROOT
BIN = os.path.join(ROOT, "scannet_b200", "bin")
GOLDEN = os.path.join(ROOT, "tests", "golden")
AFTER = {"merge_threshold": 0.0010689, "min_piece_faces": 1000}           # simplify.mlx's clean filters


def check(xyz, tri, rgb=None, after=None, **kw):
    """kw: target_faces / target_perc / quality_thr (default simplify.mlx); after: dict of clean parameters or None"""
    p, a = meshsimplify.default_params(**kw)
    ga = None
    if after is not None:
        ga = meshclean.default_params(**after)
    gx, gc, gt, rep = meshsimplify.simplify(xyz, tri, rgb, p, ga)
    okw = {"target_faces": p.target_faces, "target_perc": p.target_perc, "quality_thr": p.quality_thr}
    ox, oc, ot, cnt, ccnt = sb.oracle_simplify(xyz, tri, rgb, after=after, **okw)
    assert gx.tobytes() == ox.tobytes(), "vertices differ"
    assert (gc is None and oc is None) or gc.tobytes() == oc.tobytes(), "colours differ"
    assert gt.tobytes() == ot.tobytes(), "faces differ"
    assert {k: rep[k] for k in sb.COUNTERS} == cnt
    if after is not None:
        assert {k: rep["clean"][k] for k in mb.COUNTERS} == ccnt
    assert (rep["vertices_in"], rep["faces_in"], rep["vertices_out"], rep["faces_out"]) == (len(xyz), len(tri), len(ox), len(ot))
    return gx, gc, gt, rep


@pytest.fixture(scope="module")
def mc_clean():
    """the marching-cubes mesh of a fused synthetic scene at 4 mm voxels, after clean.mlx"""
    p = tsdf.default_params(width=160, height=120, voxel_size=0.004, max_blocks=1 << 16, hash_slots=1 << 18, batch_frames=4)
    D, Cc, P, K = synth.make_frames(8, seed=11, width=160, height=120, loop_frames=300, noise_mm=1.0)
    vol = tsdf.TsdfVolume(p, device=0)
    vol.integrate_batch(D, Cc, P, K)
    vol.sync()
    xyz, rgb, tri = vol.extract_mesh()
    x, c, t, _ = meshclean.clean(xyz, tri, rgb)
    return x, c, t


def test_gates381(built):
    xyz, rgb, tri = meshclean.load_rgb(os.path.join(GOLDEN, "gates381.ply"))
    _, _, _, rep = check(xyz, tri, rgb, after=AFTER)
    assert rep["collapses"] > 0 and rep["faces_collapsed"] + rep["faces_out"] <= len(tri)
    check(xyz, tri, rgb)


@pytest.mark.parametrize("kw", [{"target_perc": 0.5}, {"target_perc": 0.2}, {"target_perc": 0.05}, {"target_perc": 0.0, "target_faces": 7777},
                                {"target_perc": 0.2, "quality_thr": 0.0}, {"target_perc": 0.2, "quality_thr": 1.0}])
def test_marching_cubes_mesh_after_clean(built, mc_clean, kw):
    xyz, rgb, tri = mc_clean
    assert len(tri) > 20000
    _, _, gt, rep = check(xyz, tri, rgb, after=AFTER, **kw)
    assert len(tri) - rep["faces_collapsed"] <= rep["target_faces"]
    print(f"{kw}: {rep['faces_in']} -> {rep['faces_out']} faces in {rep['rounds']} rounds ({rep['collapses']} collapses, largest ring "
          f"{rep['max_vertex_faces']}), quadrics {rep['quadrics_ms']:.2f} rounds {rep['rounds_ms']:.2f} autoclean {rep['autoclean_ms']:.2f} "
          f"clean {rep['clean_ms']:.2f} ms")


def test_no_clean_filters_and_rgb_optional(built, mc_clean):
    xyz, rgb, tri = mc_clean
    check(xyz, tri, None, target_perc=0.3)
    check(xyz, tri, rgb, target_perc=0.3)


def test_small_and_degenerate_inputs(built):
    check(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32))
    check(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32), after=AFTER)
    pts = np.random.default_rng(1).uniform(-1, 1, (50, 3)).astype(np.float32)
    _, _, _, rep = check(pts, np.zeros((0, 3), np.uint32))
    assert rep["vertices_out"] == 0
    one = np.array([[0, 1, 2]], np.uint32)
    for kw in ({}, {"target_perc": 0.0, "target_faces": 0}, {"target_perc": 1.0}):
        check(pts, one, **kw)
    xyz, tri = grid(15, 14, seed=3)
    _, _, gt, rep = check(xyz, tri, target_perc=0.0, target_faces=0)          # collapse until nothing is left
    assert len(gt) == 0 and rep["faces_collapsed"] == len(tri)
    _, _, gt, rep = check(xyz, tri, target_perc=0.0, target_faces=len(tri))  # nothing to do
    assert rep["rounds"] == 0 and gt.tobytes() == tri.tobytes()
    check(xyz, tri, target_perc=0.0, target_faces=10 ** 12)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_non_manifold_duplicate_and_degenerate_faces(built, seed):
    xyz, tri = soup(400, 1500, seed=seed)
    rgb = np.random.default_rng(seed).integers(0, 256, (len(xyz), 3)).astype(np.uint8)
    for kw in ({"target_perc": 0.2}, {"target_perc": 0.0, "target_faces": 0}, {"target_perc": 0.5, "quality_thr": 1.0}):
        check(xyz, tri, rgb, **kw)
    sx, st = strip(3000, seed=seed)
    check(sx, st, target_perc=0.1)


def test_fan_around_one_hub(built):
    """every vertex is a neighbour of the hub, so a round selects one or very few collapses: the worst case for rounds"""
    xyz, tri = fan(600, seed=4)
    _, _, _, rep = check(xyz, tri)
    assert rep["rounds"] >= rep["collapses"] // 2
    print(f"fan of {len(tri)}: {rep['rounds']} rounds, {rep['rounds_ms']:.1f} ms in rounds, {rep['total_ms']:.1f} ms total")
    xyz, tri = fan(20000, seed=5)
    p, _ = meshsimplify.default_params(target_perc=0.95)
    a = meshsimplify.simplify(xyz, tri, None, p)
    b = meshsimplify.simplify(xyz, tri, None, p)
    rep = a[3]
    assert all(u.tobytes() == v.tobytes() for u, v in zip(a[:3:2], b[:3:2]))
    assert rep["rounds"] >= rep["collapses"] // 2 and len(tri) - rep["faces_collapsed"] <= rep["target_faces"]
    print(f"fan of {len(tri)} to 95 %: {rep['rounds']} rounds, {rep['rounds_ms']:.1f} ms in rounds ({rep['rounds_ms'] / rep['rounds']:.3f} ms "
          f"per round, largest ring {rep['max_vertex_faces']})")


def test_two_runs_identical(built, mc_clean):
    xyz, rgb, tri = mc_clean
    p, a = meshsimplify.default_params()
    r1 = meshsimplify.simplify(xyz, tri, rgb, p, a)
    r2 = meshsimplify.simplify(xyz, tri, rgb, p, a)
    for u, v in zip(r1[:3], r2[:3]):
        assert u.tobytes() == v.tobytes()
    assert {k: r1[3][k] for k in sb.COUNTERS} == {k: r2[3][k] for k in sb.COUNTERS}


def test_refusals(built):
    xyz, tri = grid(4, 4)
    for kw in ({"target_perc": float("nan")}, {"target_perc": -0.1}, {"target_perc": 1.5}, {"quality_thr": -1.0}, {"quality_thr": float("nan")}):
        p, _ = meshsimplify.default_params(**kw)
        with pytest.raises(ScnError) as e:
            meshsimplify.simplify(xyz, tri, None, p)
        assert e.value.code == -1
    for bad in (np.inf, -np.inf, np.nan):
        x = xyz.copy(); x[3, 1] = bad
        with pytest.raises(ScnError) as e:
            meshsimplify.simplify(x, tri)
        assert e.value.code == -1
    with pytest.raises(ScnError) as e:
        meshsimplify.simplify(xyz, np.array([[0, 1, len(xyz)]], np.uint32))
    assert e.value.code == -1
    with pytest.raises(ScnError) as e:
        meshsimplify.simplify(xyz, tri, None, None, meshclean.default_params(merge_threshold=0.0))
    assert e.value.code == -1


def save_ply(path, x, c, t):
    from scannet_b200._lib import check as scn_check, lib
    scn_check(lib().scn_mesh_save_ply(str(path).encode(), x.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p) if c is not None else None,
                                      C.c_uint64(len(x)), t.ctypes.data_as(C.c_void_p), C.c_uint64(len(t))))


def test_fuse_clean_simplify_twice_segmentator_end_to_end(built, tmp_path):
    """synthetic .sens -> fuse -> _vh.ply -> meshclean (clean.mlx) -> meshsimplify (simplify.mlx) twice -> _vh_clean_2.ply -> segmentator"""
    from scipy.spatial import cKDTree
    D, Cc, P, K = synth.make_frames(16, seed=4, width=160, height=120, loop_frames=600, noise_mm=1.5)
    sens = tmp_path / "scene.sens"
    synth.write_sens(str(sens), D, Cc, P, K, depth_comp=1, color_comp=0)
    params = tmp_path / "params.txt"
    voxel = 0.004
    params.write_text(f"s_SDFVoxelSize = {voxel}f;\ns_SDFTruncation = 0.02f;\ns_SDFTruncationScale = 0.01f;\ns_hashNumSDFBlocks = 200000;\n")
    r = subprocess.run([os.path.join(BIN, "fuse"), str(params), str(sens)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    vh, c0, c1, c2 = (tmp_path / f"scene_vh{s}.ply" for s in ("", "_clean", "_clean_1", "_clean_2"))
    r = subprocess.run([os.path.join(BIN, "meshclean"), "-i", str(vh), "-o", str(c0), "-m", "vc", "-s", os.path.join(GOLDEN, "clean.mlx")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for src, dst in ((c0, c1), (c1, c2)):
        r = subprocess.run([os.path.join(BIN, "meshsimplify"), "-i", str(src), "-o", str(dst), "-m", "vc", "-s", os.path.join(GOLDEN, "simplify.mlx")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "Quadric Edge Collapse Decimation" in r.stdout and "Merge Close Vertices" in r.stdout and "Remove Isolated pieces" in r.stdout
        print(r.stdout)
    # the oracle chain, written by the same PLY writer
    x, c, t = meshclean.load_rgb(str(c0))
    for dst in (c1, c2):
        x, c, t, _, _ = sb.oracle_simplify(x, t, c, after=AFTER)
        want = tmp_path / "want.ply"
        save_ply(want, x, c, t)
        assert dst.read_bytes() == want.read_bytes(), dst.name
    assert len(t) > 0
    r = subprocess.run([os.path.join(BIN, "segmentator"), str(c2)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seg = np.array(json.loads((tmp_path / "scene_vh_clean_2.0.010000.segs.json").read_text())["segIndices"])
    assert len(seg) == len(x) and (seg == ob.oracle_segment(x, t)).all()
    # geometric sanity: every decimated vertex lies within 2 voxels of the clean.mlx surface (sampled at 1/8 of its edges)
    ix, _, it = meshclean.load_rgb(str(c0))
    w = np.array([(i / 8, j / 8) for i in range(9) for j in range(9 - i)])
    tri_p = ix[it].astype(np.float64)
    samples = (tri_p[:, None, 0] + w[None, :, :1] * (tri_p[:, None, 1] - tri_p[:, None, 0]) + w[None, :, 1:] * (tri_p[:, None, 2] - tri_p[:, None, 0]))
    d, _ = cKDTree(samples.reshape(-1, 3)).query(x.astype(np.float64))
    print(f"decimated {len(ix)} -> {len(x)} vertices; distance to the clean surface: max {d.max() * 1e3:.2f} mm, mean {d.mean() * 1e3:.3f} mm")
    assert d.max() <= 2 * voxel
    # without -s the simplify.mlx defaults; without -m vc no colour (white)
    r = subprocess.run([os.path.join(BIN, "meshsimplify"), "-i", str(c0), "-o", str(tmp_path / "b.ply")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    bx, bc, bt = meshclean.load_rgb(str(tmp_path / "b.ply"))
    ox, _, ot, _, _ = sb.oracle_simplify(ix, it, None, after=AFTER)
    assert bx.tobytes() == ox.tobytes() and bt.tobytes() == ot.tobytes() and (bc == 255).all()
    r = subprocess.run([os.path.join(BIN, "meshsimplify"), "-i", str(c0), "-o", str(tmp_path / "c.ply"), "-s", os.path.join(GOLDEN, "clean.mlx")],
                       capture_output=True, text=True)
    assert r.returncode != 0 and "Quadric Edge Collapse Decimation" in r.stderr
